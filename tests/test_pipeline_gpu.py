"""GPU: the streaming pipeline (process() -> frames) against the oracle driven stage by stage on one thread."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tempestsdr_b200 import synth

pytestmark = pytest.mark.gpu


class StaleZeroResampler:
    """The oracle's resampler with the slot the reference leaves stale set to 0.0f, as the CUDA path writes it (DESIGN.md §2: when
    (size - offset) * r lands exactly on an integer the reference's loop writes one pixel fewer than it sizes its output for, and
    that slot keeps stale buffer content).  The pinned restatement runs beside it on the same blocks to say where that happens."""

    def __init__(self, O):
        self.rs, self.port = O.resampler(), orc.port().resampler()

    def run(self, x, up, down):
        out = self.rs.run(x, up, down)
        self.port.run(x, up, down)
        out[self.port.last_emitted:] = 0.0
        return out


def run_oracle_stream(O, iq_blocks, fs, h, fv, plots=True, resolutions=None):
    """Single-threaded replay of process() -> decimatingthread -> postprocessingthread with the reference stages.
    resolutions: {index of an IQ block: (height, refresh rate)} set before that block is processed (set_resolution between
    process() calls): groups of ten decimator blocks resampled after it use the new geometry, and frames are cut with the
    geometry of the group that completed them, pixels left from the old geometry included.  Returns (width at the end, frames)."""
    w, _, _ = O.geometry(fs, h, fv)
    rs = StaleZeroResampler(O); pp = O.postprocessor(fs, h, fv, 1, 0)
    decim = np.zeros(0, np.float32); pix = np.zeros(0, np.float32)
    frames = []
    for i, iq in enumerate(iq_blocks):
        if resolutions and i in resolutions:
            h, fv = resolutions[i]
            w, _, _ = O.geometry(fs, h, fv)
        n = w * h
        block = int(0.1 * fs / fv)
        decim = np.concatenate([decim, O.am_demod(iq)])
        while decim.size >= 10 * block:
            for k in range(10):
                pix = np.concatenate([pix, rs.run(decim[k * block:(k + 1) * block], w * h * fv, fs)])
            decim = decim[10 * block:]
            while pix.size >= n:
                out, res = pp.run(pix[:n], w, h, 0.0, 0.1, 1, 0)
                frames.append(out); pix = pix[n:]
    return w, frames


def test_pipeline_matches_stagewise_oracle():
    from tempestsdr_b200 import pipeline
    O = orc.best()
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = O.geometry(fs, h, fv)
    nblk, items = 24, 65536
    iq_all = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=21)
    blocks = [iq_all[k * items:(k + 1) * items].copy() for k in range(nblk)]
    _, want = run_oracle_stream(O, blocks, fs, h, fv)
    got, plots, values = [], [], []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1},
                          on_frame=lambda f, ww, hh: got.append(f.copy()),
                          on_plot=lambda pid, off, v, sr: plots.append((pid, off, v.copy())),
                          on_value=lambda vid, a, b: values.append((vid, a, b)))
    for b in blocks:
        p.process(b, 0)
    p.flush()
    st = p.stats()
    assert st.frames_dropped == 0 and st.frames_delivered == len(want) > 3
    for k, (g, wv) in enumerate(zip(got, want)):
        assert np.array_equal(g.view(np.uint32), wv.view(np.uint32)), f"frame {k}"
    # autocorrelation plots: capture size 3.1*fs/55 = 112727 samples -> several captures
    cap = int(3.1 * fs / 55.0)
    assert st.captures == (nblk * items // 2) // cap and len(plots) == 2 * st.captures
    mag = O.am_demod(iq_all)
    det = O.framerate_detector()
    for c in range(st.captures):
        (fo, fp), (lo, lp), calls = det.run(fs, mag[c * cap:(c + 1) * cap])
    last_frame = [v for pid, off, v in plots if pid == 0][-1]
    assert np.max(np.abs(last_frame - fp)) <= 1e-5 * np.max(np.abs(fp))      # tolerance: 1e-5 of the plot peak
    assert (2, 0.0, float(st.captures)) in values
    p.close()


def test_pipeline_autocorr_dump_parameter(tmp_path, monkeypatch):
    """PARAM_AUTOCORR_DUMP (frameratedetector.c:110-116): set once -> the next capture's autocorrelation lands in autocorr.csv in the
    working directory, value id 5 (VALUE_ID_AUTOCORRECT_DUMPED) is announced once before that capture's plots, the parameter clears
    itself, plots and frames go on as without it."""
    from tempestsdr_b200 import pipeline
    monkeypatch.chdir(tmp_path)
    fs, h, fv = 2_000_000, 125, 60.0
    iq_all = synth.video_like_iq(6 * 65536, fs, 533, h, fv, seed=5)
    events = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True, params={"autoshift": 1, "lowpass_before_sync": 1},
                          on_plot=lambda pid, off, v, sr: events.append(("plot", pid)), on_value=lambda vid, a, b: events.append(("value", vid)))
    p.set_param("autocorr_dump", 1)
    for k in range(12):
        p.process(iq_all[k * 65536:(k + 1) * 65536].copy(), 0)
    p.flush()
    st = p.stats()
    p.close()
    assert st.captures >= 2
    dumped = [i for i, e in enumerate(events) if e == ("value", 5)]
    assert len(dumped) == 1 and dumped[0] < events.index(("plot", 0))
    lines = (tmp_path / "autocorr.csv").read_text().splitlines()
    cap = int(3.1 * fs / 55.0)
    assert lines[0] == "ms, dB" and len(lines) - 1 == (1 << (int(2 * cap).bit_length() - 1)) // 4


def run_oracle_stream_pll(O, iq_blocks, fs, h, fv):
    """The same single-threaded replay with the PLL switched on (syncdetector.c:133-153): after every frame the refresh rate
    the oracle's post-processor holds moves, and the NEXT group of ten decimator blocks is cut and resampled with it -- the
    deterministic order the pipeline documents (the threaded reference races here, SURVEY F9)."""
    w, _, _ = O.geometry(fs, h, fv)
    rs = O.resampler(); pp = O.postprocessor(fs, h, fv, 1, 1)
    decim = np.zeros(0, np.float32); pix = np.zeros(0, np.float32)
    fv_live, w_live = fv, w
    frames, rates = [], []
    for iq in iq_blocks:
        decim = np.concatenate([decim, O.am_demod(iq)])
        while True:
            block = int(0.1 * fs / fv_live)
            if decim.size < 10 * block:
                break
            w_grp, fv_grp = w_live, fv_live
            for k in range(10):
                pix = np.concatenate([pix, rs.run(decim[k * block:(k + 1) * block], float(w_grp * h) * fv_grp, fs)])
            decim = decim[10 * block:]
            n = w_grp * h
            while pix.size >= n:
                out, res = pp.run(pix[:n], w_grp, h, 0.0, 0.1, 1, 0)
                frames.append((out, w_grp)); pix = pix[n:]
                if res.pll_callback_fired:
                    rates.append(res.refreshrate_after)
                fv_live, w_live = res.refreshrate_after, res.width_after
    return frames, rates


@pytest.mark.parametrize("items", [65536, 200_000])
def test_pipeline_pll_writeback(items):
    """PARAM_INT_FRAMERATE_PLL = 1, the GUI's default (Main.java): every frame whose picture moved (vx != 0) moves the refresh
    rate (syncdetector.c:141-152), the decimator's next blocks are cut and resampled with the new rate (TSDRLibrary.c:335-340)
    and the host hears about it (value id 0).  Frames bit-exact, announced rates exactly equal, for two ways of cutting the
    stream into process() calls (the write-back is applied in stream order, not on a racing thread)."""
    from tempestsdr_b200 import pipeline
    O = orc.best()
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = O.geometry(fs, h, fv)
    total = 24 * 65536
    # the source's frame rate is 2500 ppm off the configured one: the picture drifts, vx != 0 on most frames
    iq_all = synth.video_like_iq(total // 2, fs, w, h, fv, seed=61, fv_ppm=2500.0)
    blocks = [iq_all[k:k + items].copy() for k in range(0, total, items)]
    want, want_rates = run_oracle_stream_pll(O, blocks, fs, h, fv)
    assert len(want_rates) >= 5 and len(set(want_rates)) >= len(want_rates) - 2
    got, values = [], []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, batch_blocks=10, block_when_busy=True,
                          params={"autoshift": 1, "framerate_pll": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: got.append((f.copy(), ww)), on_value=lambda vid, a, b: values.append((vid, a, b)))
    for b in blocks:
        p.process(b, 0)
    p.flush()
    assert len(got) == len(want) > 5
    for k, ((g, gw), (wv, ww)) in enumerate(zip(got, want)):
        assert gw == ww and np.array_equal(g.view(np.uint32), wv.view(np.uint32)), f"frame {k}"
    assert [a for vid, a, b in values if vid == 0] == want_rates
    assert p.geometry()[2] == want_rates[-1]
    p.close()


@pytest.mark.parametrize("name,nframes,batch", [("cfg2", 7, 2), ("cfg5", 3, 1), ("cfg1", 64, 16)])
def test_pipeline_at_baseline_shapes(name, nframes, batch):
    """The streaming pipeline at BASELINE's own shapes -- cfg2: 25 MS/s -> 740x1125 frames, cfg5: 50 MS/s -> 1481x1125, cfg1:
    8 MS/s -> 507x525 at the e2e benchmark's batch_frames=16, three batches -- fed in the RawFile plugin's block size (524 288
    floats): frames bit-exact against the stage-wise replay of the reference."""
    from tempestsdr_b200 import pipeline
    from tests.test_gpu_parity import CFGS
    O = orc.best()
    fs, h, fv = CFGS[name]
    w, _, _ = O.geometry(fs, h, fv)
    items = 512 * 1024
    pairs = (nframes * int(fs / fv) + 3 * int(0.1 * fs / fv))
    nblk = (2 * pairs + items - 1) // items
    raster = (800, 525) if name == "cfg1" else (2576, 1125)          # bench.py's raster per shape
    iq_all = synth.video_like_iq(nblk * items // 2, fs, *raster, fv, seed=73, snr_db=25.0)
    blocks = [iq_all[k * items:(k + 1) * items] for k in range(nblk)]
    _, want = run_oracle_stream(O, blocks, fs, h, fv)
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=batch, batch_blocks=10 * batch, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: got.append((f.copy(), ww, hh)))
    for b in blocks:
        p.process(b.copy(), 0)
    p.flush()
    assert nframes - 1 - batch <= len(got) <= len(want) and len(got) % batch == 0      # cfg1: 64 - 17 -> three batches of 16
    for k, (g, ww, hh) in enumerate(got):
        assert (ww, hh) == (w, h) and np.array_equal(g.view(np.uint32), want[k].view(np.uint32)), f"{name} frame {k}"
    p.close()


def test_pipeline_drop_resync_and_manual_sync():
    """Upstream sample drops discard up to the next multiple of `block` (dsp.c:313-368) so frames stay aligned."""
    from tempestsdr_b200 import pipeline
    O = orc.best()
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, pt = O.geometry(fs, h, fv)[0], None, O.geometry(fs, h, fv)[2]
    items = 65536
    iq_all = synth.video_like_iq(30 * items // 2, fs, w, h, fv, seed=22)
    blocks = [iq_all[k * items:(k + 1) * items].copy() for k in range(30)]
    block = int(round(((w * h) << 1) * pt))
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 0, "autocorr_plots_off": 1}, on_frame=lambda f, ww, hh: got.append(f.copy()))
    dropped = 12345
    diff = 0
    fed = []
    for k, b in enumerate(blocks):
        d = dropped if k == 7 else 0
        if k == 15:      # an EMPTY block that only reports a loss (TSDRPlugin_UHD.cpp:294 does this)
            diff = O.dropcomp_shift_with(diff, block, 777)
            diff, fwd, skip = O.dropcomp_add(diff, 0, block, True)
            p.process(np.zeros(0, np.float32), 777)
        # oracle bookkeeping for what the decimator receives
        diff = O.dropcomp_shift_with(diff, block, d)
        diff, fwd, skip = O.dropcomp_add(diff, items // 2, block, True)
        if fwd:
            fed.append(b[2 * skip:])
        p.process(b, d)
    p.flush()
    _, want = run_oracle_stream_flat(O, np.concatenate(fed), fs, h, fv)
    assert len(got) == len(want) > 3
    for k, (g, wv) in enumerate(zip(got, want)):
        assert np.array_equal(g.view(np.uint32), wv.view(np.uint32)), f"frame {k}"
    p.close()


def run_oracle_stream_flat(O, iq, fs, h, fv):
    w, _, _ = O.geometry(fs, h, fv)
    n = w * h
    block = int(0.1 * fs / fv)
    mag = O.am_demod(iq)
    rs = O.resampler(); pp = O.postprocessor(fs, h, fv, 0, 0)
    pix = []
    for k in range(mag.size // (10 * block) * 10):
        pix.append(rs.run(mag[k * block:(k + 1) * block], w * h * fv, fs))
    pix = np.concatenate(pix)
    frames = [pp.run(pix[k * n:(k + 1) * n], w, h, 0.0, 0.1, 0, 0)[0] for k in range(pix.size // n)]
    return w, frames


def superb_case(H, devices=None, fs=400_000, fv=50.0):
    """PARAM_AUTOCORR_SUPERRESOLUTION through the streaming pipeline: superb_run's state machine (gather H hops of 10 frames, 0.5 s
    pause and a retune after each, stitch) runs inside process(); the stitched signal then flows at H x the rate through the
    frame stages.  devices: None = all hops on one GPU (the reference's 4), else one hop per listed device (superb_mgpu.cu).
    fs / fv: the front end's rate and the refresh rate; 400 kS/s at 50 Hz gives 8000 samples per frame (nd = N/2), 819 200 S/s at
    50 Hz gives 16 384, a power of two (nd = N).  Returns nothing; asserts."""
    from tempestsdr_b200 import pipeline
    from tests import fft_model as fm
    from tests import superb_model as sm
    O = orc.best()
    h = 80
    sif = int(fs / fv)
    to_gather, to_pause = 10 * sif, int(0.5 * fs)
    items = 16384
    nblk = 2 * (H * (to_gather + to_pause) // (items // 2) + 8)
    iq_all = synth.video_like_iq(nblk * items // 2, fs, 200, 80, fv, seed=41, snr_db=25)
    blocks = [iq_all[k * items:(k + 1) * items].copy() for k in range(nblk)]
    retunes, frames = [], []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: frames.append((f.copy(), ww, hh)), on_retune=lambda off: retunes.append(off))
    if devices is not None:
        p.set_superb_devices(devices)
    p.set_param("superresolution", 1)
    # host-side replay of the reference's state machine (superbandwidth.c:179-254) to know what each hop must contain
    state, buffid, gathered, hops, cur = "gather", 0, 0, [], []
    expected_hops = None
    for b in blocks:
        p.process(b, 0)
        now = b.size // 2
        if expected_hops is not None:
            continue
        if state == "pause":
            gathered += now
            if gathered > to_pause:
                gathered, state = 0, "gather"
        if state == "gather":
            take = now if gathered + now < to_gather else to_gather - gathered
            cur.append(b[: 2 * take]); gathered += take
            if gathered == to_gather:
                hops.append(np.concatenate(cur)); cur = []; gathered = 0; buffid += 1
                if buffid == H:
                    expected_hops = hops
                else:
                    state = "pause"
    p.flush()
    st = p.stats()
    assert st.stitches >= 1 and retunes[:H - 1] == [(k - H // 2) * fs for k in range(1, H)]     # (hop - H/2) * samplerate (superbandwidth.c:241 for H = 4)
    wH, _, _ = O.geometry(H * fs, h, fv)
    assert p.geometry()[0] == wH and len(frames) >= 4 and frames[0][1] == wH
    # The stitched signal of the first round through the oracle's stages gives the same first frames.  Tolerance, derived: a stitched
    # sample is within e = C_OWN_MAX u log2(H N) rms of the model of the path's own dataflow (tests/test_superb_sweep.py), and that
    # model is within max|own - reference| of the reference's model, computed here on these hops; |.| moves nothing by more than its
    # argument does.  The resampler's weights sum to <= 1 per pixel, so pixels inherit e; auto-gain maps v -> (v - lastmin) / span
    # with lastmin and span = lastmax - lastmin each off by up to e, so a delivered pixel is off by at most 3 e / span (first
    # frames: span is still small because lastmax/lastmin start at 0 and move 10 % per frame).
    want_iq, offs = O.superb_ondataready(expected_hops, sif)
    mag = O.am_demod(want_iq)
    n_hop = fm.getrealsize(expected_hops[0].size // 2)
    ref, _ = sm.stitch_reference(expected_hops, sif, offsets=[int(o) for o in offs])
    if devices is None:
        own, _ = sm.stitch_one_gpu(expected_hops, sif, offsets=[int(o) for o in offs])
    else:
        own, ref = sm.stitch_sharded(expected_hops, [int(o) // 2 for o in offs]), np.abs(ref)
    e = sm.C_OWN_MAX * fm.U * fm.log2_of(H * n_hop) * fm.rms(ref) + float(np.max(np.abs(own - ref)))
    blockH = int(0.1 * H * fs / fv)
    rs = O.resampler(); pp = O.postprocessor(H * fs, h, fv, 1, 0, superres=1)
    pix = np.concatenate([rs.run(mag[k * blockH:(k + 1) * blockH], wH * h * fv, float(H * fs)) for k in range(mag.size // blockH // 10 * 10)])
    n = wH * h
    worst = 0.0
    for k in range(min(6, pix.size // n, len(frames))):
        ref, res = pp.run(pix[k * n:(k + 1) * n], wH, h, 0.0, 0.1, 1, 0)
        got = frames[k][0]
        tol = 3 * e / (res.lastmax - res.lastmin)
        err = float(np.max(np.abs(got - ref)))
        worst = max(worst, err / tol)
        assert err <= tol, f"frame {k}: {err} > {tol}"
    print(f"superbandwidth H={H} devices={devices}: worst error / derived bound = {worst:.3f}")
    p.close()


def test_pipeline_superbandwidth_mode():
    superb_case(4, None)


def test_pipeline_superbandwidth_mode_frames_of_a_power_of_two():
    """819 200 S/s at 50 Hz: 16 384 samples per frame divide 2N, so the alignment correlates N points (nd = N)."""
    superb_case(4, None, fs=819_200)


def _superb_sharded_case(H, fs):
    """superb_case with the hops sharded, in a process of its own: every rank's stream needs a hardware queue of its own when
    the ranks share a GPU."""
    import os, subprocess, sys
    ngpu = torch.cuda.device_count()
    devs = list(range(H)) if ngpu >= H else [0] * H
    r = subprocess.run([sys.executable, "-c", f"from tests.test_pipeline_gpu import superb_case; superb_case({H}, {devs}, fs={fs}); print('case ok')"],
                       capture_output=True, text=True, timeout=150, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32", TSDRGPU_SBM_TIMEOUT_MS="1500"))
    return r


@pytest.mark.parametrize("H", [2, 4])
def test_pipeline_superbandwidth_one_hop_per_device(H):
    """The same run with the hops sharded, one per device (tsdrgpu_pipeline_set_superb_devices -> superb_mgpu.cu).  On a box with
    >= H GPUs the devices are distinct (NVLink peer access); on a one-GPU box all ranks share device 0 -- same code, same flags,
    windows in one memory."""
    r = _superb_sharded_case(H, 400_000)
    assert r.returncode == 0 and "case ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])


@pytest.mark.parametrize("H", [2, 4])
def test_pipeline_superbandwidth_one_hop_per_device_frames_of_a_power_of_two(H):
    """The sharded run at 819 200 S/s and 50 Hz: 16 384 samples per frame divide 2N, so the alignment correlates N points."""
    r = _superb_sharded_case(H, 819_200)
    assert r.returncode == 0 and "case ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])


@pytest.mark.parametrize("inverted", [False, True])
def test_pipeline_argb_output_and_raw_int8_ingest(inverted):
    """SURVEY 8f-1 + 8f-2 through the streaming pipeline: int8 samples in (converted on the device), final int32 pixels out
    (the JNI glue's rule, TSDRLibraryNDK.c:222-283).  Expected: the oracle's stage-wise replay of the host-converted floats,
    pushed through the oracle's pixel rule with a persistent host pixel buffer."""
    from tempestsdr_b200 import pipeline
    O = orc.best()
    P = orc.port()                                         # the host pixel rule lives in the JNI glue: restated in the port only
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = O.geometry(fs, h, fv)
    nblk, items = 16, 65536
    iq = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=91)
    q = np.clip(np.round(iq / np.abs(iq).max() * 110.0), -128, 127).astype(np.int8)
    as_float = (q.astype(np.float64) / 128.0).astype(np.float32)           # TSDRPlugin_RawFile.c:247
    blocks_f = [as_float[k * items:(k + 1) * items] for k in range(nblk)]
    _, frames = run_oracle_stream(O, blocks_f, fs, h, fv)
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=4, batch_blocks=40, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: got.append(f.view(np.int32).copy()))
    p.set_output_argb(True, inverted)
    for k in range(nblk):
        p.process_raw(q[k * items:(k + 1) * items].copy(), 0)
    p.flush()
    assert 4 <= len(got) <= len(frames)
    for k, g in enumerate(got):
        assert np.array_equal(g, P.pixels_argb(frames[k], inverted)), f"frame {k}"
    p.close()


def test_pixels_argb_batch_keeps_transparent_pixels():
    from tempestsdr_b200 import _native
    from tempestsdr_b200.api import Context
    O = orc.port()
    gpu = Context(0)
    rng = np.random.default_rng(3)
    n, nf = 1000, 5
    f = rng.uniform(-0.2, 1.3, (nf, n)).astype(np.float32)
    f[:, ::7] = 2048.0; f[2, ::7] = 0.5; f[:, 3::11] = 512.0; f[1, 5::13] = 256.0; f[3, 1::17] = 1024.0
    d = torch.from_numpy(f.copy()).cuda()
    last = torch.zeros(n, dtype=torch.int32, device="cuda")
    gpu.chk(_native.lib().tsdrgpu_pixels_argb_batch(gpu._h, gpu.stream, d.data_ptr(), n, nf, 0, last.data_ptr()))
    got = d.view(torch.int32).cpu().numpy()
    prev = np.zeros(n, np.int32)
    for k in range(nf):
        want = O.pixels_argb(f[k], False).astype(np.int32)
        want[f[k] == 2048.0] = prev[f[k] == 2048.0]
        assert np.array_equal(got[k], want), f"frame {k}"
        prev = want
    assert np.array_equal(last.cpu().numpy(), prev)


def test_pipeline_optional_reports_snr_and_detected_mode():
    """8f-4 / 8f-3: with the reports on, the value callback also carries (4, snr) beside each auto-gain report -- the SNR of
    dsp_autogain_run (dsp.c:84-93) -- and (100, fps, height) after each pair of plots, the GUI's auto-resolution arithmetic."""
    import ctypes as C
    from tempestsdr_b200 import pipeline, _native
    O = orc.best()
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = O.geometry(fs, h, fv)
    nblk, items = 40, 65536
    iq_all = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=55)
    values, plots = [], []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1},
                          on_value=lambda vid, a, b: values.append((vid, a, b)),
                          on_plot=lambda pid, off, v, sr: plots.append((pid, off, v.copy(), sr)))
    p.set_reports(snr=True, detect_mode=True)
    for k in range(nblk):
        p.process(iq_all[k * items:(k + 1) * items].copy(), 0)
    p.flush()
    snrs = [a for vid, a, b in values if vid == 4]
    gains = [(a, b) for vid, a, b in values if vid == 3]
    assert len(snrs) == len(gains) >= 1 and all(np.isfinite(s) and s > 0 for s in snrs)
    # the oracle's SNR for the same frames: the report comes every AUTOGAIN_REPORT_EVERY_FRAMES+2 frames (dsp.c:231)
    pp = O.postprocessor(fs, h, fv, 1, 0)
    rs = O.resampler()
    mag = O.am_demod(iq_all)
    block = int(0.1 * fs / fv)
    pix = np.concatenate([rs.run(mag[k * block:(k + 1) * block], w * h * fv, fs) for k in range(mag.size // block)])
    want = []
    for k in range(pix.size // (w * h)):
        out, res = pp.run(pix[k * w * h:(k + 1) * w * h], w, h, 0.0, 0.1, 1, 0)
        if res.autogain_callback_fired:
            want.append(float(res.snr))
    assert len(want) >= len(snrs)
    for g, wv in zip(snrs, want):
        assert abs(g - wv) <= 1e-5 * abs(wv)               # float intermediates: 1e-5 relative (north_star)
    det = [(a, b) for vid, a, b in values if vid == 100]
    fplots = [(off, v, sr) for pid, off, v, sr in plots if pid == 0]
    lplots = [(off, v, sr) for pid, off, v, sr in plots if pid == 1]
    assert len(det) == len(fplots) == len(lplots) >= 1
    lib = _native.lib()
    for (fps, hh), (fo, fpv, sr), (lo, lpv, _) in zip(det, fplots, lplots):
        fi, li = int(np.argmax(fpv)), int(np.argmax(lpv))
        assert fps == float(sr) / float(fo + fi) and hh == float(int(np.floor((fo + fi) / float(lo + li) + 0.5)))
    p.close()
