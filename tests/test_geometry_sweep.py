"""The frame path at every frame geometry the reference accepts: any w, h > 0 with w h <= 4000 x 4000 (MAX_ARR_SIZE).

The width is (int) (2 fs / (fv h)), so real front ends reach both ends of that range: 7 columns from an RTL-SDR at 250 kS/s,
71 at 2.4 MS/s (1125 lines), 8271 from 200 MS/s at 806 lines, 16666 from a B210 at 50 MS/s and 100 lines.  Every other test runs
frames 100 to 1481 pixels wide; this file sweeps the geometries below through
  (a) the compiled reference against the C restatement (CPU), so that the GPU comparisons rest on a pinned oracle;
  (b) the GPU frame stage against orc.best(), bit for bit, two batches (F = 1, then 5) so that the state crosses a batch boundary;
  (c) the wide cases with the literal cluster search only and with the serial chains only, and a frame that fails the sync
      search's exactness certificate in the middle of a 16666- and a 12698-column batch;
  (d) tsdrgpu_gaussianblur on strips up to 33332 long;
  (e) the streaming pipeline at 7, 71 and 16666 columns, and through narrow -> wide -> narrow resolution changes;
  (f) the host library at 16666 columns, and its refusal of w h > 4000 x 4000 and w = 0.
Frames and sync integers bit-exact; the auto-gain levels exact.  The SNR is not compared: it is computed only with
TSDRGPU_FS_COMPUTE_SNR, which these runs leave off (the reference's value is dead, dsp.c:234).
"""
import ctypes as C
import functools
import os
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not orc.have_ref(), reason="oracle/_ref not built (needs the reference sources)")

GEOMETRIES = (
    # degenerate: half = size >> 1 is 0..2, so most candidate lists are empty; size 1 clamps the carried strip to 0 on every
    # other frame (a zero-length strip: NaN scores); blur strips shorter than its 5 taps; minsize = 0 on both axes
    [(1, 1), (1, 7), (7, 1), (2, 3), (3, 2), (5, 5)]
    # narrow and tall: every residue of w mod 4 (16-byte rows or not), both sides of the collapse's 32-column tensor boxes
    # (most columns of a box outside the frame), minsize_x = (int) (w * 0.05f) = 0, 1 and 3
    + [(w, 1125) for w in (4, 7, 8, 12, 31, 33, 35, 36, 64, 65, 71)]
    # short: minsize_y = (int) (h * 0.01f) is 0 or 1; rows fewer than one 32-row box; a one-row frame
    + [(740, h) for h in (1, 2, 3, 17, 99, 100, 101)]
    # wide: the sync search keeps one record at a time in shared memory (w + h > ~6000), and past w + h = 16384 reads the
    # records in global memory; at, around and past the 8192 columns the search used to be limited to
    + [(w, h) for w in (5000, 8191, 8192, 8193, 12698, 16666) for h in (100, 525)]
    # X310 / 4 x 50 MS/s superbandwidth at XGA timing; the reference's largest frame
    + [(8271, 806), (4000, 4000)]
    # tall: a long row strip, and a long row strip beside a two-column one
    + [(64, 10000), (2, 8193)]
)
GEOM_IDS = [f"{w}x{h}" for w, h in GEOMETRIES]
WIDE = [(w, h) for w, h in GEOMETRIES if w >= 5000 or h > 8192]      # every geometry past two records in 96 KB (w + h > 5992)

# (low-pass before sync, auto-gain after processing, autoshift, motion blur)
FLAGSETS = {
    "default": (1, 0, 1, 0.0),      # the GUI's order (normalise-on-load collapse, motion blur 0)
    "aap_blur": (1, 1, 1, 0.3),     # auto-gain after processing, motion blur 0.3
    "noshift": (1, 0, 0, 0.0),      # autoshift off: green marker lines on a copy
}
NF = 6                              # batches of 1 and 5 frames
FS, FV = 8_000_000, 60.0            # the oracle post-processor's configuration (used by the PLL only, which is off)


@functools.lru_cache(maxsize=2)
def frames_of(w, h):
    """NF frames whose picture drifts by 3 columns and 1 row per frame."""
    return tuple(synth.video_like_frame(w, h, seed=1000 + 7 * w + h + k, shift_x=(w // 3 + 3 * k) % w, shift_y=(h // 4 + k) % h)
                 for k in range(NF))


@functools.lru_cache(maxsize=4)
def oracle_run(kind, w, h, flagset):
    """[(frame, result)] of NF frames through one post-processor of `kind` ("best", "port" or "ref")."""
    O = {"best": orc.best, "port": orc.port, "ref": orc.ref}[kind]()
    lpbs, aap, autoshift, mb = FLAGSETS[flagset]
    po = O.postprocessor(FS, h, FV, autoshift, 0)
    return tuple(po.run(f, w, h, mb, 0.1, lpbs, aap) for f in frames_of(w, h))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def same_bits(a, b, what):
    assert a.shape == b.shape, what
    bad = np.flatnonzero(bits(a) != bits(b))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} differ, first at {bad[:5]}: {a[bad[:5]]} vs {b[bad[:5]]}"


# ------------------------------------------------------------------------------------------------ (a) oracle pinning, CPU
@needs_ref
@pytest.mark.parametrize("flagset", list(FLAGSETS))
@pytest.mark.parametrize("w,h", GEOMETRIES, ids=GEOM_IDS)
def test_restatement_matches_the_reference_at_every_geometry(w, h, flagset):
    """The compiled reference and the C restatement (orc.best() on a machine without the former) over NF drifting frames: frames,
    every sync field and the auto-gain state bit for bit."""
    P, R = oracle_run("port", w, h, flagset), oracle_run("ref", w, h, flagset)
    for k, ((a, ra), (b, rb)) in enumerate(zip(P, R)):
        same_bits(a, b, f"{w}x{h} {flagset} frame {k}")
        assert ra.x.astuple() == rb.x.astuple() and ra.y.astuple() == rb.y.astuple(), (k, ra.x.astuple(), rb.x.astuple())
        for fld in ("avg_speed", "pll_state", "lastmax", "lastmin", "width_after", "autogain_callback_fired"):
            assert getattr(ra, fld) == getattr(rb, fld), (k, fld)
        assert ra.snr == rb.snr or (np.isnan(ra.snr) and np.isnan(rb.snr)), k


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def frame_stage_case(gpu, w, h, flagset, overlap=False, offset=0, frames=None, batches=(1, NF - 1)):
    """Frames through the GPU frame stage in `batches` (tsdrgpu_framestage_run_async, what the pipeline calls), input and output
    `offset` floats past a 16-byte boundary; every frame, result and auto-gain report against orc.best()."""
    import torch
    from tempestsdr_b200.api import PostProcessFlags
    from tests.test_production_batches import assert_same_result, results_of, run_async
    lpbs, aap, autoshift, mb = FLAGSETS[flagset]
    if frames is None:
        frames, want = frames_of(w, h), oracle_run("best", w, h, flagset)
    else:
        po = orc.best().postprocessor(FS, h, FV, autoshift, 0)
        want = [po.run(f, w, h, mb, 0.1, lpbs, aap) for f in frames]
    n = w * h
    pg = gpu.post_processor()
    pg.set_overlap(overlap)
    flags = PostProcessFlags(autoshift=bool(autoshift), lowpass_before_sync=bool(lpbs), autogain_after_proc=bool(aap))
    keep, k = [], 0
    for nb in batches:
        xb = torch.full((offset + nb * n,), float("nan"), device="cuda")
        xb[offset:] = dev(np.concatenate(frames[k:k + nb]))
        ob = torch.full((offset + nb * n + 1,), -7.0, device="cuda")         # one guard float past the end
        x, out = xb[offset:], ob[offset:offset + nb * n]
        keep.append((xb, ob, out, nb) + run_async(gpu, pg, x, nb, w, h, mb, flags, out))
        k += nb
    pg.join()
    torch.cuda.synchronize()
    k = 0
    for xb, ob, out, nb, res, ag in keep:
        assert ob[-1].item() == -7.0 and (offset == 0 or ob[0].item() == -7.0), "written outside the output"
        got = out.cpu().numpy().reshape(nb, -1)
        rs = results_of(res, nb)
        for i in range(nb):
            wf, wr = want[k]
            what = f"{w}x{h} {flagset} overlap={overlap} offset={offset} frame {k}"
            same_bits(got[i], wf, what)
            assert_same_result(rs[i], wr, what)
            assert ag[i] == wr.autogain_callback_fired, what
            k += 1
    del pg


# ------------------------------------------------------------------------------------------------ (b) frame stage, GPU
def _stage_variants():
    out = []
    for w, h in GEOMETRIES:
        names = ["default", "overlap"] + (["offset"] if w % 4 == 0 else [])
        if w * h < 4000 * 4000:                               # the largest frame: default flags only, to keep the file's runtime down
            names += ["aap_blur", "noshift"]
        out += [pytest.param(w, h, v, id=f"{w}x{h}-{v}") for v in names]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("w,h,variant", _stage_variants())
def test_frame_stage_at_every_geometry(gpu, w, h, variant):
    """The GPU frame stage against the reference at every geometry: default order (with and without the side-stream overlap, and
    with input and output one float off their 16-byte boundary where rows could be 16 bytes), auto-gain after processing with
    motion blur, and autoshift off."""
    flagset = variant if variant in FLAGSETS else "default"
    frame_stage_case(gpu, w, h, flagset, overlap=variant == "overlap", offset=1 if variant == "offset" else 0)


# ------------------------------------------------------------------------------------------------ (c) the sync search's other paths
def bad_frame_batch(w, h):
    """Six drifting frames; frame 3 has 15 columns of zeros around one pixel of 1e-30, so its blurred column strip spans ~2^100
    binades, far past the sync search's exactness certificate, while the other frames' strips span a few."""
    frames = [synth.video_like_frame(w, h, seed=3000 + k, shift_x=(w // 3 + 3 * k) % w, shift_y=(h // 4 + k) % h) for k in range(NF)]
    f = frames[3].reshape(h, w)
    f[:, 200:215] = 0.0
    f[0, 207] = 1e-30
    return frames


def wide_cases():
    """The wide geometries with the default flags, and the bad-frame batches (auto-gain after processing, so that the collapse
    sees the raw values), in one process: run with TSDRGPU_SYNC_NO_SPEC / TSDRGPU_SYNC_SERIAL set, which are read once."""
    from tempestsdr_b200 import api
    gpu = api.Context(0)
    for w, h in WIDE:
        frame_stage_case(gpu, w, h, "default")
    for w, h in ((16666, 100), (12698, 100)):
        frame_stage_case(gpu, w, h, "aap_blur", frames=bad_frame_batch(w, h), batches=(2, 4))


def test_bad_frame_fails_the_certificate_alone():
    """CPU: in bad_frame_batch, frame 3 and no other fails the exactness certificate, so the GPU runs hand it (alone) to the
    serial chains, on strips longer than 8192."""
    from tests.test_sync_handoff_cases import exact_ok
    for w, h in ((16666, 100), (12698, 100)):
        ok = [exact_ok(orc.port().average_v_h(f, w, h)[0])[0] for f in bad_frame_batch(w, h)]
        assert ok == [True, True, True, False, True, True], (w, h, ok)


@pytest.mark.gpu
def test_bad_frame_mid_batch_at_wide_geometries(gpu):
    for w, h in ((16666, 100), (12698, 100)):
        frame_stage_case(gpu, w, h, "aap_blur", frames=bad_frame_batch(w, h), batches=(2, 4))


@pytest.mark.gpu
@pytest.mark.parametrize("hook", ["TSDRGPU_SYNC_NO_SPEC", "TSDRGPU_SYNC_SERIAL"])
def test_wide_geometries_on_the_other_sync_paths(hook):
    """The wide cases with the literal cluster search only (no speculation tables), and with the serial chains only."""
    r = subprocess.run([sys.executable, "-c", "from tests.test_geometry_sweep import wide_cases; wide_cases(); print('cases ok')"],
                       capture_output=True, text=True, timeout=900, cwd=ROOT, env=dict(os.environ, **{hook: "1"}))
    assert r.returncode == 0 and "cases ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])


# ------------------------------------------------------------------------------------------------ (d) gaussianblur
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 8192, 16384, 16385, 33332])
def test_gaussianblur_at_every_strip_length(gpu, n):
    s = np.random.default_rng(n).uniform(0, 5, n).astype(np.float32)
    same_bits(gpu.gaussianblur(dev(s)).cpu().numpy(), orc.best().gaussianblur(s), f"gaussianblur n={n}")


# ------------------------------------------------------------------------------------------------ (e) streaming pipeline
STREAMS = {  # name: (samplerate, lines, batch_frames, items per call, calls, int8 ingest)
    "rtl_250k_w7": (250_000, 1125, 1, 16384, 8, True),
    "rtl_2m4_w71": (2_400_000, 1125, 16, 512 * 1024, 8, False),     # r = 639/320: every other block meets the stale slot
    "b210_50m_w16666": (50_000_000, 100, 1, 512 * 1024, 18, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(STREAMS))
def test_pipeline_at_narrow_and_wide_geometries(name):
    from tempestsdr_b200 import pipeline
    from tests.test_pipeline_gpu import run_oracle_stream
    fs, h, bf, items, calls, raw = STREAMS[name]
    O = orc.best()
    w, _, _ = O.geometry(fs, h, FV)
    assert w == int(name.rsplit("_w", 1)[1])
    iq = synth.video_like_iq(calls * items // 2, fs, w, h, FV, seed=17, snr_db=25.0)
    if raw:
        q = np.clip(np.round(iq / np.abs(iq).max() * 110.0), -128, 127).astype(np.int8)
        iq = (q.astype(np.float64) / 128.0).astype(np.float32)           # TSDRPlugin_RawFile.c:247
    _, want = run_oracle_stream(O, [iq[k * items:(k + 1) * items] for k in range(calls)], fs, h, FV)
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=FV, batch_frames=bf, batch_blocks=10 * bf, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: got.append((f.copy(), ww, hh)))
    for k in range(calls):
        if raw:
            p.process_raw(q[k * items:(k + 1) * items].copy(), 0)
        else:
            p.process(iq[k * items:(k + 1) * items].copy(), 0)
    p.flush()
    p.close()
    assert len(got) >= max(4, 2 * bf) and len(got) <= len(want), (len(got), len(want))
    for k, (g, ww, hh) in enumerate(got):
        assert (ww, hh) == (w, h)
        same_bits(g, want[k], f"{name} frame {k}")


def test_the_71_column_stream_meets_the_stale_slot():
    """CPU: at 2.4 MS/s and 1125 lines the resampler's ratio is 639/320, and every other 4000-sample block ends where the reference
    writes one pixel fewer than it sizes its output for: the stream above runs through the slot the CUDA path fills with 0.0f."""
    O, P = orc.best(), orc.port()
    fs, h = 2_400_000, 1125
    w, _, _ = O.geometry(fs, h, FV)
    block = int(0.1 * fs / FV)
    x = np.abs(synth.noise_iq(40 * block, seed=5).view(np.complex64)).astype(np.float32)[:40 * block]
    rs = P.resampler()
    short = sum(rs.run(x[k * block:(k + 1) * block], w * h * FV, fs).size > rs.last_emitted for k in range(40))
    assert (w, block, short) == (71, 4000, 20)


# narrow -> wide -> narrow at 2.4 MS/s: 71 x 1125, then 20000 x 4 (w + h > 16384: the sync records in global memory, fs_sync's
# serial-chain scratch and the screen buffer grow), then 71 x 1125 again (records back in shared memory)
RESOLUTIONS = {10: (4, FV), 20: (1125, FV)}


@pytest.mark.gpu
def test_pipeline_through_resolution_changes():
    """set_resolution between process() calls: the groups of blocks after it are resampled and cut into frames with the new geometry,
    pixels left from the old one included; one frame stage follows the geometry.  Frames bit-exact against the replay."""
    from tempestsdr_b200 import pipeline
    from tests.test_pipeline_gpu import run_oracle_stream
    O = orc.best()
    fs, items, calls = 2_400_000, 65536, 30
    iq = synth.video_like_iq(calls * items // 2, fs, 71, 1125, FV, seed=29, snr_db=25.0)
    blocks = [iq[k * items:(k + 1) * items] for k in range(calls)]
    _, want = run_oracle_stream(O, blocks, fs, 1125, FV, resolutions=RESOLUTIONS)
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=1125, refreshrate=FV, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_frame=lambda f, ww, hh: got.append((f.copy(), ww, hh)))
    for k, b in enumerate(blocks):
        if k in RESOLUTIONS:
            p.flush()
            p.set_resolution(*RESOLUTIONS[k])
            assert p.geometry()[:2] == (O.geometry(fs, RESOLUTIONS[k][0], FV)[0], RESOLUTIONS[k][0])
        p.process(b.copy(), 0)
    p.flush()
    p.close()
    assert len(got) == len(want), (len(got), len(want))
    sizes = [(ww, hh) for _, ww, hh in got]
    assert sizes[0] == (71, 1125) and (20000, 4) in sizes and sizes[-1] == (71, 1125), sizes
    for k, (g, ww, hh) in enumerate(got):
        same_bits(g, want[k], f"resolution change frame {k} ({ww}x{hh})")


# ------------------------------------------------------------------------------------------------ (f) host library
def _host():
    from tests.test_host_library import MINE, PLOT_CB, VALUE_CB, bind
    return MINE, bind, VALUE_CB, PLOT_CB


@needs_ref
def test_host_library_refuses_what_the_reference_refuses(tmp_path):
    """w h > 4000 x 4000 (one line at 0.5 Hz from 8 MS/s: w = 32 000 000) and w = 0 (a million lines at 60 Hz) make
    tsdr_readasync return TSDR_WRONG_VIDEOPARAMS with the reference's text, before any device is touched."""
    MINE, bind, VALUE_CB, PLOT_CB = _host()
    from tests.test_host_library import FRAME_CB
    raw = tmp_path / "iq.raw"
    synth.noise_iq(4096, seed=3).tofile(raw)
    nv, npl = VALUE_CB(lambda *a: None), PLOT_CB(lambda *a: None)
    results = {}
    for name, path in (("mine", MINE), ("ref", orc.REF_LIB_SO)):
        lib = bind(path)
        t = C.c_void_p()
        lib.tsdr_init(C.byref(t), nv, npl, None)
        assert lib.tsdr_loadplugin(t, orc.REF_RAWFILE_NOPACE_SO.encode(), f'"{raw}" 8000000 float'.encode()) == 0
        r = []
        for hgt, fv in ((1, 0.5), (1_000_000, 60.0)):
            assert lib.tsdr_setresolution(t, hgt, fv) == 0
            r.append((hgt, lib.tsdr_readasync(t, FRAME_CB(lambda *a: None), None), lib.tsdr_getlasterrortext(t), lib.tsdr_isrunning(t)))
        lib.tsdr_unloadplugin(t)
        lib.tsdr_free(C.byref(t))
        results[name] = r
    assert results["mine"] == results["ref"]
    assert [x[1] for x in results["mine"]] == [2, 2]                  # TSDR_WRONG_VIDEOPARAMS


@pytest.mark.gpu
@needs_ref
def test_host_library_delivers_frames_wider_than_8192(tmp_path, monkeypatch):
    """tsdr_readasync + the reference's RawFile plugin at 50 MS/s and 100 lines (16666 x 100 frames): the first frames equal
    the stage-wise replay of the reference, which the pipeline matches bit for bit (test_pipeline_at_narrow_and_wide_geometries)."""
    MINE, bind, VALUE_CB, PLOT_CB = _host()
    from tests.test_host_library import FRAME_CB
    from tests.test_pipeline_gpu import run_oracle_stream
    O = orc.best()
    fs, h = 50_000_000, 100
    w, _, _ = O.geometry(fs, h, FV)
    assert w == 16666
    items, nblk = 512 * 1024, 14                          # SAMPLES_TO_READ_AT_ONCE of the plugin
    iq = synth.video_like_iq(nblk * items // 2, fs, w, h, FV, seed=23, snr_db=25.0)
    raw = tmp_path / "iq.raw"
    iq.tofile(raw)
    _, want = run_oracle_stream(O, [iq[k * items:(k + 1) * items] for k in range(nblk)], fs, h, FV)
    assert len(want) >= 3
    got = []
    monkeypatch.setenv("TSDR_NO_DROP", "1")
    lib = bind(MINE)
    t = C.c_void_p()
    nv, npl = VALUE_CB(lambda *a: None), PLOT_CB(lambda *a: None)
    fcb = FRAME_CB(lambda b, ww, hh, c: got.append((np.ctypeslib.as_array(b, shape=(ww * hh,)).copy(), ww, hh)))
    lib.tsdr_init(C.byref(t), nv, npl, None)
    lib.tsdr_setresolution(t, h, FV); lib.tsdr_motionblur(t, 0.0); lib.tsdr_setgain(t, 0.5)
    for pid, v in ((0, 1), (1, 0), (6, 1)):
        lib.tsdr_setparameter_int(t, pid, v)
    assert lib.tsdr_loadplugin(t, orc.REF_RAWFILE_SO.encode(), f'"{raw}" {fs} float'.encode()) == 0
    rc = []
    th = threading.Thread(target=lambda: rc.append(lib.tsdr_readasync(t, fcb, None)))
    th.start()
    deadline = time.time() + 120
    while len(got) < 2 and time.time() < deadline:
        time.sleep(0.05)
    assert lib.tsdr_stop(t) == 0
    th.join(timeout=60)
    lib.tsdr_free(C.byref(t))
    assert rc == [0] and len(got) >= 2, (rc, len(got))
    for k in range(2):
        g, ww, hh = got[k]
        assert (ww, hh) == (w, h)
        same_bits(g, want[k], f"host library frame {k}")
