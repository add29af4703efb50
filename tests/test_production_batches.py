"""GPU: the frame stage, the autocorrelation and the frame-rate detector at the batch sizes the product runs, against the oracle.

bench.py's DeviceStep hands the frame stage 64 frames per launch (740x1125, 1481x1125 or 507x525) with the sync search on the
side stream, and the frame-rate detector ~19 captures per launch on its own stream; the e2e legs run the pipeline with
batch_frames=16.  Several code paths only run at those sizes: the scalar fs_norm_lowpass path's second group of 16 frames, the
sync walker's hand-off to the cluster kernel in the middle of a batch, the batched half-size autocorrelation with odd capture
strides.  Tolerances follow tests/test_gpu_parity.py: sample->pixel->frame floats and sync integers bit-exact; autocorrelations
within 2e-6 of the zero-lag peak; running-mean plots within 1e-5 of the plot peak.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tempestsdr_b200 import synth
from tests.test_gpu_parity import CFGS, _close, _results_tuple, assert_same_bits, dev
from tests.test_sync_handoff_cases import case_frames

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


@pytest.fixture(scope="module")
def O():
    return orc.best()


def _lib():
    from tempestsdr_b200 import _native
    return _native.lib()


def run_async(gpu, pg, x, nframes, w, h, mb, flags, out):
    """tsdrgpu_framestage_run_async (what the pipeline calls): results land in page-locked memory once the stream that carries
    them -- the side stream in overlap mode -- has passed the call.  Returns (results buffer, auto-gain report flags)."""
    from tempestsdr_b200._native import FrameResult
    res = torch.empty(nframes * C.sizeof(FrameResult), dtype=torch.uint8).pin_memory()
    ag = (C.c_int32 * nframes)()
    gpu.chk(_lib().tsdrgpu_framestage_run_async(pg._h, gpu.stream, x.data_ptr(), nframes, w, h, mb, 0.1, flags.bits(), out.data_ptr(),
                                                res.data_ptr(), C.addressof(ag)))
    return res, ag


def results_of(res, nframes):
    from tempestsdr_b200._native import FrameResult
    return list((FrameResult * nframes).from_address(res.data_ptr()))


def assert_same_result(r, wr, what):
    assert _results_tuple(r) == wr.x.astuple() + wr.y.astuple(), f"sync state {what}"
    assert r.avg_speed == wr.avg_speed and r.pll_state == wr.pll_state, f"pll averages {what}"
    assert (r.lastmax, r.lastmin) == (wr.lastmax, wr.lastmin), f"auto-gain state {what}"


# ------------------------------------------------------------------------------------------------ 1. long frame-stage batches
# motion blur 0 is the benchmark's setting; with blur > 0 the low-pass screen value carried from frame to frame matters (with 0
# it is multiplied away), which is what the scalar path's carry across its 16-frame load groups has to get right
LONG = [("cfg1", 16, 0.0, False), ("cfg1", 17, 0.0, False), ("cfg1", 33, 0.0, False), ("cfg1", 64, 0.0, False),
        ("cfg1", 17, 0.4, False), ("cfg1", 64, 0.2, False), ("cfg1", 33, 0.3, True),
        ("cfg2", 17, 0.0, False), ("cfg2", 64, 0.0, False), ("cfg2", 64, 0.3, False), ("cfg5", 64, 0.0, False), ("cfg5", 64, 0.3, False)]


@pytest.mark.parametrize("name,nf,mb,aap", LONG, ids=[f"{n}-F{f}" + (f"-blur{m}" if m else "") + ("-aap" if a else "") for n, f, m, a in LONG])
def test_long_batches_match_the_reference_frame_by_frame(gpu, O, name, nf, mb, aap):
    """Two consecutive batches of nf drifting frames (vx != 0) through the frame stage with the side-stream overlap on and the
    GUI's default flags (autoshift, low-pass before sync; runs with motion blur, one with auto-gain after processing): every
    frame bit-exact, every field of every frame result exact.  cfg1 and cfg5 frames have an odd pixel count (fs_norm_lowpass's scalar
    path, 16 frames per load group: F = 17, 33, 64 run its second and later groups), cfg2 takes the 16-byte path."""
    from tempestsdr_b200.api import PostProcessFlags
    fs, hgt, fv = CFGS[name]
    w, _, _ = O.geometry(fs, hgt, fv)
    po = O.postprocessor(fs, hgt, fv, 1, 0)
    frames = [synth.video_like_frame(w, hgt, seed=900 + k, shift_x=(60 + 3 * k) % w, shift_y=(20 + k) % hgt) for k in range(2 * nf)]
    pg = gpu.post_processor()
    pg.set_overlap(True)
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True, autogain_after_proc=aap)
    keep = []
    for b in range(2):
        x = dev(np.concatenate(frames[b * nf:(b + 1) * nf]))
        out = torch.empty_like(x)
        keep.append((x, out) + run_async(gpu, pg, x, nf, w, hgt, mb, flags, out))
    pg.join(); torch.cuda.synchronize()
    vx = 0
    for b, (_, out, res, ag) in enumerate(keep):
        got = out.cpu().numpy().reshape(nf, -1)
        rs = results_of(res, nf)
        for i in range(nf):
            k = b * nf + i
            wf, wr = po.run(frames[k], w, hgt, mb, 0.1, 1, int(aap))
            assert_same_bits(got[i], wf, f"{name} F={nf} frame {k}")
            assert_same_result(rs[i], wr, f"{name} F={nf} frame {k}")
            assert ag[i] == wr.autogain_callback_fired, f"auto-gain report frame {k}"
            vx += abs(wr.x.vx)
    assert vx > 0                                          # the picture moved: the sync state carries real motion


def test_pll_over_a_64_frame_batch(gpu, O):
    """PLL on (syncdetector.c:133-153) across two 64-frame cfg1 batches: per frame, tsdrgpu_pll_step applied to the frame stage's
    vx / pll_state / avg_speed moves the refresh rate exactly as the oracle built with PLL = 1 does (the lock toggles)."""
    from tempestsdr_b200.api import PostProcessFlags
    fs, hgt, fv = CFGS["cfg1"]
    w, _, _ = O.geometry(fs, hgt, fv)
    po = O.postprocessor(fs, hgt, fv, 1, 1)
    speed = [3] * 16 + [0] * 14 + [1] * 18 + [6] * 16 + [0] * 20 + [2] * 44
    shifts = (60 + np.cumsum(speed)) % w
    frames = [synth.video_like_frame(w, hgt, seed=k, shift_x=int(sx), shift_y=20) for k, sx in enumerate(shifts)]
    want = [po.run(f, w, hgt, 0.0, 0.1, 1, 0) for f in frames]
    assert sum(r.pll_callback_fired for _, r in want) >= 20 and len({r.pll_state for _, r in want}) == 2
    pg = gpu.post_processor()
    rr = C.c_double(fv)
    for b in range(2):
        out, res = pg.process(dev(np.concatenate(frames[64 * b:64 * (b + 1)])), w, hgt, 0.0, 0.1, PostProcessFlags())
        out = out.cpu().numpy().reshape(64, -1)
        for i in range(64):
            k = 64 * b + i
            wf, wr = want[k]
            assert_same_bits(out[i], wf, f"frame {k}")
            assert_same_result(res[i], wr, f"frame {k}")
            moved = _lib().tsdrgpu_pll_step(C.byref(rr), res[i].x_vx, res[i].pll_state, res[i].avg_speed)
            assert moved == wr.pll_callback_fired and rr.value == wr.refreshrate_after, f"refresh rate after frame {k}"


# ------------------------------------------------------------------------------------------------ 2. mid-batch sync hand-offs
def handoff_gpu_case(name):
    """Both batches of a hand-off case (tests/test_sync_handoff_cases.py) through the GPU frame stage: frames and results bit-exact."""
    from tempestsdr_b200 import api
    from tempestsdr_b200.api import PostProcessFlags
    from tests.test_sync_handoff_cases import FS, FV, H
    O = orc.best()
    gpu = api.Context(0)
    w, h, batches, fl = case_frames(name)
    po = O.postprocessor(FS, H, FV, 1, 0)
    pg = gpu.post_processor()
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=bool(fl["lpbs"]), autogain_after_proc=bool(fl["aap"]))
    k = 0
    for frames in batches:
        out, res = pg.process(dev(np.concatenate(frames)), w, h, 0.0, 0.1, flags)
        out = out.cpu().numpy().reshape(len(frames), -1)
        for i, f in enumerate(frames):
            wf, wr = po.run(f, w, h, 0.0, 0.1, fl["lpbs"], fl["aap"])
            assert_same_bits(out[i], wf, f"{name} frame {k}")
            assert_same_result(res[i], wr, f"{name} frame {k}")
            k += 1


@pytest.mark.parametrize("mode", ["default", "no_spec", "serial"])
@pytest.mark.parametrize("name", ["leave_window", "halve", "bad_frame"])
def test_sync_handoff_mid_batch(name, mode, monkeypatch):
    """(a) the carried strip size leaves the speculation window at frame 4, (b) the strip size halves at frame 10, (c) frame 20
    fails the exactness certificate -- each precondition is asserted on the oracle by tests/test_sync_handoff_cases.py.  Bit-exact
    with the table walker (default), with the literal cluster search only (TSDRGPU_SYNC_NO_SPEC, read once per process: a process
    of its own) and with the serial chains only (TSDRGPU_SYNC_SERIAL, read per call)."""
    if mode == "no_spec":
        r = subprocess.run([sys.executable, "-c", f"from tests.test_production_batches import handoff_gpu_case; handoff_gpu_case({name!r}); print('case ok')"],
                           capture_output=True, text=True, timeout=300, cwd=ROOT, env=dict(os.environ, TSDRGPU_SYNC_NO_SPEC="1"))
        assert r.returncode == 0 and "case ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])
        return
    if mode == "serial":
        monkeypatch.setenv("TSDRGPU_SYNC_SERIAL", "1")
    handoff_gpu_case(name)


# ------------------------------------------------------------------------------------------------ 3. batched autocorrelation
_AC_CACHE = {}


def _ac_captures(O, size, batch=3):
    if size not in _AC_CACHE:
        caps = [np.abs(synth.noise_iq(size, seed=size + b)[:size]).astype(np.float32) for b in range(batch)]
        _AC_CACHE.clear()
        _AC_CACHE[size] = (caps, [O.autocorrelation(c) for c in caps])
    return _AC_CACHE[size]


@pytest.mark.parametrize("size", [450_910, 1_409_090, 2_818_182])
@pytest.mark.parametrize("layout", ["even_stride", "odd_stride", "base_4_aligned"])
def test_autocorrelation_batch_capture_by_capture(gpu, O, size, layout, monkeypatch):
    """tsdrgpu_autocorrelation_batch (the public C-ABI; the API wants an even size) on 3 captures: cfg2's capture size and even
    sizes next to cfg1's / cfg5's.  The capture stride is even (16-byte complex loads), odd (every other capture starts on an odd
    sample: FftPass.in_real = 2 pair loads) or even from a base that is only 4-byte aligned (pair loads again).  Each answer
    within 2e-6 of its own capture's zero-lag peak of the oracle, the untransformed tail bit-exact; TSDRGPU_AUTOCORR_GROUP = 1 and
    2 (captures per pair of work buffers) give bit-identical answers."""
    lib = _lib()
    batch = 3
    caps, want = _ac_captures(O, size, batch)
    stride = size + (1 if layout == "odd_stride" else 2)
    off = 1 if layout == "base_4_aligned" else 0
    buf = torch.full((off + batch * stride + 8,), float("nan"), device="cuda")
    for b, c in enumerate(caps):
        buf[off + b * stride: off + b * stride + size] = dev(c)
    base = buf.data_ptr() + 4 * off
    n = gpu.fft_getrealsize(size)

    def run():
        ans = torch.full((2 * size * batch,), float("nan"), device="cuda")
        gpu.chk(lib.tsdrgpu_autocorrelation_batch(gpu._h, gpu.stream, ans.data_ptr(), base, size, batch, stride))
        return ans.cpu().numpy().reshape(batch, -1)

    got = run()
    for b in range(batch):
        _close(got[b][: 2 * n], want[b][: 2 * n], 2e-6, f"autocorrelation batch {size} {layout} capture {b}")     # 2e-6 of the peak
        assert_same_bits(got[b][2 * n:], want[b][2 * n:], f"autocorr tail {size} {layout} capture {b}")
    for g in ("1", "2"):
        monkeypatch.setenv("TSDRGPU_AUTOCORR_GROUP", g)
        assert_same_bits(run(), got, f"TSDRGPU_AUTOCORR_GROUP={g} {size} {layout}")


# ------------------------------------------------------------------------------------------------ 4. the frame-rate detector in batches
FRD = {"cfg2": (2576, 1125), "cfg5": (2576, 1125), "cfg1": (800, 525)}      # bench.py's raster per shape


@pytest.mark.parametrize("name", list(FRD))
def test_framerate_detector_batches_against_running_means(gpu, O, name):
    """tsdrgpu_frd_run_batch over contiguous captures of the detector's own size at the product's sample rates (1 409 090 at
    cfg2; 2 818 181 and 450 909 at cfg5 / cfg1 are odd: every other capture starts on an odd sample), batches of 6 and 4, in-stream
    and overlapped: after every batch both plots within 1e-5 of the plot peak of the oracle's frameratedetector run over the same
    captures, call counts equal, and tsdrgpu_frd_peaks equal to the oracle plot's argmax wherever its maximum beats the
    runner-up by more than that tolerance."""
    from tempestsdr_b200.api import FrameRateDetector
    fs, _, fv = CFGS[name]
    rw, rh = FRD[name]
    size = FrameRateDetector.capture_size(fs)
    assert size == int(3.1 * fs / 55.0)
    batches = (6, 4)
    x = np.abs(synth.video_like_iq(size * sum(batches), fs, rw, rh, fv, seed=31, snr_db=25.0).view(np.complex64)).astype(np.float32)
    det = O.framerate_detector()
    want = []
    k = 0
    for nb in batches:
        for _ in range(nb):
            r = det.run(fs, x[k * size:(k + 1) * size]); k += 1
        want.append(r)
    d = dev(x)
    for overlap in (False, True):
        g = gpu.framerate_detector()
        g.set_overlap(overlap)
        k = 0
        for nb, ((fo, fp), (lo, lp), calls) in zip(batches, want):
            got_calls = g.run_batch(fs, d[k * size:], size, nb, size)
            k += nb
            g.join()
            (gfo, gfp), (glo, glp) = g.plots(fs)
            what = f"{name} overlap={overlap} after {k} captures"
            assert (gfo, glo, got_calls) == (fo, lo, calls), what
            _close(gfp, fp, 1e-5, f"frame plot {what}"); _close(glp, lp, 1e-5, f"line plot {what}")   # 1e-5 of the plot peak
            peaks = (C.c_int32 * 2)()
            gpu.chk(_lib().tsdrgpu_frd_peaks(g._h, gpu.stream, peaks))
            for p, plot in zip(peaks, (fp, lp)):
                top2 = np.sort(plot)[-2:]
                if top2[1] - top2[0] > 1e-5 * np.max(np.abs(plot)):
                    assert p == int(np.argmax(plot)), what


# ------------------------------------------------------------------------------------------------ 7. the benchmark step itself
@pytest.mark.parametrize("shape", ["cfg2", "cfg5"])
def test_bench_device_step_against_a_stagewise_replay(shape):
    """bench.py's DeviceStep (two steps of 64 frames' worth of IQ, the same resident IQ each step) against the oracle replaying
    the same stream stage by stage: every frame handed over bit-exact, both plots within 1e-5 of their peak after each step.
    Covers the glue the kernel tests miss: pixels carried between steps, the fused magnitude output, the detector's double-
    buffered stream and the overlap of one batch's sync search with the next batch.  A process per shape (bench.py reads
    BENCH_SHAPE when it is imported); tests/bench_step_replay.py holds the comparison."""
    r = subprocess.run([sys.executable, "-m", "tests.bench_step_replay"], capture_output=True, text=True, timeout=900, cwd=ROOT,
                       env=dict(os.environ, BENCH_SHAPE=shape))
    assert r.returncode == 0 and "replay ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])
    print(r.stdout.strip().splitlines()[-1])
