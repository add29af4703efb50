"""GPU: the half-size autocorrelation with its finishing steps folded into neighbouring kernels.

The forward transform's finish (R = |X|/N from the half-size spectrum) is formed by the inverse transform's first pass as it
loads, and the frame-rate detector takes its running means straight from the inverse's half-size output (k_accumulate_half).
With TSDRGPU_AUTOCORR_GROUP below the batch, each group's running means are updated before the next group reuses the work
buffers, so the grouping must not change a single bit of the plots.  A 2^23-point autocorrelation reaches the three-pass plan
of the half-size transforms, which no other test runs through the folded load.
"""
import ctypes as C

import numpy as np
import pytest

from tempestsdr_b200 import synth
from tests.test_gpu_parity import CFGS, _close, assert_same_bits, dev

pytestmark = pytest.mark.gpu

# bench.py's raster per shape; at cfg1 (N = 2^18) the frame window reaches beyond N/2, the lags the split's second half gives
FRD = {"cfg2": (2576, 1125), "cfg1": (800, 525)}


@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


def _detector_run(gpu, fs, d, size, batches, overlap):
    """plots and peaks after every batch of one detector fed `batches` batches of consecutive captures"""
    from tempestsdr_b200 import _native
    g = gpu.framerate_detector()
    g.set_overlap(overlap)
    out, k = [], 0
    for nb in batches:
        calls = g.run_batch(fs, d[k * size:], size, nb, size)
        k += nb
        g.join()
        (_, fp), (_, lp) = g.plots(fs)
        peaks = (C.c_int32 * 2)()
        gpu.chk(_native.lib().tsdrgpu_frd_peaks(g._h, gpu.stream, peaks))
        out.append((calls, fp, lp, tuple(peaks)))
    return out


@pytest.mark.parametrize("name", list(FRD))
@pytest.mark.parametrize("overlap", [False, True])
def test_detector_grouping_is_bit_identical(gpu, name, overlap, monkeypatch):
    """tsdrgpu_frd_run_batch with TSDRGPU_AUTOCORR_GROUP = 1 and 2 (a partial last group in both batches of 5 and 3) against the
    default grouping (the whole batch): call counts, both plots after every batch bit for bit, and the device-picked peaks."""
    from tempestsdr_b200.api import FrameRateDetector
    fs, _, fv = CFGS[name]
    rw, rh = FRD[name]
    size = FrameRateDetector.capture_size(fs)
    batches = (5, 3)
    x = np.abs(synth.video_like_iq(size * sum(batches), fs, rw, rh, fv, seed=47, snr_db=25.0).view(np.complex64)).astype(np.float32)
    d = dev(x)
    monkeypatch.delenv("TSDRGPU_AUTOCORR_GROUP", raising=False)
    want = _detector_run(gpu, fs, d, size, batches, overlap)
    assert [w[0] for w in want] == [5, 8]
    for grp in ("1", "2"):
        monkeypatch.setenv("TSDRGPU_AUTOCORR_GROUP", grp)
        got = _detector_run(gpu, fs, d, size, batches, overlap)
        for b, ((gc, gfp, glp, gpk), (wc, wfp, wlp, wpk)) in enumerate(zip(got, want)):
            what = f"{name} overlap={overlap} group={grp} batch {b}"
            assert gc == wc, what
            assert_same_bits(gfp, wfp, f"frame plot {what}")
            assert_same_bits(glp, wlp, f"line plot {what}")
            assert gpk == wpk, what


def test_three_pass_half_size_autocorrelation(gpu, monkeypatch):
    """2^23 + 2 samples (N = 2^23: the half-size transforms have 2^22 points, a three-pass plan) against the N-point path
    (TSDRGPU_AUTOCORR_FULL=1): within 2e-6 of the zero-lag peak, the untransformed tail bit-exact."""
    size = (1 << 23) + 2
    x = np.abs(synth.noise_iq(size, seed=23)[:size]).astype(np.float32)
    n = gpu.fft_getrealsize(size)
    assert n == 1 << 23
    d = dev(x)
    monkeypatch.delenv("TSDRGPU_AUTOCORR_FULL", raising=False)
    half = gpu.fft_autocorrelation(d).cpu().numpy()
    monkeypatch.setenv("TSDRGPU_AUTOCORR_FULL", "1")
    full = gpu.fft_autocorrelation(d).cpu().numpy()
    assert np.all(np.isfinite(half))
    _close(half[: 2 * n], full[: 2 * n], 2e-6, "half-size vs N-point autocorrelation at 2^23")
    assert_same_bits(half[2 * n:], full[2 * n:], "autocorrelation tail at 2^23")
