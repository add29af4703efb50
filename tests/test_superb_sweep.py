"""The superbandwidth alignment and stitch against float64 models of the reference (tests/superb_model.py), at every lag class,
hop shape and rank layout the code reaches.

Units are those of the FFT tests (fft_model.rounding_units): for an output Y of n points, its model M and u = 2^-24, the largest
|Y - M| in units of u log2(n) rms(M) and the rms in units of u sqrt(log2 n) rms(M).  Every GPU result is compared with the model
of its own dataflow within C_OWN_MAX / C_OWN_RMS (superb_model; the measured worst case on an H100 plus headroom), and with the
reference's model within that plus the pinned deviation of the two models (ONE_GPU_DEVIATION, SHARDED_DEVIATION), which the CPU
tests below measure on the same inputs.  Lags are integers and must equal the compiled reference's; every generated case's
correlation peak stands above the second-largest value by far more than the rounding of an nd-point correlation
(superb_model.lag_bound), and the model asserts that it does.

The CPU tests (no GPU) check the models against the compiled reference; the GPU tests (-m gpu) check the library.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tests import fft_model as fm
from tests import sbm_one_device as sbm
from tests import superb_model as sm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu_only = pytest.mark.gpu
MARGIN_FACTOR = 100.0          # generated cases clear the lag bound by at least this factor


# ------------------------------------------------------------------------------------------------ cases
ABS_SIZES = [2, 4, 6, 4094, 4096, 4098, (1 << 21) - 2, (1 << 21) + 2]
ABS_KINDS = ["noise", "zero", "neg_zero", "subnormal", "square_overflow", "inf", "nan_first", "nan_inside", "huge_first"]


def abs_input(size, kind):
    x = np.random.default_rng(size).standard_normal(size).astype(np.float32)
    if kind == "zero":
        x[:] = 0.0
    elif kind == "neg_zero":
        x[:] = -0.0
    elif kind == "subnormal":
        x *= np.float32(1e-40)                          # I, Q subnormal: I^2 underflows to 0
    elif kind == "square_overflow":
        x[0::3] = np.float32(3e20)                      # I^2 = inf, I finite
    elif kind == "inf":
        x[size // 2 - (size // 2) % 2] = np.inf
        x[-1] = -np.inf
    elif kind == "nan_first":
        x[0] = np.nan
    elif kind == "nan_inside":
        x[(size // 2) | 1] = np.nan
    elif kind == "huge_first":
        x[0], x[1] = np.float32(3e18), np.float32(-1e18)    # the seed I^2 + Q^2 = 1e37 dominates the first difference
    return x


def peak_classes(nd):
    return [0, 1, nd // 2 - 1, nd // 2, nd // 2 + 1, nd - 2, nd - 1]


def chunk_peaks(nd, chunk):
    """First and last element of chunk `chunk` of k_argmax_partial (parts = min(ceil(nd / 4096), 1024), ceil(nd / parts) each)."""
    parts = min(max((nd + 4095) // 4096, 1), 1024)
    per = (nd + parts - 1) // parts
    return [chunk * per, chunk * per + per - 1]


def bestfit_cases():
    """(id, pairs, size_floats, sif, lag, kind): the hops are built by bestfit_hops; lag None = not a generated peak."""
    out = []
    # nd = N/2: sif = 8000 at N = 2^16 (2N / 8000 = 16.384)
    for lag in peak_classes(1 << 15):
        out.append((f"halfN_2^16_lag{lag}", 80_000, 1 << 17, 8000, lag, "shift"))
    # nd = N: sif = 2^14 divides 2N
    for lag in peak_classes(1 << 16):
        out.append((f"fullN_2^16_lag{lag}", (1 << 16) + 3, 1 << 17, 1 << 14, lag, "shift"))
    # configs[3]'s sizing: sif = 416 666 at N = 2^21, nd = 2^20
    for lag in (1, (1 << 20) - 1):
        out.append((f"halfN_2^21_sif416666_lag{lag}", 4_166_660, 1 << 22, 416_666, lag, "shift"))
    # k_argmax_partial's cut points: 4096 per chunk up to nd = 2^22, 8192 above the 1024-part cap
    for lag in chunk_peaks(1 << 16, 5):
        out.append((f"chunk_2^16_lag{lag}", 1 << 16, 1 << 17, 1 << 14, lag, "shift"))
    for lag in chunk_peaks(1 << 22, 1000):
        out.append((f"chunk_2^22_lag{lag}", 1 << 22, 1 << 23, 1 << 14, lag, "shift"))
    out.append((f"chunk_2^23_lag{chunk_peaks(1 << 23, 2)[1]}", 1 << 23, 1 << 24, 1 << 14, chunk_peaks(1 << 23, 2)[1], "shift"))
    # small correlations
    out.append(("nd64_lag3", 64, 128, 16, 3, "shift"))
    out.append(("nd1", 64, 2, 2, None, "shift0"))
    # special hops: the lag must equal the reference's
    for kind in ("nan_hop", "inf_hop0", "identical", "zero"):
        out.append((kind, 1 << 12, 1 << 13, 1000, None, kind))
    return out


def bestfit_hops(pairs, size_floats, sif, lag, kind, seed=3):
    nd = sm.correlation_pairs(size_floats, sif)
    if kind == "shift":
        return sm.shifted_hops(pairs, [0, sm.shift_for_lag(lag, nd)], seed=seed)
    a, b = sm.shifted_hops(pairs, [0, 0], seed=seed)
    if kind == "nan_hop":
        b[2 * 100 + 1] = np.nan
    elif kind == "inf_hop0":
        a[2 * 7] = np.inf
    elif kind == "identical":
        b = a.copy()
    elif kind == "zero":
        a[:] = 0.0
        b[:] = 0.0
    return [a, b]


BESTFIT = bestfit_cases()
BIG = 1 << 21                    # correlations above this many pairs: one model each, seconds on a CPU


def stitch_cases():
    """(id, H, pairs, sif, lags): one-GPU stitches, H in {1, 2, 3, 4, 5, 8, 16}, N from 64 to 2^18 and configs[3]'s 4 x 2^21;
    count_pairs a power of two, one more, and one less than the next; nd = N/2 and nd = N; lag classes mixed across the hops."""
    def mix(nd, H, j):
        cls = peak_classes(nd) + [3, nd - 5]
        return [0] + [cls[(j + 3 * q) % len(cls)] for q in range(H - 1)]
    return [
        ("H1_N64", 1, 64, 50, [0]),
        ("H2_N2^10_halfN", 2, 1 << 10, 700, mix(1 << 9, 2, 0)),
        ("H3_N2^12_plus1", 3, (1 << 12) + 1, 3000, mix(1 << 11, 3, 1)),
        ("H4_N2^13_fullN", 4, (1 << 14) - 1, 1 << 12, mix(1 << 13, 4, 2)),
        ("H5_N2^16_halfN", 5, 1 << 16, 8000, mix(1 << 15, 5, 3)),
        ("H8_N2^17_fullN", 8, 1 << 17, 1 << 15, mix(1 << 17, 8, 4)),
        ("H16_N2^18_halfN", 16, (1 << 19) - 1, 8000, mix(1 << 17, 16, 5)),
        ("H4_N2^21_configs3", 4, 4_166_660, 416_666, [0, 1234, (1 << 20) - 77, (1 << 19) + 1]),
    ]


STITCH = stitch_cases()


def stitch_hops(H, pairs, sif, lags, seed):
    n = fm.getrealsize(pairs)
    nd = sm.correlation_pairs(2 * n, sif)
    return sm.shifted_hops(pairs, [sm.shift_for_lag(l, nd) for l in lags], seed=seed), n, nd


# ------------------------------------------------------------------------------------------------ CPU: the models
@pytest.fixture(scope="module")
def O():
    return orc.best()


@pytest.fixture(scope="module")
def R():
    if not orc.have_ref():
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    return orc.ref()


@pytest.mark.parametrize("size", ABS_SIZES)
def test_abs_diff_model_is_the_reference_bit_for_bit(R, size):
    for kind in ABS_KINDS:
        x = abs_input(size, kind)
        got, want = sm.abs_diff(x), R.complex_to_abs_diff(x)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (size, kind)


@pytest.mark.parametrize("cid,pairs,size_floats,sif,lag,kind", [c for c in BESTFIT if c[1] <= BIG], ids=[c[0] for c in BESTFIT if c[1] <= BIG])
def test_bestfit_model_is_the_reference(R, cid, pairs, size_floats, sif, lag, kind):
    a, b = bestfit_hops(pairs, size_floats, sif, lag, kind)
    off, margin, nd = sm.bestfit(a, b, size_floats, sif)
    want = R.superb_bestfit(a[:size_floats], b[:size_floats], sif)
    assert off == want, (off, want)
    if lag is not None:
        assert off == 2 * lag and margin >= MARGIN_FACTOR * sm.lag_bound(nd), (off, lag, margin)
    print(f"{cid}: nd = {nd}, offset {off}, margin {margin:.3g} (lag bound {sm.lag_bound(nd):.3g})")


def test_bestfit_refuses_less_than_two_floats():
    assert sm.correlation_pairs(100, 200) is None and sm.correlation_pairs(1, 1) is None and sm.correlation_pairs(2, 2) == 1


@pytest.mark.parametrize("cid,H,pairs,sif,lags", STITCH, ids=[c[0] for c in STITCH])
def test_stitch_models_against_the_reference(R, cid, H, pairs, sif, lags):
    """stitch_reference is within float32 rounding of the compiled reference (REFERENCE_UNITS), and the one-GPU model within the
    pinned deviation of stitch_reference (ONE_GPU_DEVIATION)."""
    hops, n, nd = stitch_hops(H, pairs, sif, lags, seed=H)
    want, offs = R.superb_ondataready(hops, sif)
    ref, moffs = sm.stitch_reference(hops, sif)
    assert list(offs) == moffs == [2 * l for l in lags], (list(offs), moffs, lags)
    tp = fm.getrealsize(H * n)
    w = fm.as_complex(want)
    u = sm.units(w[:tp], ref[:tp], tp)
    one, _ = sm.stitch_one_gpu(hops, sif, moffs)
    d = sm.units(one[:tp], ref[:tp], tp)
    line = f"{cid}: reference vs model max {u[0]:.3f} rms {u[1]:.3f}; one-GPU model vs reference model max {d[0]:.3f} rms {d[1]:.3f}"
    assert u[0] <= sm.REFERENCE_UNITS[0] and u[1] <= sm.REFERENCE_UNITS[1], line
    pin = sm.one_gpu_deviation(H, n)
    assert d[0] <= pin[0] and d[1] <= pin[1], (line, pin)
    if tp < H * n:                    # the tail stays as spectra, in the reference as in the models
        ut, dt = sm.units(w[tp:], ref[tp:], n), sm.units(one[tp:], ref[tp:], n)
        line += f"; tail: reference {ut[0]:.3f} / {ut[1]:.3f}, one-GPU model {dt[0]:.3f} / {dt[1]:.3f}"
        assert ut[0] <= sm.REFERENCE_UNITS[0] and ut[1] <= sm.REFERENCE_UNITS[1], line
        assert dt[0] <= pin[2] and dt[1] <= pin[3], (line, pin)
    print(line)


def _sharded_params():
    out = []
    for H in (2, 4, 8):
        for root, cs in sbm.sweep_cases(H) + (sbm.FULL_CASES if H == 4 else []):
            for i, c in enumerate(cs):
                out.append(pytest.param(H, c, id=f"H{H}_root{root}_{i}_N2^{fm.log2_of(fm.getrealsize(c['pairs']))}"))
    return out


@pytest.mark.parametrize("H,c", _sharded_params())
def test_sharded_model_against_the_reference_model(H, c):
    """The sharded dataflow's model equals |stitch_reference| within SHARDED_DEVIATION on the sweep's inputs."""
    pairs, sif = c["pairs"], c["sif"]
    n = fm.getrealsize(pairs)
    nd = sm.correlation_pairs(2 * n, sif)
    hops = sm.shifted_hops(pairs, [sm.shift_for_lag(l, nd) for l in c["lags"]], seed=c["seed"])
    offs = [2 * l for l in c["lags"]]
    ref, _ = sm.stitch_reference(hops, sif, offsets=offs)
    d = sm.units(sm.stitch_sharded(hops, c["lags"]), np.abs(ref), H * n)
    pin = sm.sharded_deviation(H, n)
    print(f"H={H} N=2^{fm.log2_of(n)}: sharded model vs reference model max {d[0]:.3f} rms {d[1]:.3f} (pinned {pin})")
    assert d[0] <= pin[0] and d[1] <= pin[1], (d, pin)


def test_sharded_model_with_exact_angles_is_the_true_dft():
    """With exact stage angles both models are the DFT: they agree to float64 rounding, not to the pinned deviation."""
    hops = sm.shifted_hops(1 << 12, [0, -5, 7, 100], seed=4)
    lags = [0, 5, (1 << 11) - 7, (1 << 11) - 100]
    ref, _ = sm.stitch_reference(hops, 3000, offsets=[2 * l for l in lags], true_dft=True)
    d = sm.units(sm.stitch_sharded(hops, lags, true_dft=True), np.abs(ref), 4 << 12)
    assert d[0] < 0.7 and d[1] < 0.7, d                  # the float32 twiddle tables of the plan model only


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


WORST = {}


def _record(what, u):
    old = WORST.get(what, (0.0, 0.0))
    WORST[what] = (max(old[0], u[0]), max(old[1], u[1]))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for what, (mx, rm) in sorted(WORST.items()):
        print(f"worst {what:<40} max {mx:.3f}  rms {rm:.3f}")


def same_bits_nan_as_nan(got, want):
    """Bit for bit, except that any NaN matches any NaN: x86 makes inf - inf the NaN 0xffc00000 and passes an input NaN's payload
    on, the GPU writes 0x7fffffff for both."""
    gn, wn = np.isnan(got), np.isnan(want)
    return np.array_equal(gn, wn) and np.array_equal(got[~gn].view(np.uint32), want[~wn].view(np.uint32))


@gpu_only
@pytest.mark.parametrize("size", ABS_SIZES)
def test_abs_diff_bit_for_bit(gpu, O, size):
    bad = []
    for kind in ABS_KINDS:
        x = abs_input(size, kind)
        d = dev(x)
        gpu.complex_to_abs_diff(d)
        want = O.complex_to_abs_diff(x)
        if not same_bits_nan_as_nan(d.cpu().numpy(), want):
            bad.append(kind)
    assert not bad, (size, bad)


@gpu_only
@pytest.mark.parametrize("cid,pairs,size_floats,sif,lag,kind", BESTFIT, ids=[c[0] for c in BESTFIT])
def test_bestfit_lag(gpu, O, cid, pairs, size_floats, sif, lag, kind):
    a, b = bestfit_hops(pairs, size_floats, sif, lag, kind)
    got = gpu.superb_bestfit(dev(a), dev(b), size_floats, sif)
    want = O.superb_bestfit(a[:size_floats], b[:size_floats], sif)
    off, margin, nd = sm.bestfit(a, b, size_floats, sif)
    assert got == want == off, (got, want, off)
    if lag is not None:
        assert off == 2 * lag and margin >= MARGIN_FACTOR * sm.lag_bound(nd), (off, lag, margin)
    if kind in ("nan_hop", "identical", "zero"):
        assert got == 0


@gpu_only
def test_bestfit_refuses_less_than_two_floats(gpu):
    from tempestsdr_b200 import _native as N
    a = dev(np.ones(200, np.float32))
    for size_floats, sif in ((100, 200), (1, 1), (199, 200)):
        with pytest.raises(N.TsdrGpuError):
            gpu.superb_bestfit(a, a, size_floats, sif)
    assert gpu.superb_bestfit(a, a, 2, 2) == 0


@gpu_only
@pytest.mark.parametrize("cid,H,pairs,sif,lags", STITCH, ids=[c[0] for c in STITCH])
def test_one_gpu_stitch(gpu, O, cid, H, pairs, sif, lags):
    hops, n, nd = stitch_hops(H, pairs, sif, lags, seed=H)
    want, offs = O.superb_ondataready(hops, sif)
    got, goffs = gpu.superb_stitch([dev(h) for h in hops], sif)
    assert list(goffs) == list(offs) == [2 * l for l in lags], (goffs, list(offs), lags)
    g = fm.as_complex(got.cpu().numpy())
    own, _ = sm.stitch_one_gpu(hops, sif, list(goffs))
    ref, _ = sm.stitch_reference(hops, sif, list(goffs))
    tp = fm.getrealsize(H * n)
    pin = sm.one_gpu_deviation(H, n)
    parts = [("head", slice(0, tp), tp, pin[:2])] + ([("tail", slice(tp, H * n), n, pin[2:])] if tp < H * n else [])
    for what, sl, pts, dv in parts:
        uo, ur = sm.units(g[sl], own[sl], pts), sm.units(g[sl], ref[sl], pts)
        _record(f"one-GPU {what} vs own model", uo)
        _record(f"one-GPU {what} vs reference model - pin", (ur[0] - dv[0], ur[1] - dv[1]))
        print(f"{cid} {what}: vs own model max {uo[0]:.3f} rms {uo[1]:.3f}; vs reference model max {ur[0]:.3f} rms {ur[1]:.3f} (pin {dv[0]:.3f} / {dv[1]:.3f})")
        assert uo[0] <= sm.C_OWN_MAX and uo[1] <= sm.C_OWN_RMS, (what, uo)
        assert ur[0] <= sm.C_OWN_MAX + dv[0] and ur[1] <= sm.C_OWN_RMS + dv[1], (what, ur, dv)


@gpu_only
def test_one_gpu_stitch_refuses_bad_hop_counts(gpu):
    from tempestsdr_b200 import _native as N
    h = dev(np.ones(2 * 256, np.float32))
    with pytest.raises(N.TsdrGpuError):
        gpu.superb_stitch([h] * 17, 100)


def _run_sbm(args, timeout, **env):
    r = subprocess.run([sys.executable, "-m", "tests.sbm_one_device"] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT,
                       env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32", TSDRGPU_SBM_TIMEOUT_MS="3000", **env))
    print(r.stdout[-6000:])
    assert r.returncode == 0 and "sbm ok" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


@gpu_only
@pytest.mark.parametrize("H", [2, 4, 8])
def test_sharded_stitch_on_one_device(H):
    """tsdrgpu_superb_mgpu_* with all H ranks on this GPU: every root, both hop-0 modes, copy-out and in-place, three stitches in a
    row per group (N = 2^16, 2^12, 2^16), nd = N/2 and nd = N, every lag class, and refusals by one rank (tests/sbm_one_device.py)."""
    _run_sbm([str(H)], 400)


@gpu_only
def test_sharded_stitch_at_the_baseline_hop_size():
    """BASELINE configs[3]'s own size: 4 hops of 10 frames of 25 MS/s IQ (N = 2^21 per hop, a 2^23-point inverse), where the
    reference's last stages are furthest from the true DFT."""
    _run_sbm(["4", "full"], 400)


@gpu_only
def test_sharded_stitch_with_exact_stage_angles():
    """TSDRGPU_FFT_TRUE_DFT=1 at 4 x 2^21: within the bound of the exact-angle models, and outside the bound of the reference's
    model -- the reference's angle errors at 2^23 points are what the bound must be able to see."""
    _run_sbm(["4", "full"], 400, TSDRGPU_FFT_TRUE_DFT="1")


@gpu_only
def test_sharded_group_sizes(gpu):
    """Groups of 2, 4 and 8 ranks; anything else (16 included: a node has at most eight GPUs) is refused."""
    lib = gpu._lib
    for H in (1, 3, 16, 32):
        h = C.c_void_p()
        assert lib.tsdrgpu_superb_mgpu_create(gpu._h, H, 0, 0, 4096, C.byref(h)) != 0 and not h.value, H
    for H in (2, 4, 8):
        h = C.c_void_p()
        assert lib.tsdrgpu_superb_mgpu_create(gpu._h, H, H - 1, 0, 4096, C.byref(h)) == 0 and h.value, H
        lib.tsdrgpu_superb_mgpu_destroy(h)
