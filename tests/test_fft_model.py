"""The float64 FFT models of tests/fft_model.py, checked without a GPU: against the host library's stage-angle helper, against
numpy.fft with exact angles, and against the compiled reference within the float32 rounding bound of
tests/test_fft_float64_model.py (max|e| <= u log2 N r, rms(e) <= u sqrt(log2 N) r, r = rms of the model, u = 2^-24).  The
bound has teeth: outputs carrying a plausible transform bug are rejected at the sizes listed in COVERED."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import _native, synth
from tests import fft_model as fm

SIZES = range(23)             # 2^0 .. 2^22; 2^23 and 2^24 are checked on the GPU box, where the models are computed anyway
_CACHE = {}


@pytest.fixture(scope="module")
def O():
    return orc.best()


def case(O, m, inv):
    """noise(m), the compiled reference's transform of it and the reference model, computed once per module."""
    key = (m, inv)
    if key not in _CACHE:
        x = synth.noise_iq(1 << m, seed=m)
        xc = fm.as_complex(x)
        _CACHE[key] = (xc, fm.as_complex(O.fft(x, inv)), fm.reference_fft(xc, inv))
    return _CACHE[key]


def test_eps_matches_the_host_library_bit_for_bit():
    lib = _native.lib()
    for inv in (0, 1):
        for stages in range(1, 41):
            buf = (C.c_double * stages)()
            lib.tsdrgpu_fft_reference_eps(stages, inv, buf)
            want = np.frombuffer(buf, np.float64)
            assert np.array_equal(fm.eps(stages, bool(inv)).view(np.uint64), want.view(np.uint64)), (stages, inv)


@pytest.mark.parametrize("m", SIZES)
def test_models_with_exact_angles_equal_numpy(m):
    """eps = 0 turns every model into the exact DFT: the reference's radix-2, each plan shape and the half-size real transform."""
    n = 1 << m
    z = np.zeros(max(m, 1))
    xc = fm.as_complex(synth.noise_iq(n, seed=m))
    shapes = {tuple(fm.default_plan(m, **kw)) for kw in fm.PLAN_SHAPES.values()}
    for inv in (False, True):
        want = np.fft.ifft(xc) * n if inv else np.fft.fft(xc) / n
        tol = 1e-12 * fm.rms(want)
        assert np.max(np.abs(fm.reference_fft(xc, inv, z) - want)) <= tol
        for p in shapes:
            assert np.max(np.abs(fm.plan_fft(xc, inv, list(p), z) - want)) <= tol, p
        if m >= 1:
            re = xc.real
            want = np.fft.ifft(re) * n if inv else np.fft.fft(re)
            assert np.max(np.abs(fm.half_real_fft(re, inv, stage_eps=z) - want)) <= 1e-12 * fm.rms(want)


@pytest.mark.parametrize("m", SIZES)
def test_compiled_reference_meets_the_rounding_bound(O, m):
    """The reference's float32 transform against its float64 model: within the bound with C = 1 at every size (measured worst
    case 0.62 max / 0.49 rms at 2^1, <= 0.43 / 0.44 from 2^2 to 2^22)."""
    for inv in (False, True):
        _, y, ref = case(O, m, inv)
        u = fm.rounding_units(y, ref, 1 << m)
        assert u[0] <= 0.75 and u[1] <= 0.6, (m, inv, u)
        assert fm.bin_units(y, ref, 1 << m)[0] <= 0.75, (m, inv)


@pytest.mark.parametrize("size", [5, 17, 4096, 70_001, 450_909, 1_409_090, (1 << 22) + 3])
def test_compiled_reference_correlations_meet_twice_the_bound(O, size):
    """Autocorrelation and cross-correlation of the compiled reference against the composed reference model, per lag within twice
    fft_model.bin_scale and in rms within twice the transform constant (tests/test_fft_float64_model.py derives the factor)."""
    n = fm.getrealsize(size)
    x = np.abs(fm.as_complex(synth.noise_iq(size, seed=size))).astype(np.float32)
    got = fm.as_complex(O.autocorrelation(x)[: 2 * n])
    u = fm.bin_units(got, fm.autocorrelation(x, "reference"), n)
    assert u[0] <= 2.0 and u[1] <= 2.0, ("autocorrelation", size, u)
    a, b = synth.noise_iq(size, seed=1), synth.noise_iq(size, seed=2)
    got = fm.as_complex(O.crosscorrelation(a, b)[: 2 * n])
    u = fm.bin_units(got, fm.crosscorrelation(fm.as_complex(a), fm.as_complex(b)), n)
    assert u[0] <= 2.0 and u[1] <= 2.0, ("crosscorrelation", size, u)


@pytest.mark.parametrize("m", range(12, 23))
def test_plan_deviation_from_the_reference_model_is_pinned(O, m):
    """Each plan shape lies within its pinned deviation of the reference model (the measured value with 2x headroom), and not
    far below it: a model change that moved it would show here."""
    for shape, kw in fm.PLAN_SHAPES.items():
        pin = fm.plan_deviation(m, shape)
        dev = 0.0
        for inv in (False, True):
            xc, _, ref = case(O, m, inv)
            plan = fm.plan_fft(xc, inv, fm.default_plan(m, **kw))
            dev = max(dev, float(np.max(np.abs(plan - ref))) / (fm.U * m * fm.rms(ref)))
        assert pin / 4 <= dev <= pin, (shape, m, dev, pin)


def _mutants(m, inv):
    e = fm.eps(m, inv)
    swapped = e.copy()
    if m >= 2:
        swapped[[m - 1, m - 2]] = e[[m - 2, m - 1]]
    top_zero = e.copy()
    top_zero[m - 1 if m else 0:] = 0.0
    return {"eps_dropped": np.zeros(max(m, 1)), "top_two_swapped": swapped, "top_eps_zero": top_zero}


# (mutant, log2 N) pairs where the mutant's largest deviation from the model exceeds twice the bound, in both directions: the
# bound must reject each of them.  eps grows with the stage, so the eps mutants stand out from 2^20 on; a wrong-signed inter-pass
# twiddle is caught at every size with more than one pass.  (At 2^22 the top two stages' errors are nearly equal, so
# swapping them changes little.)
COVERED = ({("eps_dropped", m) for m in (20, 21, 22)} | {("top_two_swapped", m) for m in (20, 21)}
           | {("top_eps_zero", m) for m in (20, 21, 22)} | {("twiddle_sign", m) for m in range(12, 23)})


def test_the_bound_rejects_plausible_bugs(O):
    """The compiled reference's output plus (mutant model - model) for: the stage-angle errors dropped (the true DFT), the top two
    stages' errors swapped, the top stage's error set to zero, and every inter-pass twiddle with the wrong sign (against the plan
    model, with the pinned plan deviation added to the bound)."""
    caught = {False: set(), True: set()}
    for m in SIZES:
        n = 1 << m
        L = max(m, 1)
        for inv in (False, True):
            xc, y, ref = case(O, m, inv)
            r = fm.rms(ref)
            muts = {k: (fm.reference_fft(xc, inv, e), ref, 0.0) for k, e in _mutants(m, inv).items()}
            if m >= 12:
                plan = fm.plan_fft(xc, inv)
                muts["twiddle_sign"] = (fm.plan_fft(xc, inv, twiddle_sign=-1.0), plan, fm.plan_deviation(m))
            for name, (mut, model, extra) in muts.items():
                big = float(np.max(np.abs(mut - model))) / (fm.U * L * r) > 2 * (1.0 + extra)
                if not big:
                    continue
                u = fm.rounding_units(y + (mut - model), model, n)
                assert u[0] > 1.0 + extra or u[1] > 1.0 + extra * np.sqrt(L), (name, m, inv, u)
                caught[inv].add((name, m))
    covered = caught[False] & caught[True]
    assert covered == COVERED, (sorted(covered - COVERED), sorted(COVERED - covered))
    for need in [("eps_dropped", 20), ("eps_dropped", 21), ("top_two_swapped", 20), ("top_two_swapped", 21)]:
        assert need in covered


@pytest.mark.parametrize("m", [14, 21])
def test_float32_twiddle_tables_explain_the_tone_deviation(m):
    """The library's twiddles are float32 (rounded on the host from double) and shared by every block of a stage.  Rounding them
    alone, with exact arithmetic otherwise, moves a bin-centred tone's transform by more than the per-bin rounding scale (the errors
    of all blocks add coherently on the tone's bins) and a noise transform by far less: the GPU tests therefore compare with the
    model that carries float32 twiddles."""
    from tests.test_fft_float64_model import inputs
    n = 1 << m
    for name, x in inputs(m):
        xc = fm.as_complex(x)
        dev = fm.bin_units(fm.plan_fft(xc, f32=True), fm.plan_fft(xc), n)[0]
        if name == "noise":
            assert dev <= 0.35, dev
        elif name == f"tone@{n // 2}":
            assert dev == 0.0                           # W^0 and W^(N/2) are exact in float32
        elif name.startswith("tone"):
            assert dev >= (1.2 if m == 14 else 10.0), (name, dev)
