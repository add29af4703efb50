"""The FFT family on the GPU bin by bin against float64 models (tests/fft_model.py), with bounds set by float32 rounding.

The bound.  For an output Y, its model M, e = Y - M, r = rms(M) over the transformed points and u = 2^-24:
    |e_k| <= C_MAX bin_scale_k (= u log2 N r for a flat spectrum)        rms(e) <= C_RMS u sqrt(log2 N) r
A radix-2 transform rounds every output once per stage, and each rounding moves it by at most u times its magnitude, so the error
grows like u sqrt(log2 N) in rms and like u log2 N at worst.  The compiled reference meets this with C = 1 against its own model:
0.62 (max) and 0.49 (rms) at two points, <= 0.43 and 0.43 from 2^3 to 2^22 (tests/test_fft_model.py).  The GPU's transform is
compared with the model of its own factorisation (plan_fft), and with the reference's (reference_fft) within C plus the pinned
deviation of the plan (fft_model.PLAN_DEVIATION: up to 5.6 at 2^24, where the exact inter-pass twiddles leave out the stage-angle
errors of the reference's upper stages).

Per bin.  The max criterion is applied bin by bin with fft_model.bin_scale, which is u log2 N r for a flat spectrum (noise,
impulses, the falling spectrum) and larger only on the bins where a concentrated output's rounding lands: the bins of a tone's
residue class modulo large powers of two, a non-negative capture's zero lag and its multiples of large powers of two.  A plain
max|e| <= u log2 N r cannot hold there for any float32 radix-2 transform: the compiled reference reaches 29 u log2 N r on a
2^22-point tone and 5 on a 2^16-point autocorrelation, but stays within 0.42 (transforms) and 0.75 (autocorrelations) of the
per-bin scale.

Twiddle tables.  The library's twiddles are float32 values rounded from double on the host, used by every block of a stage,
so their rounding is systematic: for a flat spectrum it is one more rounding among many, but a tone's bin meets the same rounded
twiddle in all N / 2^(l+1) blocks and the errors add coherently (fft_model with exact twiddles is 12.6 bin scales from its own
float32-table version on a 2^21-point tone, 5.0 on a 2^22-point N-point autocorrelation; tests/test_fft_model.py).  So the GPU is
compared with the plan model carrying float32-rounded twiddles (f32=True), which is what its tables hold; the reference's
twiddles are double, so its own model has exact ones.

Correlations.  r = IFFT(|FFT x| / N) with an unscaled inverse: rms(r) = sqrt(N) rms(|X| / N) = rms(X) / sqrt(N), so the forward
transform's error reaches r at the same size relative to rms(r) as it had relative to rms(X) (|.| moves nothing by more than
the error of its argument), and the inverse adds its own: twice the transform constants, per lag with the scale of r (not
relative to the zero-lag value, which for a non-negative capture is hundreds of times the other lags).  The cross-correlation's product
conj(A) B carries the errors of both forward transforms; they are independent, so with the inverse's they add to sqrt(3) < 2
times one transform's error in rms, the same factor of two.  The frame-rate detector's plots are running means of |r| over the
captures, and ||a| - |b|| <= |a - b|, so each element is within the largest capture's lag bound.

Every measured worst case is printed (max: of the per-bin scale; rms: in units of u sqrt(log2 N) r) per size and path.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tempestsdr_b200 import synth
from tests import fft_model as fm
from tests.spectrum_model import WelchModel, segments_per_report, window64

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C_MAX = 1.0         # measured worst case on an H100 SXM: see DESIGN.md, "FFT numerics"
C_RMS = 1.0
C_CORR = 2.0        # correlations: twice the transform constants (module docstring)
WORST = {}          # (what, path) -> (max units, rms units), printed at the end of the module


def _record(what, path, units):
    key = (what, path)
    old = WORST.get(key, (0.0, 0.0))
    WORST[key] = (max(old[0], units[0]), max(old[1], units[1]))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for (what, path), (mx, rm) in sorted(WORST.items()):
        print(f"worst {what:>28} {path:<22} max {mx:.3f}  rms {rm:.3f}")


@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check(y, model, n, what, path, c_max=C_MAX, c_rms=C_RMS, extra=0.0):
    """The rounding bound per bin (fft_model.bin_scale) and in rms, plus `extra` units of u log2 N r on both: a pinned plan
    deviation."""
    L = max(fm.log2_of(n), 1)
    r = fm.rms(model)
    e = np.abs(np.asarray(y) - np.asarray(model))
    u = (float(np.max(e / (c_max * fm.bin_scale(model, n) + extra * fm.U * L * r))) * c_max if e.any() else 0.0,
         fm.rounding_units(y, model, n)[1])
    _record(what, path, u)
    assert u[0] <= c_max, f"{what} [{path}] N={n}: max_k |e_k| / bin scale = {u[0]:.3f} > {c_max}"
    assert u[1] <= c_rms + extra * np.sqrt(L), f"{what} [{path}] N={n}: rms(e) = {u[1]:.3f} u sqrt(log2N) r > {c_rms}"
    return u


# ------------------------------------------------------------------------------------------------ inputs
def noise(m):
    return synth.noise_iq(1 << m, seed=m)        # the input PLAN_DEVIATION was pinned with


def impulse(m, pos):
    x = np.zeros(2 << m, np.float32)
    x[2 * pos] = 1.0
    return x


def tone(m, k):
    n = 1 << m
    j = np.arange(n, dtype=np.int64)
    return np.exp(2j * np.pi * ((k * j) % n) / n).astype(np.complex64).view(np.float32)


def falling(m):
    """A spectrum falling by 120 dB across the band, random phases, built in float64 and rounded to float32."""
    n = 1 << m
    rng = np.random.default_rng(100 + m)
    mag = 10.0 ** (-6.0 * np.arange(n) / max(n - 1, 1))
    return np.fft.ifft(mag * np.exp(2j * np.pi * rng.random(n))).astype(np.complex64).view(np.float32)


def inputs(m):
    n = 1 << m
    rng = np.random.default_rng(7 + m)
    out = [("noise", noise(m))]
    pos = sorted(p for p in {0, 1, max(n // 2 - 1, 0), n - 1, int(rng.integers(n))} if p < n)
    if m >= 23:                                  # the float64 models take seconds here: noise and one impulse
        return out + [(f"impulse@{pos[-1]}", impulse(m, pos[-1]))]
    out += [(f"impulse@{p}", impulse(m, p)) for p in pos]
    out += [(f"tone@{k}", tone(m, k)) for k in sorted({int(rng.integers(n)), n // 2})]
    return out + [("falling_120dB", falling(m))]


def gpu_fft(gpu, x, inverse):
    d = dev(x)
    gpu.fft_perform(d, x.size // 2, inverse)
    return d.cpu().numpy()


# ------------------------------------------------------------------------------------------------ the transform
@pytest.mark.parametrize("m", range(25))
def test_fft_against_the_plan_model(gpu, m):
    """tsdrgpu_fft at every size from 2^0 to 2^24, both directions, on noise, impulses (every bin of the model has magnitude 1/N
    or 1, so a wrong index or twiddle cannot hide behind a peak), bin-centred tones and a spectrum falling by 120 dB; against the
    model of its own plan, and the noise also against the reference's model with the pinned plan deviation."""
    n = 1 << m
    for name, x in inputs(m):
        xc = fm.as_complex(x)
        for inv in (False, True):
            y = fm.as_complex(gpu_fft(gpu, x, inv))
            path = "inverse" if inv else "forward"
            check(y, fm.plan_fft(xc, inv, f32=True), n, f"fft 2^{m} {name}", f"plan {path}")
            _record("fft 2^0..2^24 all inputs", f"plan {path}", WORST[(f"fft 2^{m} {name}", f"plan {path}")])
            if name == "noise":
                check(y, fm.reference_fft(xc, inv), n, f"fft 2^{m} noise", f"reference {path}", extra=fm.plan_deviation(m))


@pytest.mark.parametrize("m", range(25))
def test_fft_bitwise_relations(gpu, m):
    """Relations that hold by construction: scaling the input by 2^+-30 scales the output by the same power bit for bit (no
    subnormals, every operation is a rounded product or sum), and the inverse is the conjugated forward, inverse(x) =
    N conj(forward(conj x)) (the forward's 1/N is one exact product by a power of two)."""
    n = 1 << m
    x = noise(m)
    for inv in (False, True):
        y = gpu_fft(gpu, x, inv)
        for p in (30, -30):
            s = np.float32(2.0 ** p)
            ys = gpu_fft(gpu, x * s, inv)
            assert np.array_equal((y * s).view(np.uint32), ys.view(np.uint32)), f"2^{m} inv={inv}: scale by 2^{p}"
    xc = x.copy()
    xc[1::2] = -xc[1::2]
    fwd = gpu_fft(gpu, xc, False)
    fwd[1::2] = -fwd[1::2]
    fwd = fwd * np.float32(n)
    assert np.array_equal(fwd.view(np.uint32), gpu_fft(gpu, x, True).view(np.uint32)), f"2^{m}: inverse != N conj fwd(conj x)"


# ------------------------------------------------------------------------------------------------ the study knobs
def knob_case(sizes, path):
    """Run in a process of its own (the FFT knobs are read once per process): tsdrgpu_fft of noise(m) in both directions."""
    from tempestsdr_b200 import api
    gpu = api.Context(0)
    out = {}
    for m in sizes:
        for inv in (0, 1):
            out[f"{m}_{inv}"] = gpu_fft(gpu, noise(m), bool(inv))
    np.savez(path, **out)


def run_knob(tmp_path, env, sizes):
    path = str(tmp_path / "knob.npz")
    r = subprocess.run([sys.executable, "-c", f"from tests.test_fft_float64_model import knob_case; knob_case({list(sizes)!r}, {path!r}); print('case ok')"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, **env))
    assert r.returncode == 0 and "case ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])
    return np.load(path)


def test_plain_loads_give_the_same_bits_as_bulk_copies(gpu, tmp_path):
    """TSDRGPU_FFT_NO_TMA=1: the passes that take their lines by TMA bulk copy take them by plain loads instead; the arithmetic is
    shared, so every size gives the same bits."""
    sizes = range(25)
    got = run_knob(tmp_path, {"TSDRGPU_FFT_NO_TMA": "1"}, sizes)
    for m in sizes:
        for inv in (0, 1):
            want = gpu_fft(gpu, noise(m), bool(inv))
            assert np.array_equal(got[f"{m}_{inv}"].view(np.uint32), want.view(np.uint32)), f"2^{m} inv={inv}"


@pytest.mark.parametrize("knob,shape,sizes", [
    ({"TSDRGPU_FFT_2PASS_MAX": "20"}, "2pass_max_20", [21]),
    ({"TSDRGPU_FFT_SPLIT": "ceil"}, "split_ceil", [13, 15, 17, 19, 21]),
    ({"TSDRGPU_FFT_SMALL_BUNDLE": "512"}, "default", [12, 13, 16, 19, 21, 22, 23]),
], ids=["2pass_max_20", "split_ceil", "small_bundle_512"])
def test_plan_shape_knobs_against_their_own_plan_model(tmp_path, knob, shape, sizes):
    """Plans the default never builds (three passes at 2^21, the longer line first, bundles of 512 points on the contiguous passes)
    exercise the pass kernel's generality; each against the model of its own plan."""
    got = run_knob(tmp_path, knob, sizes)
    for m in sizes:
        xc = fm.as_complex(noise(m))
        for inv in (0, 1):
            want = fm.plan_fft(xc, bool(inv), passes=fm.default_plan(m, **fm.PLAN_SHAPES[shape]), f32=True)
            check(fm.as_complex(got[f"{m}_{inv}"]), want, 1 << m, f"fft 2^{m}", f"{shape} {'inverse' if inv else 'forward'}")


def test_true_dft_knob_against_numpy(tmp_path):
    """TSDRGPU_FFT_TRUE_DFT=1: exact stage angles, so every plan is the mathematically exact DFT: against numpy.fft directly."""
    sizes = list(range(0, 25, 2)) + [21, 23]
    got = run_knob(tmp_path, {"TSDRGPU_FFT_TRUE_DFT": "1"}, sizes)
    for m in sizes:
        n = 1 << m
        xc = fm.as_complex(noise(m))
        check(fm.as_complex(got[f"{m}_0"]), np.fft.fft(xc) / n, n, f"fft 2^{m}", "true DFT forward")
        check(fm.as_complex(got[f"{m}_1"]), np.fft.ifft(xc) * n, n, f"fft 2^{m}", "true DFT inverse")


# ------------------------------------------------------------------------------------------------ correlations
AC_SIZES = [1, 5, 15, 16, 17, 4096, 70_001, 450_909, 450_910, 1_409_090, 2_818_181, (1 << 22) + 3]


def ac_capture(size, kind, seed=0):
    if kind == "noise":
        return np.abs(fm.as_complex(synth.noise_iq(size, seed=size + seed))).astype(np.float32)
    iq = synth.video_like_iq(size, 25_000_000, 2200, 1125, 60.0, seed=seed)
    return np.abs(fm.as_complex(iq)).astype(np.float32)


def ac_model(x, full):
    n = fm.getrealsize(x.size)
    return fm.autocorrelation(x, "plan" if (full or n < 16) else "half", f32=True)


def check_ac(got, x, model, what, path):
    n = fm.getrealsize(x.size)
    y = fm.as_complex(got[: 2 * x.size])
    check(y[:n], model, n, what, path, C_CORR * C_MAX, C_CORR * C_RMS)
    tail = np.zeros(2 * (x.size - n), np.float32)
    tail[0::2] = np.abs(x[n:])
    assert np.array_equal(got[2 * n: 2 * x.size].view(np.uint32), tail.view(np.uint32)), f"{what}: untransformed tail"


def _ac_params(sizes):
    return [pytest.param(size, full, id=f"{size}-{'full_size' if full else 'half_size'}",
)
            for size in sizes for full in (False, True)]


@pytest.mark.parametrize("size,full", _ac_params(AC_SIZES))
def test_autocorrelation_per_lag(gpu, size, full, monkeypatch):
    """tsdrgpu_autocorrelation, per lag relative to rms(r): the default half-size path (N >= 16) against the half-size plan model,
    TSDRGPU_AUTOCORR_FULL=1 against the N-point plan model; |noise| and a video-like capture."""
    if full:
        monkeypatch.setenv("TSDRGPU_AUTOCORR_FULL", "1")
    for kind in ("noise", "video"):
        x = ac_capture(size, kind)
        got = gpu.fft_autocorrelation(dev(x)).cpu().numpy()
        check_ac(got, x, ac_model(x, full), f"autocorr {size} {kind}", "full" if full else "half")


@pytest.mark.parametrize("size,full", _ac_params([16, 4096, 450_910, 1_409_090, (1 << 22) + 4]))
@pytest.mark.parametrize("layout", ["even_stride", "odd_stride", "base_4_aligned"])
def test_autocorrelation_batch_per_lag(gpu, size, layout, full, monkeypatch):
    """tsdrgpu_autocorrelation_batch (even sizes) on three captures in the three layouts of the production batches: even stride,
    odd stride (pair loads), even stride from a base that is only 4-byte aligned."""
    from tempestsdr_b200 import _native
    if full:
        monkeypatch.setenv("TSDRGPU_AUTOCORR_FULL", "1")
    batch = 3
    caps = [ac_capture(size, "noise" if b != 1 else "video", seed=b) for b in range(batch)]
    stride = size + (1 if layout == "odd_stride" else 2)
    off = 1 if layout == "base_4_aligned" else 0
    buf = torch.full((off + batch * stride + 8,), float("nan"), device="cuda")
    for b, c in enumerate(caps):
        buf[off + b * stride: off + b * stride + size] = dev(c)
    ans = torch.full((2 * size * batch,), float("nan"), device="cuda")
    gpu.chk(_native.lib().tsdrgpu_autocorrelation_batch(gpu._h, gpu.stream, ans.data_ptr(), buf.data_ptr() + 4 * off, size, batch, stride))
    got = ans.cpu().numpy().reshape(batch, -1)
    for b, c in enumerate(caps):
        check_ac(got[b], c, ac_model(c, full), f"autocorr batch {size} {layout} #{b}", "batch full" if full else "batch half")


@pytest.mark.parametrize("size", [4, 5, 4096, 70_001, 450_909, 1_409_090, 2_818_181])
def test_crosscorrelation_per_lag(gpu, size):
    """tsdrgpu_crosscorrelation against the N-point plan model, per lag relative to rms of the result."""
    n = fm.getrealsize(size)
    a, b = synth.noise_iq(size, seed=11), synth.noise_iq(size, seed=12)
    a[: 2 * n] += tone(fm.log2_of(n), n // 3) * np.float32(0.5)   # a correlated part, so the result is not flat noise
    b[: 2 * n] += tone(fm.log2_of(n), n // 3) * np.float32(0.5)
    da, db = dev(a), dev(b)
    gpu.fft_crosscorrelation(da, db, size)
    y = fm.as_complex(da.cpu().numpy()[: 2 * n])
    check(y, fm.crosscorrelation(fm.as_complex(a), fm.as_complex(b), "plan", f32=True), n, f"xcorr {size}", "plan", C_CORR * C_MAX, C_CORR * C_RMS)


# ------------------------------------------------------------------------------------------------ consumers
def test_framerate_detector_plots_per_element(gpu):
    """At the 25 MS/s capture size (1 409 090 samples, 2^20-point transforms), over three captures: both plots against float64
    running means of |r| of the half-size model, each element within the largest capture's lag bound."""
    from tempestsdr_b200.api import FrameRateDetector
    fs = 25_000_000
    size = FrameRateDetector.capture_size(fs)
    fmin, fmax, lmin, lmax = FrameRateDetector.windows(fs)
    n = fm.getrealsize(size)
    det = gpu.framerate_detector()
    mags, scales = [], []
    for k in range(3):
        x = ac_capture(size, "video" if k != 1 else "noise", seed=k)
        r = ac_model(x, False)
        mags.append(np.abs(r))
        scales.append(C_CORR * C_MAX * fm.bin_scale(r, n))
        (fo, fp), (lo, lp), calls = det.run(fs, dev(x))
        assert (fo, lo, calls) == (fmin, lmin, k + 1)
        want_f = np.mean([v[fmin:fmax] for v in mags], axis=0)
        want_l = np.mean([v[lmin:lmax] for v in mags], axis=0)
        tol_f = np.mean([v[fmin:fmax] for v in scales], axis=0)
        tol_l = np.mean([v[lmin:lmax] for v in scales], axis=0)
        for got, want, tol, what in ((fp, want_f, tol_f, "frame plot"), (lp, want_l, tol_l, "line plot")):
            worst = float(np.max(np.abs(got - want) / tol))
            _record(f"framerate {what}", "half", (C_CORR * worst, 0.0))
            assert worst <= 1.0, f"{what} after {k + 1} captures: {worst:.3f} of its bound"


def test_welch_spectrum_per_bin(gpu):
    """A 0 dB tone over a white floor 100 dB down, each bin against the float64 Welch model.  Bin k of segment s is within
    e_sk = C bin_scale(X_s)_k of its exact value; |X + e|^2 - |X|^2 <= 2 |X| |e| + |e|^2, and over the K segments of a report
    sum_s |X_sk| e_sk <= sqrt(sum_s |X_sk|^2) sqrt(sum_s e_sk^2) by Cauchy-Schwarz: with the report's normalisation each bin is
    held to its own power and to the rounding that reaches it, not to the largest bin."""
    fs, n, rate = 25_000_000, 4096, 100
    spec = f"welch:{n}:{rate}"
    K = segments_per_report(n, rate, fs)
    pairs = K * n // 2 + n // 2
    rng = np.random.default_rng(5)
    t = np.arange(pairs)
    x = np.exp(2j * np.pi * 0.1234567 * t) + 1e-5 * (rng.standard_normal(pairs) + 1j * rng.standard_normal(pairs)) / np.sqrt(2)
    iq = x.astype(np.complex64).view(np.float32)
    sp = gpu.spectrum()
    sp.set(spec, fs)
    got = sp.run(dev(iq)).cpu().numpy()
    want = WelchModel(spec, fs).run(iq)
    assert got.shape == (1, n) and len(want) == 1
    w = window64(n).astype(np.float32).astype(np.float64)
    xc = fm.as_complex(iq)
    segs = np.lib.stride_tricks.sliding_window_view(xc, n)[: K * n // 2: n // 2][:K]
    X = np.fft.fft(segs * w, axis=1)
    e2 = np.sum([(C_MAX * fm.bin_scale(s, n)) ** 2 for s in X], axis=0)       # sum over the segments of e_s,k^2
    norm = K * w.sum() ** 2
    P = want[0]
    err = np.abs(got[0] - P)
    allowed = np.fft.fftshift(2 * np.sqrt(np.sum(np.abs(X) ** 2, axis=0) * e2) + e2) / norm
    _record("welch per bin", "exact DFT", (float(np.max(err / allowed)), 0.0))
    assert np.all(err <= allowed), f"worst bin {int(np.argmax(err / allowed))}: {np.max(err / allowed):.3f} of its bound"
    assert np.max(P) / np.median(P) > 1e8                     # the floor really is far below the tone
