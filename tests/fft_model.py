"""numpy float64 models of the FFT family: the reference's radix-2 transform and the CUDA library's pass plans.

Both are written from their definitions, in float64 throughout, so that a float32 result can be compared with them bin by bin
and the difference read as float32 rounding.

* The reference transform (fft.c) is a radix-2 decimation-in-time FFT whose stage l rotates by (pi / 2^l)(1 + eps_l): it derives
  each stage's twiddle from the previous one by the half-angle recurrence c2 = sqrt((1 - c1) / 2), c1 = sqrt((1 + c1) / 2), which
  loses accuracy for small angles.  eps() replays that recurrence.  Forward transforms are scaled by 1/N, inverse ones are not,
  and only the first getrealsize(size) points are transformed.
* The CUDA library (fft.cu, fft_run) factors N = 2^m into 1, 2 or 3 passes of radix-2 layers.  The layers of a pass carry the
  same stage angles as the reference's stages at the same index bits (pass p's layer s uses eps[l_base + s]), but the twiddles
  between passes are exact: W_M^(m k) with M = N for the first split and M = N2 N3 inside a three-pass plan.  So a one-pass plan
  is the reference transform, and a plan of several passes differs from it by the stage-angle errors of its upper stages that
  the exact inter-pass twiddles leave out.  plan_fft() models that factorisation.
* The autocorrelation's default path transforms a real sequence of N points as N/2 complex pairs and finishes with the
  reference's last radix-2 stage (half_real_fft(); fft.cu, real_split_rn).
"""
import numpy as np

U = 2.0 ** -24        # unit roundoff of float32


def log2_of(n):
    return int(n).bit_length() - 1


def getrealsize(size):
    """fft.c's fft_getrealsize: the largest power of two <= size (1 for size 0)."""
    return 1 << max(log2_of(size), 0)


def eps(stages, inverse=False):
    """Relative angle error of each of the reference's first `stages` stages: the angle of stage l's twiddle step is
    (pi / 2^l)(1 + eps[l]).  The recurrence runs in double like the reference's; the error is read off in long double."""
    pi_l = np.longdouble("3.14159265358979323846264338327950288")
    out = np.zeros(stages)
    c1, c2 = -1.0, 0.0
    for l in range(stages):
        if l:
            ideal = pi_l / np.longdouble(1 << l)
            got = np.arctan2(np.longdouble(abs(c2)), np.longdouble(c1))
            out[l] = float(got / ideal - np.longdouble(1.0))
        n2 = np.sqrt((1.0 - c1) / 2.0)
        c1, c2 = float(np.sqrt((1.0 + c1) / 2.0)), float(-n2 if not inverse else n2)
    return out


_BITREV = {}


def _bitrev(m):
    if m not in _BITREV:
        r = np.zeros(1, np.int64)
        for _ in range(m):
            r = np.concatenate([2 * r, 2 * r + 1])
        _BITREV[m] = r
    return _BITREV[m]


def _tw(w, f32):
    """Twiddles as the library stores them (f32: rounded to float32 from double, as its host-built tables are) or exact."""
    return w.astype(np.complex64).astype(np.complex128) if f32 else w


def radix2(x, stage_eps, sign, f32=False):
    """Unscaled radix-2 DIT transform along the last axis, stage l rotating by sign * (pi / 2^l)(1 + stage_eps[l]); f32: with the
    twiddles rounded to float32."""
    n = x.shape[-1]
    m = log2_of(n)
    lead = x.shape[:-1]
    y = np.asarray(x, np.complex128)[..., _bitrev(m)]
    z = np.empty_like(y)
    for l in range(m):
        h = 1 << l
        w = _tw(np.exp(sign * 1j * np.pi * (np.arange(h) / h) * (1.0 + stage_eps[l])), f32)
        yv, zv = y.reshape(lead + (n // (2 * h), 2, h)), z.reshape(lead + (n // (2 * h), 2, h))
        t = yv[..., 1, :] * w
        np.add(yv[..., 0, :], t, out=zv[..., 0, :])
        np.subtract(yv[..., 0, :], t, out=zv[..., 1, :])
        y, z = z, y
    return y


def reference_fft(x, inverse=False, stage_eps=None):
    """The reference's fft_perform on complex x: the first getrealsize(len(x)) points, forward scaled by 1/N.  stage_eps: the
    stage errors to use instead of eps() (zeros give the true DFT)."""
    n = getrealsize(len(x))
    m = log2_of(n)
    e = eps(m, inverse) if stage_eps is None else stage_eps
    y = radix2(np.asarray(x, np.complex128)[:n], e, 1.0 if inverse else -1.0)
    return y if inverse else y / n


def default_plan(m, two_pass_max=21, split="floor"):
    """Line lengths (log2) of fft_run's passes for N = 2^m: one pass up to 2^11, two up to 2^two_pass_max (the shorter line first
    unless split == "ceil"), three above."""
    if m <= 11:
        return [m]
    if m <= two_pass_max and m <= 22:
        l1 = (m + 1) // 2 if split == "ceil" else m // 2
        return [l1, m - l1]
    l1 = (m + 2) // 3
    l2 = (m - l1 + 1) // 2
    return [l1, l2, m - l1 - l2]


def _plan(x, stage_eps, sign, passes, twiddle_sign, f32=False):
    if len(passes) == 1:
        return radix2(x, stage_eps, sign, f32)
    lead, n = x.shape[:-1], x.shape[-1]
    l1 = passes[0]
    n1, n2 = 1 << l1, n >> l1
    a = np.swapaxes(x.reshape(lead + (n1, n2)), -1, -2)                  # [n2, n1]: n = n2 + N2 n1
    a = radix2(a, stage_eps[:l1], sign, f32)                             # [n2, k1]
    e = (np.arange(n2, dtype=np.int64)[:, None] * np.arange(n1, dtype=np.int64)[None, :]) & (n - 1)
    a = a * _tw(np.exp(twiddle_sign * sign * 2j * np.pi * (e / n)), f32)     # W_N^(n2 k1)
    b = _plan(np.swapaxes(a, -1, -2), stage_eps[l1:], sign, passes[1:], twiddle_sign, f32)    # [k1, k2]
    return np.swapaxes(b, -1, -2).reshape(lead + (n,))                   # k = k1 + N1 k2


def plan_transform(x, inverse=False, passes=None, stage_eps=None, twiddle_sign=1.0, f32=False):
    """Unscaled transform of a power-of-two length along the last axis, as the CUDA library factors it.  f32: every twiddle rounded
    to float32, as the library's tables hold them (the inter-pass ones only approximately: the library forms them as a table entry
    times sincospif)."""
    n = x.shape[-1]
    m = log2_of(n)
    e = eps(m, inverse) if stage_eps is None else stage_eps
    p = default_plan(m) if passes is None else passes
    assert sum(p) == m, (p, m)
    if m == 0:
        return np.asarray(x, np.complex128).copy()
    return _plan(np.asarray(x, np.complex128), e, 1.0 if inverse else -1.0, p, twiddle_sign, f32)


def plan_fft(x, inverse=False, passes=None, stage_eps=None, twiddle_sign=1.0, f32=False):
    """tsdrgpu_fft's transform of complex x: the first getrealsize(len(x)) points, forward scaled by 1/N.  twiddle_sign = -1
    gives every inter-pass twiddle the wrong sign (a mutant for the tests)."""
    n = getrealsize(len(x))
    y = plan_transform(np.asarray(x, np.complex128)[:n], inverse, passes, stage_eps, twiddle_sign, f32)
    return y if inverse else y / n


def half_real_fft(x, inverse=False, passes=None, stage_eps=None, f32=False):
    """Unscaled N-point transform of a real sequence the way the autocorrelation's default path forms it: the N/2-point plan of
    z[j] = x[2j] + i x[2j+1], then E = (Z[k] + conj Z[-k]) / 2, O = (Z[k] - conj Z[-k]) / 2i and the reference's last stage,
    X[k] = E + w O, X[k + N/2] = E - w O with w = exp(-+ i pi k / (N/2) (1 + eps_{m-1}))."""
    x = np.asarray(x, np.float64)
    n = x.size
    m = log2_of(n)
    half = n // 2
    e = eps(m, inverse) if stage_eps is None else stage_eps
    z = plan_transform(x[0::2] + 1j * x[1::2], inverse, passes, e[: m - 1], f32=f32)
    zm = np.conj(z[(-np.arange(half)) % half])
    ev, od = (z + zm) / 2, (z - zm) / 2j
    w = _tw(np.exp((1.0 if inverse else -1.0) * 1j * np.pi * (np.arange(half) / half) * (1.0 + e[m - 1])), f32)
    return np.concatenate([ev + w * od, ev - w * od])


def autocorrelation(real, path="reference", f32=False):
    """fft.c's fft_autocorrelation: the first N = getrealsize(size) lags (complex), IFFT(|FFT(x)| / N) with the inverse unscaled.
    path: "reference" (the reference's transforms), "plan" (the library's N-point plans, TSDRGPU_AUTOCORR_FULL=1) or "half" (the
    library's default half-size transforms; N >= 16)."""
    x = np.asarray(real, np.float64)
    n = getrealsize(x.size)
    x = x[:n]
    if path == "reference":
        return reference_fft(np.abs(reference_fft(x + 0j)) + 0j, inverse=True)
    if path == "plan":
        return plan_fft(np.abs(plan_fft(x + 0j, f32=f32)) + 0j, inverse=True, f32=f32)
    assert path == "half" and n >= 16
    return half_real_fft(np.abs(half_real_fft(x, f32=f32)) / n, inverse=True, f32=f32)


def crosscorrelation(a, b, path="reference", f32=False):
    """fft.c's fft_crosscorrelation on complex a, b: IFFT(conj(FFT a) FFT b), the first getrealsize(len) points.
    path: "reference" or "plan"."""
    if path == "reference":
        return reference_fft(np.conj(reference_fft(a)) * reference_fft(b), inverse=True)
    return plan_fft(np.conj(plan_fft(a, f32=f32)) * plan_fft(b, f32=f32), inverse=True, f32=f32)


# How far each plan model lies from reference_fft: max|plan - reference| over a transform of complex unit-variance noise
# (synth.noise_iq(N, seed=log2 N)), in units of u log2 N rms(reference), the larger of the two directions, times two.  Below 2^12 the
# plan is one pass and equals the reference model.  The deviation is the stage-angle error of the upper stages that the exact
# inter-pass twiddles leave out; it grows with eps (1.2e-6 at stage 20, 7.5e-5 at stage 23) and reaches float32 rounding at 2^23.
PLAN_DEVIATION = {
    "default": {12: 1e-6, 13: 3.3e-6, 14: 5.5e-6, 15: 3.1e-5, 16: 2e-4, 17: 1.7e-4, 18: 9.2e-4, 19: 2.1e-3, 20: 1.33e-2,
                21: 2.5e-2, 22: 1.0, 23: 5.9, 24: 11.2},
    "2pass_max_20": {21: 0.39},                                                 # 7+7+7 instead of 10+11
    "split_ceil": {13: 6.3e-6, 15: 6.4e-5, 17: 3.4e-4, 19: 3.6e-3, 21: 5.3e-2},  # the longer line first
}
PLAN_SHAPES = {"default": {}, "2pass_max_20": {"two_pass_max": 20}, "split_ceil": {"split": "ceil"}}


def plan_deviation(m, shape="default"):
    """The pinned deviation of a plan shape from the reference model at N = 2^m (units of u log2 N rms)."""
    return PLAN_DEVIATION[shape].get(m, PLAN_DEVIATION["default"].get(m, 0.0))


def as_complex(iq):
    """Interleaved float32 I,Q -> complex128."""
    return np.ascontiguousarray(iq, np.float32).view(np.complex64).astype(np.complex128)


def rms(v):
    return float(np.sqrt(np.mean(np.abs(v) ** 2))) if np.size(v) else 0.0


def bin_scale(model, n):
    """Per-bin error scale of a float32 radix-2 transform whose exact output is `model` (N bins): u sqrt(log2 N) sqrt(G_k) with
    G_k = sum over s = 0..log2 N of 2^s / N * S_s(k), S_s(k) = sum of |model_k'|^2 over k' = k mod 2^s.

    In a decimation-in-time transform, bin b of a block after stage l holds the part of the output at the bins k = b mod 2^(l+1)
    (a pass plan keeps that correspondence: k = k1 + N1 k2).  Each block value is rounded with an error up to u times its size,
    and that error reaches only the output bins of its class, unchanged in size by the later stages.  The N / 2^(l+1) blocks round
    independently, so stage l adds u^2 2^(l+1) / N S_(l+1)(k) to the error variance of bin k.  For a flat spectrum (noise,
    impulses) every term is rms^2 and the scale is about u log2 N rms, the bound of the module docstring of
    tests/test_fft_float64_model.py; where the output is concentrated -- a tone's bin, a non-negative capture's zero lag -- the
    error lands on the bins (lags) that share its residue modulo large powers of two, and the scale grows there and only there."""
    p = np.abs(np.asarray(model)) ** 2
    L = max(log2_of(n), 1)
    k = np.arange(n, dtype=np.int64)
    g = np.zeros(n)
    for s in range(log2_of(n) + 1):
        g += (2.0 ** s / n) * p.reshape(n >> s, 1 << s).sum(axis=0)[k & ((1 << s) - 1)]
    return U * np.sqrt(L) * np.sqrt(g)


def bin_units(y, model, n):
    """(max_k |e_k| / bin_scale_k, rms(e) in units of u sqrt(log2 N) rms(model)), e = y - model."""
    e = np.abs(np.asarray(y) - np.asarray(model))
    if not e.any():
        return 0.0, 0.0
    return float(np.max(e / bin_scale(model, n))), rounding_units(y, model, n)[1]


def rounding_units(y, model, n):
    """(max|e|, rms(e)) of e = y - model in units of u log2 N rms(model) and u sqrt(log2 N) rms(model).  A one-point transform is
    counted as one stage."""
    e = np.abs(np.asarray(y) - np.asarray(model))
    r = rms(model)
    L = max(log2_of(n), 1)
    if r == 0.0:
        return (0.0, 0.0) if not e.any() else (np.inf, np.inf)
    return float(e.max()) / (U * L * r), rms(e) / (U * np.sqrt(L) * r)
