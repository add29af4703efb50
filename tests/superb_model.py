"""numpy models of the superbandwidth alignment and stitch (superbandwidth.c:67-152; csrc/fft.cu, csrc/superb_mgpu.cu).

* abs_diff() is complex_to_abs_diff in float32, seed quirk included: the first pair's "previous magnitude" is I^2 + Q^2 without
  the square root.  numpy's float32 arithmetic rounds every operation and never contracts, so it is exact.
* bestfit() is superb_bestfit: the reference's sizing of the correlation, abs_diff, the float64 cross-correlation of
  tests/fft_model.py with the reference's stage angles, and the first maximum of |xcorr|.  It also returns the margin, the gap
  between the largest and second-largest |xcorr| in units of u log2(nd) rms(xcorr): a lag is only required to be exact where
  the margin exceeds the rounding of an nd-point correlation (lag_bound()).
* stitch_reference() is superb_ondataready in float64: rotate each hop by its offset, transform it (scaled by 1/N), place the
  spectra side by side and invert the leading power of two of the H N points (fft.c:101-105); for H not a power of two the
  rest stays as spectra.
* stitch_one_gpu() is the dataflow of tsdrgpu_superb_stitch: the same steps with the library's pass plans (fft_model.plan_fft,
  float32 twiddle tables).
* stitch_sharded() is the dataflow of tsdrgpu_superb_mgpu_stitch: the plan's forward transform per hop, the alignment as a
  phase ramp e^{+2 pi i m lag / N} on the spectrum, the plan's inverse of every block B_t[u] = X~[H u + t], then the
  reference's last log2 H radix-2 stages across the blocks with their own angle errors, then |.|.

Every model takes true_dft=True to use exact stage angles (TSDRGPU_FFT_TRUE_DFT=1).
"""
import numpy as np

from tests import fft_model as fm

C_CORR = 2.0          # rounding of a float32 correlation in units of u log2(n) rms (tests/test_fft_float64_model.py)


def _eps(m, true_dft):
    return np.zeros(m) if true_dft else fm.eps(m)


def abs_diff(iq):
    """complex_to_abs_diff on interleaved float32 (an even number of floats): out[2i] = |x_i| - |x_{i-1}|, out[2i+1] = 0, with
    |x_{-1}| replaced by I_0^2 + Q_0^2."""
    d = np.array(iq, dtype=np.float32, copy=True)
    assert d.size % 2 == 0
    if d.size == 0:
        return d
    i, q = d[0::2], d[1::2]
    with np.errstate(all="ignore"):
        cur = np.sqrt(i * i + q * q)
        prev = np.empty_like(cur)
        prev[0] = i[0] * i[0] + q[0] * q[0]
        prev[1:] = cur[:-1]
        out = np.zeros_like(d)
        out[0::2] = cur - prev
    return out


def correlation_pairs(size_floats, sif):
    """superb_bestfit's sizing (superbandwidth.c:84-86): nd complex pairs, or None where (size / sif) sif < 2 (the library refuses
    this; the reference reads past a one-float buffer)."""
    size = (size_floats // sif) * sif
    if size < 2:
        return None
    return fm.getrealsize(size) // 2


def first_max(mag):
    """The reference's scan: element 0 first, then move on a strict '>' only (NaN never wins, a NaN at 0 keeps 0)."""
    if mag.size == 0 or np.isnan(mag[0]):
        return 0
    return int(np.argmax(np.where(np.isnan(mag), -np.inf, mag)))


def lag_bound(nd):
    """How far the GPU's |xcorr| may lie from the reference model's at nd points, in units of u log2(nd) rms: the float32
    correlation's rounding plus the plan's pinned deviation (twice: forward and inverse), on each of the two top values."""
    m = fm.log2_of(nd)
    return 2.0 * (C_CORR + 2.0 * fm.plan_deviation(m))


def bestfit(hop0, hopi, size_floats, sif, true_dft=False):
    """(offset in floats as superb_bestfit returns it, margin in units of u log2(nd) rms(xcorr), nd)."""
    nd = correlation_pairs(size_floats, sif)
    assert nd is not None and nd >= 1
    a = fm.as_complex(abs_diff(np.asarray(hop0, np.float32)[: 2 * nd]))
    b = fm.as_complex(abs_diff(np.asarray(hopi, np.float32)[: 2 * nd]))
    m = fm.log2_of(nd)
    e = _eps(m, true_dft)
    with np.errstate(all="ignore"):
        xc = fm.reference_fft(np.conj(fm.reference_fft(a, stage_eps=e)) * fm.reference_fft(b, stage_eps=e), inverse=True, stage_eps=e)
        mag = np.abs(xc)
    lag = first_max(mag)
    if nd < 2 or not np.all(np.isfinite(mag)):
        return 2 * lag, 0.0, nd
    top = np.partition(mag, nd - 2)[nd - 2:]
    r = fm.rms(xc)
    margin = float(top[1] - top[0]) / (fm.U * max(m, 1) * r) if r > 0 else 0.0
    return 2 * lag, margin, nd


def _rotate(hop, n, offset_floats):
    return np.roll(fm.as_complex(np.asarray(hop, np.float32)[: 2 * n]), -(offset_floats // 2))


def _stitch(hops, sif, offsets, forward, inverse):
    n = fm.getrealsize(np.asarray(hops[0]).size // 2)
    if offsets is None:
        offsets = [0] + [bestfit(hops[0], h, 2 * n, sif)[0] for h in hops[1:]]
    big = np.concatenate([forward(_rotate(h, n, o)) for h, o in zip(hops, offsets)])
    tp = fm.getrealsize(big.size)
    return np.concatenate([inverse(big[:tp]), big[tp:]]), list(offsets)


def stitch_reference(hops, sif, offsets=None, true_dft=False):
    """superb_ondataready: (H N complex samples, offsets in floats).  offsets: the alignment to use instead of bestfit()'s."""
    n = fm.getrealsize(np.asarray(hops[0]).size // 2)
    tp = fm.getrealsize(len(hops) * n)
    ef, ei = _eps(fm.log2_of(n), true_dft), _eps(fm.log2_of(tp), true_dft)
    return _stitch(hops, sif, offsets, lambda x: fm.reference_fft(x, stage_eps=ef),
                   lambda x: fm.reference_fft(x, inverse=True, stage_eps=ei))


def stitch_one_gpu(hops, sif, offsets=None, true_dft=False):
    """tsdrgpu_superb_stitch's dataflow: the reference's steps with the library's pass plans (float32 twiddles)."""
    n = fm.getrealsize(np.asarray(hops[0]).size // 2)
    tp = fm.getrealsize(len(hops) * n)
    ef, ei = _eps(fm.log2_of(n), true_dft), _eps(fm.log2_of(tp), true_dft)
    return _stitch(hops, sif, offsets, lambda x: fm.plan_fft(x, stage_eps=ef, f32=True),
                   lambda x: fm.plan_fft(x, inverse=True, stage_eps=ei, f32=True))


def stitch_sharded(hops, lags, true_dft=False):
    """tsdrgpu_superb_mgpu_stitch's dataflow: |y| of the H N-point stitch, from the hops and their lags in complex samples."""
    H = len(hops)
    n = fm.getrealsize(np.asarray(hops[0]).size // 2)
    log2n, log2h = fm.log2_of(n), fm.log2_of(H)
    assert 1 << log2h == H
    e = _eps(log2n + log2h, true_dft)
    m = np.arange(n, dtype=np.int64)
    spec = []
    for h, lag in zip(hops, lags):
        x = fm.plan_fft(fm.as_complex(np.asarray(h, np.float32)[: 2 * n]), stage_eps=e[:log2n], f32=True)
        spec.append(x * np.exp(2j * np.pi * ((m * int(lag)) & (n - 1)) / n))
    big = np.concatenate(spec)
    rev = fm._bitrev(log2h)
    y = np.concatenate([fm.plan_transform(big[rev[b]::H], inverse=True, stage_eps=e[:log2n], f32=True) for b in range(H)])
    for s in range(log2h):
        h = n << s
        w = np.exp(1j * np.pi * (np.arange(h) / h) * (1.0 + e[log2n + s]))
        yv = y.reshape(H * n // (2 * h), 2, h)
        t = yv[:, 1, :] * w
        y = np.stack([yv[:, 0, :] + t, yv[:, 0, :] - t], axis=1).reshape(-1)
    return np.abs(y)


def units(got, model, n):
    """(max, rms) of got - model in units of u log2(n) rms(model) and u sqrt(log2 n) rms(model) (fft_model.rounding_units)."""
    return fm.rounding_units(got, model, n)


def lag_of_shift(shift, nd):
    """The lag superb_bestfit finds for a hop that starts `shift` complex samples after hop 0 (before it: shift < 0)."""
    return (-shift) % nd


def shift_for_lag(lag, nd):
    """A hop start that puts the correlation peak on `lag`: before hop 0 for lags in the lower half, after it above."""
    return -lag if lag <= nd // 2 else nd - lag


def shifted_hops(pairs, shifts, seed, noise=0.05):
    """Hop q = hop 0's signal starting shifts[q] complex samples later (earlier if negative), with independent noise on top:
    complex unit-variance noise as the common signal, so the correlation peak is known and stands far above the rest."""
    from tempestsdr_b200 import synth
    lo, hi = min(0, min(shifts)), max(0, max(shifts))
    base = synth.noise_iq(pairs + hi - lo, seed=seed)
    return [np.ascontiguousarray(base[2 * (s - lo): 2 * (s - lo + pairs)] + synth.noise_iq(pairs, seed=seed + 1 + q, scale=noise))
            for q, s in enumerate(shifts)]


# ---- pinned numbers
# The compiled reference against stitch_reference (tests/test_superb_sweep.py, CPU), head and tail: a forward and an inverse
# float32 transform in a row, so twice one transform's constant, as for the correlations (measured up to 1.03 max, 0.62 rms).
REFERENCE_UNITS = (2.0, 2.0)
# The GPU against the model of its own dataflow, one-GPU and sharded alike: measured worst case on an H100 SXM (700 W) 1.49 max
# (sharded, H = 8) and 0.82 rms (one-GPU, 3 x 2^12 and 4 x 2^21), plus a third to a half again.
C_OWN_MAX = 2.0
C_OWN_RMS = 1.25
# stitch_one_gpu against stitch_reference, (head max, head rms, tail max, tail rms) per (H, log2 N), and stitch_sharded
# against |stitch_reference|, (max, rms) per (H, log2 N): measured on the sweep's inputs, rounded up by a quarter.
ONE_GPU_DEVIATION = {(1, 6): (0.77, 0.66, 0.0, 0.0), (2, 10): (0.75, 0.51, 0.0, 0.0), (3, 12): (1.12, 0.73, 0.45, 0.42),
                     (4, 13): (1.17, 0.69, 0.0, 0.0), (5, 16): (1.0, 0.66, 0.43, 0.4), (8, 17): (1.6, 0.62, 0.0, 0.0),
                     (16, 18): (1.88, 0.73, 0.0, 0.0), (4, 21): (4.88, 2.96, 0.0, 0.0)}
SHARDED_DEVIATION = {(2, 12): (1.0, 0.7), (2, 16): (0.97, 0.65), (4, 12): (1.34, 0.64), (4, 16): (1.38, 0.62), (4, 21): (6.68, 4.6),
                     (8, 12): (1.46, 0.58), (8, 16): (1.68, 0.61)}


def one_gpu_deviation(H, n):
    return ONE_GPU_DEVIATION[(H, fm.log2_of(n))]


def sharded_deviation(H, n):
    return SHARDED_DEVIATION[(H, fm.log2_of(n))]
