"""Richardson-Lucy deconvolution along the lines (the deblur step) as include/tsdrgpu.h defines it, in numpy float32.

Every float operation here is one numpy float32 operation (rounded to float32, never contracted), in the order the definition
gives, so the GPU's output is expected bit for bit.  `deblur_frame` works on whole frames one tap at a time; `deblur_literal`
walks the definition pixel by pixel and is only fast enough for tiny frames.  The taps come from the library's own
`tsdrgpu_deblur_taps` (`deblur_taps`), or from `taps_reference`, an independent float64 computation the tests compare it with.
"""
import ctypes as C
import math

import numpy as np

F32 = np.float32
EPS = F32(2.0 ** -30)                   # TSDRGPU_DEBLUR_EPS


def valid_mask(img):
    """Not a marker (|v| > 250, which includes +-inf) and not NaN."""
    with np.errstate(invalid="ignore"):
        return ~((img > 250.0) | (img < -250.0)) & (img == img)


def radius(sigma_centi):
    """R = ceil(3 sigma) for sigma = sigma_centi / 100, in integers."""
    return (3 * sigma_centi + 99) // 100


def taps_reference(sigma_centi):
    """exp(-j^2 / (2 sigma^2)) / sum over j in [-R, R], in float64, then rounded once to float32."""
    s = sigma_centi / 100.0
    r = radius(sigma_centi)
    e = [math.exp(-(j * j) / (2.0 * s * s)) for j in range(-r, r + 1)]
    tot = math.fsum(e)
    return np.array([x / tot for x in e], F32)


def deblur_taps(sigma_centi):
    """The taps as the library computes them (tsdrgpu_deblur_taps)."""
    from tempestsdr_b200 import _native as N
    lib = N.lib()
    r = C.c_int()
    buf = (C.c_float * 25)()
    assert lib.tsdrgpu_deblur_taps(sigma_centi, buf, C.byref(r)) == 0
    return np.array(buf[:2 * r.value + 1], F32)


def _lines(frame, w, h):
    img = np.asarray(frame, F32).reshape(h, w)
    m = valid_mask(img)
    with np.errstate(invalid="ignore"):
        d = np.where(m & (img > 0), np.minimum(img, F32(1)), F32(0)).astype(F32)
    return img, m, d


def _corr(a, k):
    """B(a) for every line of a (rows), a already zero where m = 0: left to right over the taps, zeros outside the line."""
    h, w = a.shape
    r = (len(k) - 1) // 2
    p = np.pad(a, ((0, 0), (r, r)))
    s = np.zeros((h, w), F32)
    for j in range(2 * r + 1):
        s = s + k[j] * p[:, j:j + w]
    return s


def deblur_frame(frame, w, h, sigma_centi, iterations=20, taps=None):
    """One frame (w * h float32 pixels, row-major) -> its deblurred output; invalid pixels pass through bit for bit."""
    k = deblur_taps(sigma_centi) if taps is None else np.asarray(taps, F32)
    img, m, d = _lines(frame, w, h)
    with np.errstate(divide="ignore"):
        rn = np.where(m, F32(1) / _corr(m.astype(F32), k), F32(0)).astype(F32)
    u = d
    for _ in range(iterations):
        b = _corr(u, k) * rn
        q = np.where(m, d / np.maximum(b, EPS), F32(0)).astype(F32)
        u = np.where(m, u * (_corr(q, k) * rn), F32(0)).astype(F32)
    out = np.where(m, np.minimum(u, F32(1)), img).astype(F32)
    return out.reshape(-1)


def deblur_frames(frames, w, h, sigma_centi, iterations=20, taps=None):
    """Frames back to back (any number) -> the deblurred output of each."""
    k = deblur_taps(sigma_centi) if taps is None else taps
    f = np.asarray(frames, F32).reshape(-1, w * h)
    return np.concatenate([deblur_frame(x, w, h, sigma_centi, iterations, k) for x in f]) if len(f) else np.zeros(0, F32)


def deblur_literal(frame, w, h, sigma_centi, iterations=20, taps=None):
    """The definition pixel by pixel, with float32 scalars: a check on deblur_frame, for tiny frames only."""
    k = [F32(x) for x in (deblur_taps(sigma_centi) if taps is None else taps)]
    r = (len(k) - 1) // 2
    img = np.asarray(frame, F32).reshape(h, w)
    out = img.copy()

    def valid(v):
        return not (v > 250.0 or v < -250.0) and v == v

    for y in range(h):
        row = img[y]
        m = [1 if valid(v) else 0 for v in row]
        d = [F32(min(max(F32(v), F32(0)), F32(1))) + F32(0) if m[x] else F32(0) for x, v in enumerate(row)]

        def B(a, x):
            s = None
            for j in range(-r, r + 1):
                xx = x + j
                mj, aj = (m[xx], a[xx]) if 0 <= xx < w else (0, F32(0))
                t = F32(k[j + r] * F32(F32(mj) * aj))
                s = t if s is None else F32(s + t)
            return s

        rn = [F32(F32(1) / B([F32(1)] * w, x)) if m[x] else None for x in range(w)]
        u = list(d)
        for _ in range(iterations):
            q = [F32(d[x] / max(F32(B(u, x) * rn[x]), EPS)) if m[x] else F32(0) for x in range(w)]
            u = [F32(u[x] * F32(B(q, x) * rn[x])) if m[x] else F32(0) for x in range(w)]
        for x in range(w):
            if m[x]:
                out[y, x] = min(u[x], F32(1))
    return out.reshape(-1)
