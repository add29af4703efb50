"""float64 numpy model of the coherent superbandwidth stitch (include/tsdrgpu.h, tsdrgpu_superb_stitch_coherent; csrc/superband.cu).

* schedule() is the hop plan: N, D, the centres c_i and the retune offsets round(c_i fs / N) (tsdrgpu_superband_schedule).
* stitch() is the definition with numpy's transforms: the hops' spectra, the joins in their chaining order (tau0 from the N-point
  inverse of u C, the two refinement stages, g and rho) and the assembled L-point inverse.  The candidates' phasors are stepped from
  a base formed from integers, so a stage costs two exponentials per bin.
* literal() restates the same definition with direct DFTs and per-bin and per-candidate loops, for small N only.
* assemble() is step 5-6 alone, from given estimates: the GPU's own estimates put into it isolate the samples' rounding from the
  estimates' (a pick of T that differs by one step changes every sample of a hop).
* hops_from_truth() cuts synthetic hops from a wideband truth at H fs: shift to c_i, a linear-phase FIR band limit to +-fs/2,
  decimation, then a known circular fractional delay, LO phase and gain per hop and noise at a given SNR.
"""
import numpy as np

from tests import fft_model as fm

CAND = np.arange(-32, 33)


def _round(x):
    """round half away from zero, as llround"""
    return int(np.sign(x) * np.floor(abs(x) + 0.5))


def schedule(fs, fv, H, o):
    """(N, D, centres c_i, offsets in Hz) of coherent:<H>:<o> at fs and refresh rate fv."""
    n = fm.getrealsize(10 * int(np.floor(fs / fv)))
    d = 2 * _round((1.0 - o / 100.0) * n / 2.0)
    c = [(2 * i - (H - 1)) * d // 2 for i in range(H)]
    return n, d, c, [_round(ci * fs / n) for ci in c]


def spacing(n, o):
    return 2 * _round((1.0 - o / 100.0) * n / 2.0)


def join_order(H):
    """[(b, a)] in chaining order: outward from r = (H-1)//2, upward first."""
    r = (H - 1) // 2
    return [(b, b - 1) for b in range(r + 1, H)] + [(b, b + 1) for b in range(r - 1, -1, -1)]


def record_index(b, H):
    r = (H - 1) // 2
    return b - (1 if b > r else 0)


def _first_max(mag):
    return int(np.argmax(mag))


def _crossfade(M):
    t = np.pi * (2 * np.arange(M) + 1) / (2 * M)
    return np.sin(t), np.cos(t)


def _ramp(x, T, n, sign):
    """e^{sign 2 pi i x T / (1024 n)} with x T reduced mod 1024 n in integers"""
    q = 1024 * n
    e = (np.asarray(x, np.int64) * np.int64(T)) % q
    return np.exp(sign * 2j * np.pi * (e / q))


class _Hops:
    def __init__(self, hops, d, spectra=None):
        self.H = len(hops)
        pairs = min(np.asarray(h).size // 2 for h in hops)
        self.n = fm.getrealsize(pairs)
        self.d, self.m = d, self.n - d
        self.c = [(2 * i - (self.H - 1)) * d // 2 for i in range(self.H)]
        self.X = spectra if spectra is not None else [np.fft.fft(fm.as_complex(h)[: self.n]) / self.n for h in hops]
        self.corr = {(self.H - 1) // 2: None}          # hop -> (g, T, kappa0), None: the reference hop

    def bins(self, i, kappa, corrected=True):
        v = self.X[i][(np.asarray(kappa, np.int64) - self.c[i]) % self.n]
        cr = self.corr.get(i) if corrected else None
        if cr is not None:
            g, T, k0 = cr
            v = g * v * _ramp(np.asarray(kappa, np.int64) - k0, T, self.n, -1.0)
        return v


def _estimate(P, a, b, evaluate):
    n, M = P.n, P.m
    kappa0 = P.c[max(a, b)] - n // 2
    kap = kappa0 + np.arange(M, dtype=np.int64)
    A, B = P.bins(a, kap), P.bins(b, kap, corrected=False)
    s, c = _crossfade(M)
    u = s * s * (c * c)
    C = u * A * np.conj(B)
    S_int = evaluate("int", C, None)
    t0 = _first_max(np.abs(S_int))
    if t0 > n // 2:
        t0 -= n
    T1 = 1024 * t0 + 32 * CAND
    S1 = evaluate("cand", C, T1)
    T1 = int(T1[_first_max(np.abs(S1))])
    T2 = T1 + CAND
    S2 = evaluate("cand", C, T2)
    k = _first_max(np.abs(S2))
    T, S = int(T2[k]), S2[k]
    na, nb = float(np.sum(u * np.abs(A) ** 2)), float(np.sum(u * np.abs(B) ** 2))
    if nb == 0.0:
        g, T, rho = 0j, 0, 0.0
    else:
        g = S / nb
        rho = float(abs(S) / np.sqrt(na * nb)) if na * nb > 0 else 0.0
    return dict(hop=b, neighbour=a, tau0=t0, kappa0=int(kappa0), tau_1024=T, tau=T / 1024.0, g=complex(g), rho=rho)


def _evaluate_fast(n):
    def ev(kind, C, T):
        M = C.size
        if kind == "int":
            z = np.zeros(n, complex)
            z[:M] = C
            return np.fft.ifft(z) * n
        m = np.arange(M, dtype=np.int64)
        step = int(T[1] - T[0])
        base = C * _ramp(m, int(T[32]), n, 1.0)
        w = _ramp(m, step, n, 1.0)
        out = np.empty(T.size, complex)
        out[32] = base.sum()
        up, dn = base.copy(), base.copy()
        for j in range(1, 33):
            up *= w
            dn *= np.conj(w)
            out[32 + j], out[32 - j] = up.sum(), dn.sum()
        return out
    return ev


def assemble(P, records):
    """steps 5-6 from the records (dicts with hop, kappa0, tau_1024, g): the L interleaved float64 pairs as complex"""
    H, n, M = P.H, P.n, P.m
    for r in records:
        P.corr[r["hop"]] = (r["g"], r["tau_1024"], r["kappa0"])
    L = H * n
    Y = np.zeros(L, complex)
    s, c = _crossfade(M)
    for i in range(H):
        kap = P.c[i] - n // 2 + np.arange(n, dtype=np.int64)
        w = np.ones(n)
        if i > 0:
            w[:M] = s * s
        if i + 1 < H:
            w[n - M:] = c * c
        Y[kap % L] += w * P.bins(i, kap)
    return np.fft.ifft(Y) * L


def stitch(hops, d, spectra=None):
    """(y as complex, records in record_index order) of the coherent stitch of interleaved float32 hops with spacing d."""
    P = _Hops(hops, d, spectra)
    recs = {}
    for b, a in join_order(P.H):
        e = _estimate(P, a, b, _evaluate_fast(P.n))
        P.corr[b] = (e["g"], e["tau_1024"], e["kappa0"])
        recs[b] = e
    out = [recs[b] for b in sorted(recs)]
    return assemble(_Hops(hops, d, P.X), out), out


def second_peak_gap(hops, d):
    """Per join, (|S| at tau0 - the second largest |S| over integers) / (u log2 N rms |S|): where it is small, float32 rounding
    may pick another integer lag than float64 does."""
    P = _Hops(hops, d)
    gaps = {}
    ev = _evaluate_fast(P.n)

    def spy(kind, C, T):
        out = ev(kind, C, T)
        if kind == "int":
            mag = np.sort(np.abs(out))
            gaps[len(gaps)] = (mag[-1] - mag[-2]) / (fm.U * fm.log2_of(P.n) * fm.rms(out))
        return out
    for b, a in join_order(P.H):
        e = _estimate(P, a, b, spy)
        P.corr[b] = (e["g"], e["tau_1024"], e["kappa0"])
    return [gaps[k] for k in range(len(gaps))]


def literal(hops, d):
    """The definition restated with direct DFTs and loops (small N): (y, records)."""
    H = len(hops)
    pairs = min(np.asarray(h).size // 2 for h in hops)
    n = fm.getrealsize(pairs)
    M, L, r = n - d, H * n, (H - 1) // 2
    kk = np.arange(n)
    F = np.exp(-2j * np.pi * np.outer(kk, kk) / n)
    X = [F @ fm.as_complex(h)[:n] / n for h in hops]
    c = [(2 * i - (H - 1)) * d / 2 for i in range(H)]
    corr = {r: (1.0, 0.0, 0)}

    def bin_of(i, kappa, corrected=True):
        v = X[i][int(kappa - c[i]) % n]
        if corrected:
            g, tau, k0 = corr[i]
            v = g * v * np.exp(-2j * np.pi * (kappa - k0) * tau / n)
        return v

    def S(Cm, tau):
        return sum(Cm[m] * np.exp(2j * np.pi * m * tau / n) for m in range(M))

    recs = {}
    for b, a in join_order(H):
        k0 = int(c[max(a, b)] - n / 2)
        Cm, na, nb = [], 0.0, 0.0
        for m in range(M):
            th = np.pi * (m + 0.5) / M
            u = np.sin(th) ** 2 * np.cos(th) ** 2
            A, B = bin_of(a, k0 + m), bin_of(b, k0 + m, corrected=False)
            Cm.append(u * A * np.conj(B))
            na += u * abs(A) ** 2
            nb += u * abs(B) ** 2
        Cv = np.array(Cm)
        mags = [abs(np.sum(Cv * np.exp(2j * np.pi * np.arange(M) * t / n))) for t in range(n)]
        t0 = int(np.argmax(mags))
        t0 = t0 - n if t0 > n // 2 else t0
        best = None
        for j in CAND:
            v = abs(S(Cm, t0 + j / 32))
            if best is None or v > best[0]:
                best = (v, t0 + j / 32)
        t1, best = best[1], None
        for j in CAND:
            Sv = S(Cm, t1 + j / 1024)
            if best is None or abs(Sv) > abs(best[0]):
                best = (Sv, t1 + j / 1024)
        Sv, tau = best
        if nb == 0:
            g, tau, rho = 0.0, 0.0, 0.0
        else:
            g, rho = Sv / nb, (abs(Sv) / np.sqrt(na * nb) if na * nb > 0 else 0.0)
        corr[b] = (g, tau, k0)
        recs[b] = dict(hop=b, neighbour=a, tau0=t0, kappa0=k0, tau_1024=int(round(tau * 1024)), tau=tau, g=complex(g), rho=float(rho))
    Y = np.zeros(L, complex)
    for kappa in range(-L // 2, L // 2):
        for i in range(H):
            if not (c[i] - n / 2 <= kappa < c[i] + n / 2):
                continue
            w = 1.0
            if i > 0 and kappa - (c[i] - n / 2) < M:
                w = np.sin(np.pi * (kappa - (c[i] - n / 2) + 0.5) / M) ** 2
            elif i + 1 < H and kappa >= c[i + 1] - n / 2:
                w = np.cos(np.pi * (kappa - (c[i + 1] - n / 2) + 0.5) / M) ** 2
            Y[kappa % L] += w * bin_of(i, kappa)
    y = np.zeros(L, complex)
    t = np.arange(L)
    for k0 in range(0, L, 512):
        ks = np.arange(k0, min(L, k0 + 512))
        y += np.exp(2j * np.pi * np.outer(t, ks) / L) @ Y[ks]
    return y, [recs[b] for b in sorted(recs)]


# ---- synthetic hops from a known wideband truth
def lowpass(taps, cutoff):
    """linear-phase Kaiser-windowed FIR, cutoff in cycles per sample"""
    d = np.arange(taps) - (taps - 1) / 2
    h = 2 * cutoff * np.sinc(2 * cutoff * d) * np.kaiser(taps, 8.0)
    return h / h.sum()


def noise_truth(L, seed, band=0.9):
    """band-limited complex noise of L samples at H fs, occupying the middle `band` of the spectrum (circular)"""
    rng = np.random.default_rng(seed)
    Z = (rng.standard_normal(L) + 1j * rng.standard_normal(L)) / np.sqrt(2)
    f = np.fft.fftfreq(L)
    Z[np.abs(f) > band / 2] = 0
    return np.fft.ifft(Z) * np.sqrt(L / max(1, np.count_nonzero(Z)))


def hops_from_truth(truth, H, n, d, delays, phases, gains, snr_db, seed, taps=None, cutoff=0.49, fir=True):
    """Hop i: truth (L = H n samples at H fs, taken as periodic) shifted by -c_i bins, low-passed to +-cutoff fs by a linear-phase
    FIR (its delay removed), decimated by H, delayed circularly by delays[i] samples, times gains[i] e^{i phases[i]}, plus complex
    noise at snr_db below the hop's power.  Returns interleaved float32 hops."""
    L = H * n
    x = np.asarray(truth, complex)
    t = np.arange(L)
    rng = np.random.default_rng(seed)
    taps = taps or 256 * H + 1
    h = lowpass(taps, cutoff / H) if fir else None
    k = np.fft.fftfreq(n) * n
    out = []
    for i in range(H):
        ci = (2 * i - (H - 1)) * d // 2
        s = x * np.exp(-2j * np.pi * ci * t / L)
        if fir:
            ext = np.concatenate([s[-(taps // 2):], s, s[: taps // 2]])      # circular
            s = np.convolve(ext, h, mode="valid")
        v = s[::H][:n]
        V = np.fft.fft(v) * np.exp(-2j * np.pi * k * delays[i] / n)
        v = np.fft.ifft(V) * gains[i] * np.exp(1j * phases[i])
        p = np.mean(np.abs(v) ** 2)
        v = v + np.sqrt(p * 10 ** (-snr_db / 10) / 2) * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        out.append(np.ascontiguousarray(v.astype(np.complex64)).view(np.float32))
    return out


def truth_in_band(truth, H, n, d):
    """the truth restricted to the stitched band (the bins some hop covers)"""
    L = H * n
    T = np.fft.fft(np.asarray(truth, complex))
    span = (n + (H - 1) * d) // 2
    kap = np.fft.fftfreq(L) * L
    T[(kap < -span) | (kap >= span)] = 0
    return np.fft.ifft(T)


def expected_join(b, n, d, H, delays, phases, gains):
    """(tau^, g) that undo hop b's delay, LO phase and gain against the truth (hop r is taken to carry none)"""
    c = [(2 * i - (H - 1)) * d // 2 for i in range(H)]
    a = b - 1 if b > (H - 1) // 2 else b + 1
    k0 = c[max(a, b)] - n // 2
    g = np.exp(-1j * phases[b]) * np.exp(2j * np.pi * (k0 - c[b]) * delays[b] / n) / gains[b]
    return -delays[b], complex(g)


def nmse_db(y, ref):
    return float(10 * np.log10(np.sum(np.abs(y - ref) ** 2) / np.sum(np.abs(ref) ** 2)))
