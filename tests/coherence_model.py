"""numpy float64 model of the spectral coherence at the line rate of include/tsdrgpu.h (tsdrgpu_coherence_*,
tsdrgpu_pipeline_set_coherence).

It takes the same blocks, discontinuities, resets and sets as the object and keeps the same state: the open segment (fewer than N
pairs), the completed segments of the report in progress and the alpha that report was started with.  The complex window is rounded
to float32 and the input is float32, as on the device; everything else is float64.  `literal` is the definition written as a per-bin
loop of direct DFTs, the check on the vectorised model."""
import re

import numpy as np

from tests.spectrum_model import segments_per_report, window64


def parse(spec):
    """"line[:<rate>]" -> rate; the library's parser is the one that refuses bad spellings."""
    m = re.fullmatch(r"line(?::(\d+))?", spec)
    return int(m.group(1) or 1)


def n_for(fs, alpha):
    """N of the definition; 0 when unresolvable."""
    if fs <= 0 or not alpha > 0:
        return 0
    need, n = 16.0 * fs / alpha, 256
    while n < need:
        if n >= 65536:
            return 0
        n *= 2
    return n


def window_plus64(n, alpha, fs):
    """w+[n] = w[n] e^{-i pi alpha n / fs} in double, the angle reduced as tsdrgpu_coherence_window reduces it."""
    i = np.arange(n, dtype=np.float64)
    a = -np.pi * np.fmod(alpha * i / fs, 2.0)
    w = window64(n)
    return w * np.cos(a) + 1j * (w * np.sin(a))


def window_plus32(n, alpha, fs):
    w = window_plus64(n, alpha, fs)
    return w.real.astype(np.float32).astype(np.float64) + 1j * w.imag.astype(np.float32).astype(np.float64)


def seg_phase(alpha, s, fs):
    """e^{-2 pi i alpha s / fs}, alpha s / fs in double reduced mod 1 first."""
    t = (alpha * np.asarray(s, np.float64)) / fs
    t = t - np.floor(t)
    return np.exp(-2j * np.pi * t)


def gamma(C, Pp, Pm):
    den = Pp * Pm
    out = np.zeros(C.shape)
    ok = den > 0
    out[ok] = np.abs(C[ok]) / np.sqrt(den[ok])
    return out


class CoherenceModel:
    def __init__(self, spec, fs, alpha):
        self.key = None
        self.set(spec, fs, alpha)

    def set(self, spec, fs, alpha):
        rate, n = parse(spec), n_for(fs, alpha)
        assert n, "unresolvable"
        self.alpha = alpha
        if (rate, fs, n) == self.key:
            return
        self.key, self.n, self.fs, self.K = (rate, fs, n), n, fs, segments_per_report(n, rate, fs)
        self.open = np.zeros(0, np.complex128)
        self.reset()

    def reset(self):
        self.open = np.zeros(0, np.complex128)
        self._new_report()

    def _new_report(self):
        n = self.n
        self.C, self.Pp, self.Pm = np.zeros(n, np.complex128), np.zeros(n), np.zeros(n)
        self.done = 0

    def run(self, iq, discontinuity=False):
        """iq: interleaved float32 I,Q.  Returns the reports this run completes, each (gamma, C, P+, P-) in fftshift order."""
        if discontinuity:
            self.reset()
        x = np.asarray(iq, np.float32).view(np.complex64).astype(np.complex128)
        v = np.concatenate([self.open, x])
        n, H = self.n, self.n // 2
        count = (v.size - n) // H + 1 if v.size >= n else 0
        reports = []
        q = 0
        while q < count:
            if self.done == 0:                                   # alpha is read at the first segment of a report
                self.alpha_rep = self.alpha
                self.wp = window_plus32(n, self.alpha, self.fs)
            take = min(count - q, self.K - self.done, max(1, (1 << 21) // n))
            segs = np.lib.stride_tricks.sliding_window_view(v, n)[q * H:(q + take - 1) * H + 1:H]
            Up = np.fft.fft(segs * self.wp, axis=1)
            Um = np.fft.fft(segs * np.conj(self.wp), axis=1)
            e = seg_phase(self.alpha_rep, (self.done + np.arange(take)) * H, self.fs)
            self.C += np.sum(Up * np.conj(Um) * e[:, None], axis=0)
            self.Pp += np.sum(Up.real ** 2 + Up.imag ** 2, axis=0)
            self.Pm += np.sum(Um.real ** 2 + Um.imag ** 2, axis=0)
            self.done += take
            q += take
            if self.done == self.K:
                sh = np.fft.fftshift
                reports.append((sh(gamma(self.C, self.Pp, self.Pm)), sh(self.C), sh(self.Pp), sh(self.Pm)))
                self._new_report()
        self.open = v[count * H:].copy()
        return reports


def literal(x, n, alpha, fs, K, starts):
    """The definition over one report, bin by bin: segments at `starts` (pairs into x, complex128), direct DFTs."""
    wp = window_plus32(n, alpha, fs)
    wm = np.conj(wp)
    idx = np.arange(n)
    C, Pp, Pm = np.zeros(n, complex), np.zeros(n), np.zeros(n)
    assert len(starts) == K
    for k in range(n):
        ek = np.exp(-2j * np.pi * k * idx / n)
        for j, s0 in enumerate(starts):
            seg = x[s0:s0 + n]
            up = np.sum(wp * seg * ek)
            um = np.sum(wm * seg * ek)
            t = (alpha * float(j * (n // 2))) / fs
            t -= np.floor(t)
            C[k] += up * np.conj(um) * np.exp(-2j * np.pi * t)
            Pp[k] += abs(up) ** 2
            Pm[k] += abs(um) ** 2
    sh = np.fft.fftshift
    return sh(gamma(C, Pp, Pm)), sh(C), sh(Pp), sh(Pm)
