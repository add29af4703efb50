"""The spectral coherence at the line rate (tsdrgpu_coherence_*, tsdrgpu_pipeline_set_coherence, TSDR_COHERENCE): the float64 model
against the literal definition, the spelling, N, K and window, the estimator's properties on a synthetic scene, and on the GPU the
object and the pipeline against the model."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import _native as N
from tempestsdr_b200 import synth
from tests.coherence_model import CoherenceModel, literal, n_for, window_plus64
from tests.spectrum_model import segments_per_report

BENCH = {"cfg1": (8_000_000, 525, 60.0, 4096), "cfg2": (25_000_000, 1125, 60.0, 8192), "cfg5": (50_000_000, 1125, 60.0, 16384)}


# ============================================================================================================== CPU
def _noise(rng, pairs, scale=0.3):
    return (rng.standard_normal(2 * pairs) * scale).astype(np.float32)


@pytest.mark.parametrize("n,fs,alpha,rate", [(256, 25_600, 1700.0, 100), (256, 12_800, 900.0, 100), (256, 25_600, 2345.678, 50),
                                             (1024, 102_400, 1700.0, 100), (1024, 51_200, 1000.5, 100)])
def test_model_equals_the_literal_definition(n, fs, alpha, rate):
    """Ragged runs, a discontinuity part way (which drops the report in progress) and K down to 1."""
    assert n_for(fs, alpha) == n
    K = segments_per_report(n, rate, fs)
    H = n // 2
    rng = np.random.default_rng(n + fs)
    # two reports, then (K > 1) one segment of a third that the drop discards with the open segment; then two more reports
    a_pairs = 2 * K * H + n - 1 + (H if K > 1 else 0)
    b_pairs = 2 * K * H + n - 1
    x = _noise(rng, a_pairs + b_pairs)
    m = CoherenceModel(f"line:{rate}", fs, alpha)
    got, pos = [], 0
    cuts = [1, 3, H - 1, n + 2, 5 * H]
    k = 0
    while pos < a_pairs + b_pairs:
        c = min(cuts[k % len(cuts)], (a_pairs if pos < a_pairs else a_pairs + b_pairs) - pos)
        got.extend(m.run(x[2 * pos:2 * (pos + c)], discontinuity=(pos == a_pairs)))
        pos += c
        k += 1
    xc = x.view(np.complex64).astype(np.complex128)
    starts = [r * K * H + np.arange(K) * H for r in range(2)] + [a_pairs + r * K * H + np.arange(K) * H for r in range(2)]
    assert len(got) == 4
    for r, s0 in enumerate(starts):
        want = literal(xc, n, alpha, fs, K, list(s0))
        for g, w in zip(got[r], want):
            assert np.allclose(g, w, rtol=1e-9, atol=1e-9 * np.max(np.abs(w))), r


@pytest.mark.parametrize("n,alpha,fs", [(256, 2e6, 25_000_000), (4096, 31_500.0, 8_000_000), (16384, 67_500.0, 50_000_000),
                                        (65536, 8333.0, 25_000_000)])
def test_window_matches_the_model(n, alpha, fs):
    from tempestsdr_b200 import api
    got = api.Coherence.window(n, alpha, fs)
    want = window_plus64(n, alpha, fs)
    assert np.max(np.abs(got - want)) <= 1e-15


def test_n_and_k_at_the_bench_shapes():
    from tempestsdr_b200 import api
    for name, (fs, h, fv, n) in BENCH.items():
        assert api.Coherence.n_for(fs, h * fv) == n == n_for(fs, h * fv), name
        for rate in (1, 10, 100):
            w = N.WelchSpec(n, rate)
            assert N.lib().tsdrgpu_spectrum_k(C.byref(w), fs) == segments_per_report(n, rate, fs)
    assert api.Coherence.n_for(1_000_000, 1e6 / 16) == 256                   # exactly 16 bins: the floor
    assert api.Coherence.n_for(1_000_000, 1e6 / 20) == 512
    assert api.Coherence.n_for(25_000_000, 25e6 * 16 / 65536) == 65536
    assert api.Coherence.n_for(25_000_000, 25e6 * 16 / 65536 * 0.999) == 0   # unresolvable
    assert api.Coherence.n_for(50_000_000, 10_000.0) == 0
    assert api.Coherence.n_for(0, 31_500.0) == 0 and api.Coherence.n_for(8_000_000, 0.0) == 0
    assert api.Coherence.n_for(8_000_000, -1.0) == 0 and api.Coherence.n_for(8_000_000, float("nan")) == 0


GOOD = {"off": 0, "line": 1, "line:1": 1, "line:7": 7, "line:100": 100, "line:007": 7}
BAD = ["", "on", "line:", "line:0", "line:101", "line:-1", "line:+1", "line: 1", "line:1 ", "line:1:2", "line:1e1", "line,1",
       "line:1234567", "lines", "Line", "frame:1", "off:1"]


def test_the_spelling_is_parsed_and_refused_as_documented():
    for text, want in GOOD.items():
        assert N.coherence_spec(text).rate == want, text
    for text in BAD:
        out = N.CoherenceSpec(678)
        assert N.lib().tsdrgpu_coherence_parse(text.encode(), C.byref(out)) == -3, text
        assert out.rate == 678, text                                             # untouched
        with pytest.raises(ValueError):
            N.coherence_spec(text)


def test_bogus_coherence_setting_is_refused_by_the_host_library(tmp_path, monkeypatch):
    """TSDR_COHERENCE that does not parse: tsdr_readasync fails with TSDR_INVALID_PARAMETER_VALUE before touching the GPU."""
    from tests.test_host_library import FRAME_CB, MINE, PLOT_CB, VALUE_CB, bind
    raw = tmp_path / "iq.int8"
    np.zeros(1 << 16, np.int8).tofile(raw)
    plugin = os.path.join(os.path.dirname(MINE), "TSDRPlugin_RawFileGPU.so")
    lib = bind(MINE)
    t = C.c_void_p()
    nv, npl = VALUE_CB(lambda *a: None), PLOT_CB(lambda *a: None)
    lib.tsdr_init(C.byref(t), nv, npl, None)
    lib.tsdr_setresolution(t, 525, 60.0)
    assert lib.tsdr_loadplugin(t, plugin.encode(), f'"{raw}" 2000000 int8 nopace'.encode()) == 0
    monkeypatch.setenv("TSDR_COHERENCE", "line:0")
    assert lib.tsdr_readasync(t, FRAME_CB(lambda *a: None), None) == 9          # TSDR_INVALID_PARAMETER_VALUE
    assert b"TSDR_COHERENCE" in lib.tsdr_getlasterrortext(t)
    assert lib.tsdr_isrunning(t) == 0
    lib.tsdr_free(C.byref(t))


# ---------------------------------------------------------------------------------------------- the estimator on a scene
SC_FS, SC_H, SC_FV = 8_000_000, 525, 60.0
SC_ALPHA = SC_H * SC_FV


def scene(seconds, seed=5):
    """video_like_iq at 8 MS/s in 525-line / 60 Hz geometry band-limited to +-1 MHz, a CW tone about 10 dB above the video at
    2.5 MHz, a stationary noise band of twice the video's power over -3 .. -2 MHz and white noise 13 dB below the video."""
    fs = SC_FS
    pairs = int(seconds * fs)
    w = int(2 * (fs / (SC_FV * SC_H)))
    v = synth.video_like_iq(pairs, fs, w, SC_H, SC_FV, seed=seed, snr_db=200.0).view(np.complex64).astype(np.complex128)
    f = np.fft.fftfreq(pairs, 1.0 / fs)
    V = np.fft.fft(v)
    V[np.abs(f) > 1e6] = 0
    v = np.fft.ifft(V)
    pv = np.mean(np.abs(v) ** 2)
    rng = np.random.default_rng(seed)
    t = np.arange(pairs)
    tone = np.sqrt(10 * pv) * np.exp(2j * np.pi * 2.5e6 * t / fs)
    nb = np.fft.fft(rng.standard_normal(pairs) + 1j * rng.standard_normal(pairs))
    nb[(f < -3e6) | (f > -2e6)] = 0
    nb = np.fft.ifft(nb)
    nb *= np.sqrt(2 * pv / np.mean(np.abs(nb) ** 2))
    wn = (rng.standard_normal(pairs) + 1j * rng.standard_normal(pairs)) * np.sqrt(pv * 10 ** (-1.3) / 2)
    return (v + tone + nb + wn).astype(np.complex64).view(np.float32)


def _report(x, rate, alpha=SC_ALPHA, fs=SC_FS):
    m = CoherenceModel(f"line:{rate}", fs, alpha)
    reps = m.run(x)
    assert reps
    return reps[0][0]


def _bands(n, fs=SC_FS):
    f = (np.arange(n) - n // 2) * fs / n
    video = (np.abs(f) < 0.9e6) & (np.abs(f) > 0.05e6)
    noise = (f > -2.9e6) & (f < -2.1e6)
    tone = np.abs(f - 2.5e6) <= 4 * fs / n
    quiet = (np.abs(f) > 1.1e6) & ~noise & ~tone & (np.abs(f) < 3.8e6) & ~((f > -3.1e6) & (f < -1.9e6))
    return video, noise, tone, quiet


@pytest.fixture(scope="module")
def scene_1s():
    return scene(1.01)


def test_video_stands_above_the_floor_and_interference_does_not(scene_1s):
    x = scene_1s[:2 * 810_000]                                                 # 0.1 s: K = 390 at rate 10
    g = _report(x, 10)
    n = n_for(SC_FS, SC_ALPHA)
    video, noise, tone, quiet = _bands(n)
    med = {k: float(np.median(g[b])) for k, b in (("video", video), ("noise", noise), ("tone", tone), ("quiet", quiet))}
    floor = med["quiet"]
    assert 0.02 <= floor <= 0.07, med
    assert med["video"] >= 1.8 * floor, med
    assert med["noise"] <= 1.3 * floor and med["tone"] <= 1.5 * floor, med


def test_the_floor_falls_as_one_over_sqrt_k(scene_1s):
    n = n_for(SC_FS, SC_ALPHA)
    quiet = _bands(n)[3]
    f10 = np.median(_report(scene_1s, 10)[quiet])
    f1 = np.median(_report(scene_1s, 1)[quiet])
    k10, k1 = segments_per_report(n, 10, SC_FS), segments_per_report(n, 1, SC_FS)
    ratio = f10 / f1
    assert abs(ratio / np.sqrt(k1 / k10) - 1.0) <= 0.2, (f10, f1, ratio)


def test_the_wrong_alpha_gives_the_floor_and_a_pll_sized_error_does_not(scene_1s):
    x = scene_1s[:2 * 810_000]
    n = n_for(SC_FS, SC_ALPHA)
    video, _, _, quiet = _bands(n)
    g0 = _report(x, 10)
    wrong = _report(x, 10, alpha=1.37 * SC_ALPHA)
    assert n_for(SC_FS, 1.37 * SC_ALPHA) == n
    assert np.median(wrong[video]) <= 1.3 * np.median(g0[quiet])
    for s in (1 + 1e-5, 1 - 1e-5):
        g = _report(x, 10, alpha=s * SC_ALPHA)
        assert abs(np.median(g[video]) - np.median(g0[video])) < 0.01


def test_a_frequency_offset_moves_gamma_with_it(scene_1s):
    n = n_for(SC_FS, SC_ALPHA)
    x = scene_1s[:2 * 450_000].view(np.complex64).astype(np.complex128)
    d = 37
    delta = d * SC_FS / n
    t = np.arange(x.size)
    y = (x * np.exp(2j * np.pi * delta * t / SC_FS)).astype(np.complex64).view(np.float32)
    g0 = _report(x.astype(np.complex64).view(np.float32), 20)
    g1 = _report(y, 20)
    assert np.max(np.abs(g1[d:] - g0[:-d])) <= 1e-6


def test_a_zero_input_gives_zero():
    g = _report(np.zeros(2 * 200_000, np.float32), 100)
    assert np.all(g == 0)


# ============================================================================================================== GPU
FS = 25_000_000
EPS = 2.0 ** -24


def _ctx():
    from tempestsdr_b200 import api
    return api.Context(0)


def _cuts(rng, total, n):
    cuts, done = [], 0
    while done < total:
        r = rng.random()
        c = 1 if r < 0.15 else (int(rng.integers(2, n // 2)) if r < 0.45 else int(rng.integers(n // 2, 6 * n)))
        cuts.append(min(c, total - done))
        done += cuts[-1]
    return cuts


def _data(rng, pairs, alpha, fs):
    """Noise, a tone and a line-rate cyclostationary component (a carrier keyed at alpha), so gamma has a range of values."""
    t = np.arange(pairs)
    x = (rng.standard_normal(pairs) + 1j * rng.standard_normal(pairs)) * 0.05
    x += 0.5 * np.exp(2j * np.pi * (0.0371 * t + 0.2))
    x += 0.3 * (np.cos(2 * np.pi * alpha * t / fs) > 0.6) * np.exp(2j * np.pi * 0.11 * t)
    return x.astype(np.complex64).view(np.float32)


def gpu_runs(co, x, events, offset_floats=0):
    """events: ('run', pairs, discontinuity) | ('reset',) | ('set', spec, fs, alpha).  The reports of every run."""
    import torch
    buf = torch.zeros(x.size + offset_floats + 8, dtype=torch.float32, device="cuda")
    buf[offset_floats:offset_floats + x.size] = torch.from_numpy(x)
    dx = buf[offset_floats:offset_floats + x.size]
    out, pos = [], 0
    for ev in events:
        if ev[0] == "reset":
            co.reset()
        elif ev[0] == "set":
            co.set(*ev[1:])
        else:
            r = co.run(dx[2 * pos:2 * (pos + ev[1])], discontinuity=ev[2])
            out.extend(list(r.cpu().numpy()))
            pos += ev[1]
    torch.cuda.synchronize()
    return out


def model_runs(spec, fs, alpha, x, events):
    m = CoherenceModel(spec, fs, alpha)
    out, pos = [], 0
    for ev in events:
        if ev[0] == "reset":
            m.reset()
        elif ev[0] == "set":
            m.set(*ev[1:])
        else:
            out.extend(m.run(x[2 * pos:2 * (pos + ev[1])], ev[2]))
            pos += ev[1]
    return out


# The bound.  Each float32 transform of a segment is off by at most ETA = 2 log2(N) units of 2^-24 of the segment's largest |U| per
# bin (the FFT tests' unit: rounding relative to the peak), and the windowed product adds one more unit.  At a bin where both summed
# powers are at least FRAC of the largest, U+- are each off by at most rel = ETA sqrt(Pmax / P+-) relative, so
# |C| moves by at most 2 rel sqrt(P+ P-) and sqrt(P+ P-) by rel sqrt(P+ P-): |d gamma| <= 3 rel (gamma <= 1), taken with the larger rel.
FRAC = 1e-8


def _gamma_bound(n, want):
    _, _, Pp, Pm = want
    pmax = max(Pp.max(), Pm.max())
    eta = (2 * np.log2(n) + 1) * EPS
    ok = (Pp >= FRAC * pmax) & (Pm >= FRAC * pmax)
    rel = eta * np.sqrt(pmax / np.minimum(Pp, Pm))
    return ok, 3 * rel


def _compare(n, got, want, min_reports=2):
    assert len(got) == len(want) >= min_reports
    worst = 0.0
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.shape == (n,)
        ok, bound = _gamma_bound(n, w)
        assert ok.sum() >= n // 4
        err = np.abs(g - w[0])
        assert np.all(err[ok] <= bound[ok]), (k, float(np.max(err[ok] / bound[ok])))
        assert np.all((g >= 0) & (g <= 1 + 1e-6))
        worst = max(worst, float(np.max(err[ok] / bound[ok])))
    return worst


CASES = {256: (2e6, 2.2e6, 24_000_000), 4096: (120_000.0, 130_000.0, 24_000_000), 65536: (8333.0, 8400.0, 24_000_000)}


@pytest.mark.gpu
@pytest.mark.parametrize("n", [256, 4096, 65536])
@pytest.mark.parametrize("offset_floats", [0, 2])
def test_object_matches_the_model(n, offset_floats):
    """Random cuts down to 1 pair, drops, a reset, a set with a new alpha (from the next report on) and a set with a new fs
    (discards), at both 8-byte phases of a 16-byte line."""
    alpha, alpha2, fs2 = CASES[n]
    assert n_for(FS, alpha) == n_for(FS, alpha2) == n_for(fs2, alpha2) == n
    rng = np.random.default_rng(n + offset_floats)
    spec = "line:100"
    K = segments_per_report(n, 100, FS)
    total = 9 * K * n // 2 + 3 * n + 17
    x = _data(rng, total, alpha, FS)
    cuts = _cuts(rng, total, n)
    events = []
    for k, c in enumerate(cuts):
        if k == len(cuts) // 4:
            events.append(("reset",))
        if k == len(cuts) // 3:
            events.append(("set", spec, FS, alpha2))
        if k == 2 * len(cuts) // 3:
            events.append(("set", spec, fs2, alpha2))
        events.append(("run", c, k in (5, len(cuts) // 2)))
    co = _ctx().coherence()
    co.set(spec, FS, alpha)
    got = gpu_runs(co, x, events, offset_floats)
    want = model_runs(spec, FS, alpha, x, events)
    worst = _compare(n, got, want, min_reports=3)
    print(f"N={n} offset={offset_floats}: {len(got)} reports, worst error {worst:.3f} of the bound")


@pytest.mark.gpu
def test_the_same_blocks_give_the_same_bits():
    rng = np.random.default_rng(7)
    for n, alpha in ((1024, 400_000.0), (16384, 25_000.0)):
        assert n_for(FS, alpha) == n
        total = 1_200_000
        x = _data(rng, total, alpha, FS)
        events = [("run", c, k == 9) for k, c in enumerate(_cuts(rng, total, n))]
        ctx = _ctx()
        runs = []
        for _ in range(2):
            co = ctx.coherence()
            co.set("line:100", FS, alpha)
            runs.append(gpu_runs(co, x, events))
        assert len(runs[0]) == len(runs[1]) >= 2
        for a, b in zip(*runs):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


@pytest.mark.gpu
def test_refusals_leave_the_state_alone():
    import torch
    ctx = _ctx()
    lib = ctx._lib
    co = ctx.coherence()
    n = C.c_uint32(0)
    buf = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")
    assert lib.tsdrgpu_coherence_run(co._h, ctx.stream, buf.data_ptr(), 100, 0, None, 0, C.byref(n)) == -3     # no spec yet
    s = N.coherence_spec("line:100")
    assert lib.tsdrgpu_coherence_set(co._h, C.byref(s), 0, 1000.0) == -3
    assert lib.tsdrgpu_coherence_set(co._h, C.byref(s), 50_000_000, 10_000.0) == -3                            # unresolvable
    s.rate = 101
    assert lib.tsdrgpu_coherence_set(co._h, C.byref(s), 25_600, 1700.0) == -3
    co.set("line:100", 25_600, 1700.0)                                          # N = 256, K = 2: a report every 256 pairs
    assert lib.tsdrgpu_coherence_run(co._h, ctx.stream, buf.data_ptr() + 4, 100, 0, None, 0, C.byref(n)) == -3   # 4-byte aligned
    assert lib.tsdrgpu_coherence_run(co._h, ctx.stream, buf.data_ptr(), 1000, 0, None, 0, C.byref(n)) == -5      # no room
    assert lib.tsdrgpu_coherence_plan(co._h, 1000, 0, C.byref(n)) == 0 and n.value == 3
    assert lib.tsdrgpu_coherence_plan(co._h, 1000, 1, C.byref(n)) == 0 and n.value == 3
    torch.cuda.synchronize()


# -------------------------------------------------------------------------------------------------- pipeline
COH = "line:10"


def run_pipeline(fs, h, fv, calls, coherence="off", spectrum="off", batch=1, params=None, channel="off", argb=False):
    """calls: list of dicts {iq (float32) | raw (int8), dropped, sync, superres, resolution}.  Returns frames, plots without spectra
    and coherence, values, coherence reports, the stats, spectrum reports and the line rate each call started with."""
    from tempestsdr_b200 import pipeline
    frames, plots, values, cohs, spectra, alphas = [], [], [], [], [], []

    def on_plot(pid, off, v, sr):
        (cohs if pid == N.PLOT_ID_COHERENCE else spectra if pid == N.PLOT_ID_SPECTRUM else plots).append((pid, off, v.copy(), sr))

    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=batch, batch_blocks=10 * batch, block_when_busy=True,
                          params=params, channel=channel, spectrum=spectrum, coherence=coherence,
                          on_frame=lambda f, ww, hh: frames.append((f.copy(), ww)), on_plot=on_plot,
                          on_value=lambda vid, a, b: values.append((vid, a, b)))
    p.set_reports(snr=True, detect_mode=True)
    if argb:
        p.set_output_argb(True)
    for c in calls:
        if "superres" in c:
            p.set_param("superresolution", c["superres"])
        if "resolution" in c:
            p.set_resolution(*c["resolution"])
        _, gh, gfv = p.geometry()
        alphas.append(gh * gfv)
        if "raw" in c:
            p.process_raw(c["raw"], c.get("dropped", 0))
        else:
            p.process(c["iq"], c.get("dropped", 0))
        if c.get("sync"):
            p.sync(c["sync"])
    p.flush()
    st = p.stats()
    p.close()
    return frames, plots, values, cohs, st, spectra, alphas


def model_reports(fs, calls, spec, alphas):
    """What the pipeline's coherence sees: every block's converted floats at the line rate of its call, a new report after a drop,
    a new N or superbandwidth mode."""
    m, out, fresh, on = None, [], False, 0
    for c, alpha in zip(calls, alphas):
        on = c.get("superres", on)
        if on:
            fresh = True
            continue
        if m is None:
            m = CoherenceModel(spec, fs, alpha)
        else:
            m.set(spec, fs, alpha)
        if fresh:
            m.reset()
            fresh = False
        iq = c["iq"] if "iq" in c else c["raw"].astype(np.float32) * np.float32(0.0078125)
        out.extend(m.run(iq, c.get("dropped", 0) != 0))
    return out


def _check_reports(res, fs, calls, spec):
    cohs, st, alphas = res[3], res[4], res[6]
    want = model_reports(fs, calls, spec, alphas)
    assert len(cohs) >= 1 and len(cohs) + st.coherence_skipped == len(want) and st.coherence_delivered == len(cohs)
    k = 0
    for off, v, sr in [(s[1], s[2], s[3]) for s in cohs]:
        n = v.size
        assert off == -n // 2 and sr == fs
        while True:
            assert k < len(want), "a delivered report matches none of the model's"
            w = want[k]
            k += 1
            if w[0].size == n:
                ok, bound = _gamma_bound(n, w)
                if np.all(np.abs(v - w[0])[ok] <= bound[ok]):
                    break


def _case(case):
    from tests.test_spectrum import SMALL, _blocks, _pipeline_case
    if case == "both":
        fs, h, fv, calls, kw = _pipeline_case("small_plots")
        kw["spectrum"] = "welch:1024:10"
    elif case == "geometry":
        fs, h, fv = SMALL
        calls = [{"iq": b} for b in _blocks(*SMALL, 30, 65536, seed=48)]
        calls[12]["resolution"] = (250, 60.0)                                   # alpha doubles: N 8192 -> 4096
        calls[22]["resolution"] = (125, 60.0)
        kw = {"params": {"autoshift": 1, "lowpass_before_sync": 1}}
    else:
        fs, h, fv, calls, kw = _pipeline_case(case)
    return fs, h, fv, calls, kw


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["small_plots", "cfg1", "pll_drops_sync", "int8", "channel", "both", "superres", "argb", "geometry"])
def test_pipeline_coherence_changes_nothing_else_and_matches_the_model(case):
    """With the coherence on and off the same blocks give bit-identical frames, autocorrelation plots, spectrum reports and value
    callbacks; the coherence reports are the model's reports of the unfiltered stream at the line rate of each call."""
    from tests.test_spectrum import _same_outputs
    fs, h, fv, calls, kw = _case(case)
    on = run_pipeline(fs, h, fv, calls, coherence=COH, **kw)
    off = run_pipeline(fs, h, fv, calls, **kw)
    _same_outputs(on, off)
    assert len(on[5]) == len(off[5])
    for a, b in zip(on[5], off[5]):
        assert a[1] == b[1] and a[3] == b[3] and np.array_equal(a[2].view(np.uint64), b[2].view(np.uint64))
    assert off[3] == [] and off[4].coherence_delivered == 0
    _check_reports(on, fs, calls, COH)
    if case == "geometry":
        assert {v[2].size for v in on[3]} == {4096, 8192}


@pytest.mark.gpu
def test_host_library_delivers_coherence_plots(tmp_path, monkeypatch):
    """TSDR_COHERENCE=line:10: tsdr_readasync driven by a RawFile plugin hands coherence plots to plot_cb beside ids 0 and 1."""
    from tests.test_host_library import FRAME_CB, MINE, PLOT_CB, VALUE_CB, bind
    fs, h, fv = 2_000_000, 125, 60.0
    w = int(2 * (fs / (fv * h)))
    iq = synth.video_like_iq(6 * 256 * 1024, fs, w, h, fv, seed=31)
    raw = tmp_path / "iq.raw"
    iq.tofile(raw)
    if orc.have_ref():
        plugin, args = orc.REF_RAWFILE_SO, f'"{raw}" {fs} float'
    else:
        plugin, args = os.path.join(os.path.dirname(MINE), "TSDRPlugin_RawFileGPU.so"), f'"{raw}" {fs} float'
    monkeypatch.setenv("TSDR_NO_DROP", "1")
    monkeypatch.setenv("TSDR_COHERENCE", "line:10")
    plots = []
    lib = bind(MINE)
    t = C.c_void_p()
    nv = VALUE_CB(lambda *a: None)
    npl = PLOT_CB(lambda pid, off, vals, size, sr, c: plots.append((pid, off, size, sr)))
    fcb = FRAME_CB(lambda *a: None)
    lib.tsdr_init(C.byref(t), nv, npl, None)
    lib.tsdr_setresolution(t, h, fv); lib.tsdr_motionblur(t, 0.0); lib.tsdr_setgain(t, 0.5)
    assert lib.tsdr_loadplugin(t, plugin.encode(), args.encode()) == 0
    rc = []
    th = threading.Thread(target=lambda: rc.append(lib.tsdr_readasync(t, fcb, None)))
    th.start()
    deadline = time.time() + 60
    while not ({0, 1, 101} <= {p[0] for p in plots}) and time.time() < deadline:
        time.sleep(0.05)
    assert lib.tsdr_stop(t) == 0
    th.join(timeout=30)
    assert rc == [0]
    cohs = [p for p in plots if p[0] == 101]
    assert cohs and {0, 1} <= {p[0] for p in plots}
    assert all(p[1:] == (-4096, 8192, fs) for p in cohs)
    lib.tsdr_free(C.byref(t))
