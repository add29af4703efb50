"""Percentile auto-gain (clip mode, include/tsdrgpu.h): the reference of tests/autogain_clip_model.py pinned to the oracle, then
the GPU selection, frame stage, pipeline and host library against it."""
import ctypes as C
import math
import os
import re
import threading
import time

import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import synth
from tests.autogain_clip_model import (KINDS, ClipPostProcessor, adversarial, clip_levels, levels_from_sorted, minmax_levels,
                                       valid_sorted_keys)
from tests.autogain_clip_model import synth_stream as _synth_stream

SMALL = (2_000_000, 125, 60.0)                              # fs, height, refresh rate of the small geometry


# ============================================================================================================== CPU
def test_model_selection_matches_an_independent_order_statistic():
    """The key order and k arithmetic against np.partition on float64 order plus explicit tie / sign / NaN handling."""
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 4, 5, 17, 1000, 4096):
        for kind in range(KINDS):
            f = adversarial(n, kind, rng)
            for ppm in (0, 1, 3500, 10_000, 250_000):
                lo, hi, nv = clip_levels(f, ppm)
                v = f[~((f > 250.0) | (f < -250.0)) & ~np.isnan(f)]
                assert nv == v.size
                if nv == 0:
                    assert lo.tobytes() == hi.tobytes() == np.float32(f[0]).tobytes()
                    continue
                # sort by (value, sign bit first for zeros): total order among the non-NaN floats
                order = np.lexsort((~np.signbit(v), v.astype(np.float64)))
                s = v[order]
                k = nv * ppm // 1_000_000
                assert lo.tobytes() == s[k].tobytes() and hi.tobytes() == s[nv - 1 - k].tobytes(), (n, kind, ppm)


def test_model_ppm0_is_min_max_when_pixel_0_is_valid():
    rng = np.random.default_rng(6)
    for n in (1, 2, 3, 1000):
        for kind in (1, 2, 4, 6):
            f = adversarial(n, kind, rng)
            lo, hi, _ = clip_levels(f, 0)
            assert (lo, hi) == minmax_levels(f)


FLAGS = [(a, l, g) for a in (0, 1) for l in (0, 1) for g in (0, 1)]       # autoshift, lowpass before sync, auto-gain after


def _assert_same_as_oracle(gf, gr, wf, wr, what):
    assert np.array_equal(gf.view(np.uint32), wf.view(np.uint32)), what
    assert gr["x"] == wr.x.astuple() and gr["y"] == wr.y.astuple(), f"sync state {what}"
    assert gr["avg_speed"] == wr.avg_speed and gr["pll_state"] == wr.pll_state, f"pll averages {what}"
    assert (gr["lastmax"], gr["lastmin"]) == (np.float32(wr.lastmax), np.float32(wr.lastmin)), f"auto-gain state {what}"
    assert gr["report"] == wr.autogain_callback_fired, f"auto-gain report {what}"
    assert (gr["pll_fired"], gr["refreshrate"], gr["width"]) == (wr.pll_callback_fired, wr.refreshrate_after, wr.width_after), f"pll {what}"
    if np.isfinite(wr.snr):
        assert abs(float(gr["snr"]) - wr.snr) <= 1e-6 * abs(wr.snr), f"snr {what}"     # float64 sums in another order
    else:
        assert not np.isfinite(gr["snr"]), f"snr {what}"


def _oracle_sequence(O, fs, h, fv, lpbs):
    """(frame, w, h, motion blur, lowpass_before_sync) for 26 drifting frames: motion blur on and off, a smaller geometry
    in the middle (screen kept, not zeroed) and back (regrown and zeroed), and the stage order flipped for the last six."""
    w, _, _ = O.geometry(fs, h, fv)
    seq = []
    for k, f in enumerate(_synth_stream(w, h, 10, 300)):
        seq.append((f, w, h, 0.3 if k % 3 else 0.0, lpbs))
    for k, f in enumerate(_synth_stream(w - 8, h - 5, 6, 400)):
        seq.append((f, w - 8, h - 5, 0.2, lpbs))
    for k, f in enumerate(_synth_stream(w, h, 10, 500)):
        seq.append((f, w, h, 0.0 if k % 2 else 0.4, lpbs if k < 4 else 1 - lpbs))
    return seq


@pytest.mark.parametrize("superres", [0, 1])
@pytest.mark.parametrize("pll", [0, 1])
@pytest.mark.parametrize("autoshift,lpbs,aap", FLAGS)
def test_restatement_in_min_max_mode_is_the_oracle(autoshift, lpbs, aap, pll, superres):
    """The restatement with min/max levels equals orc_pp_run frame by frame on every branch it has: both stage orders and a
    switch between them, AUTOSHIFT or the green lines (drawn in place or on a copy, suppressed in super-resolution), motion
    blur on and off, a geometry change and back, the PLL on and off.  Frames bit for bit; sync state, PLL averages, refresh
    rate and width after the PLL, auto-gain state and report exactly; SNR within 1e-6."""
    O = orc.port()
    fs, h, fv = SMALL
    po = O.postprocessor(fs, h, fv, autoshift, pll, superres)
    pr = ClipPostProcessor(O, fs, h, fv, autoshift, pll, superres)
    fired = 0
    for k, (f, w, hh, mb, lp) in enumerate(_oracle_sequence(O, fs, h, fv, lpbs)):
        wf, wr = po.run(f, w, hh, mb, 0.1, lp, aap)
        gf, gr = pr.run(f, w, hh, mb, 0.1, lp, aap)
        _assert_same_as_oracle(gf, gr, wf, wr, f"frame {k}")
        fired += wr.pll_callback_fired
    assert (fired > 0) == bool(pll)


@pytest.mark.parametrize("autoshift,lpbs,aap", FLAGS)
def test_ppm0_clip_is_bit_identical_to_min_max_on_synth_sequences(autoshift, lpbs, aap):
    """Clip at ppm = 0 against orc_pp_run itself on synth sequences, whose pixel 0 is always valid."""
    O = orc.port()
    fs, h, fv = SMALL
    po = O.postprocessor(fs, h, fv, autoshift, 1)
    pr = ClipPostProcessor(O, fs, h, fv, autoshift, 1, ppm=0)
    for k, (f, w, hh, mb, lp) in enumerate(_oracle_sequence(O, fs, h, fv, lpbs)):
        wf, wr = po.run(f, w, hh, mb, 0.1, lp, aap)
        gf, gr = pr.run(f, w, hh, mb, 0.1, lp, aap)
        _assert_same_as_oracle(gf, gr, wf, wr, f"frame {k}")


def _contrast(f, w, h, lo, hi):
    img = f.reshape(h, w)
    act, blank = img[: int(h * 0.95), : int(w * 0.86)], img[int(h * 0.95) + 1:, :]
    return (act.mean() - blank.mean()) / (hi - lo)


@pytest.mark.parametrize("spikes,gain", [(0, 1.35), (20, 3.0)])
def test_clipping_raises_the_contrast_of_noisy_frames(spikes, gain):
    """740x1125, noise sigma = 0.1: clip at 0.35 % at least 1.35x the min/max contrast, 3x with 20 impulsive samples per frame."""
    w, h = 740, 1125
    f = synth.video_like_frame(w, h, seed=1, noise=0.1).astype(np.float32)
    if spikes:
        f[np.random.default_rng(2).integers(0, w * h, spikes)] = 5.0
    lo0, hi0 = minmax_levels(f)
    lo, hi, _ = clip_levels(f, 3500)
    assert _contrast(f, w, h, lo, hi) >= gain * _contrast(f, w, h, lo0, hi0)


@pytest.mark.parametrize("value", ["clip:30", "clip:x", "median", "clip: 1", "clip:1_0", "clip:0x1p2", "clip:1e1"])
def test_bogus_autogain_setting_is_refused_by_the_host_library(tmp_path, monkeypatch, value):
    """TSDR_AUTOGAIN other than "minmax" / "clip:<percent in [0, 25]>": tsdr_readasync fails with TSDR_INVALID_PARAMETER_VALUE
    before touching the GPU, and the error text names the variable."""
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
    monkeypatch.setenv("TSDR_AUTOGAIN", value)
    assert lib.tsdr_readasync(t, FRAME_CB(lambda *a: None), None) == 9          # TSDR_INVALID_PARAMETER_VALUE
    assert b"TSDR_AUTOGAIN" in lib.tsdr_getlasterrortext(t)
    assert lib.tsdr_isrunning(t) == 0
    lib.tsdr_free(C.byref(t))


PERCENTS = ["0", "25", "25.0", "0.35", "1", "0.00005", "0.00015", "0.000049999", "12.345678", "24.99995", "3.14159265358979",
            "25.00001", "30", "1e1", "0x1p2", " 1", "1 ", "1_0", "+1", "-0", "-1", ".5", "5.", "", "x", "1.2.3", "nan", "inf"]


def _model_ppm(percent: str) -> int:
    """tsdrgpu_autogain_ppm restated from tsdrgpu.h: digits with an optional fraction, value in [0, 25] -> floor(percent * 1e4 + 0.5);
    else -1."""
    if not re.fullmatch(r"[0-9]+(\.[0-9]+)?", percent):
        return -1
    v = float(percent)
    return math.floor(v * 1e4 + 0.5) if v <= 25.0 else -1


def test_autogain_spec_parsing():
    """tsdrgpu_autogain_ppm (what the host library's TSDR_AUTOGAIN and Python's auto-gain spelling use) agrees with the model on
    every spelling, including halves of a ppm and 20 000 random decimals; only digits with an optional fraction, at most 25, are
    accepted."""
    import random
    from tempestsdr_b200 import _native as N
    rng = random.Random(1)
    cases = PERCENTS + [f"{rng.randint(0, 25)}.{rng.randint(0, 10 ** rng.randint(1, 9))}" for _ in range(20_000)]
    lib = N.lib()
    for c in cases:
        assert lib.tsdrgpu_autogain_ppm(c.encode()) == _model_ppm(c), c
    assert [_model_ppm(c) for c in PERCENTS[:11]] == [0, 250_000, 250_000, 3500, 10_000, 1, 1, 0, 123_457, 249_999, 31_416]
    assert all(_model_ppm(c) == -1 for c in PERCENTS[11:])
    assert N.autogain_mode("minmax") == (N.AG_MINMAX, 0)
    assert N.autogain_mode("clip:0.35") == (N.AG_CLIP, 3500)
    for bad in ["clip:" + c for c in PERCENTS[11:]] + ["max", "clip"]:
        with pytest.raises(ValueError):
            N.autogain_mode(bad)


# ============================================================================================================== GPU
def _ctx():
    from tempestsdr_b200 import api
    return api.Context(0)


def _lib():
    from tempestsdr_b200 import _native
    return _native.lib()


LEVEL_SIZES = [1, 2, 3, 5, 4096, 507 * 525, 740 * 1125, 1481 * 1125]


@pytest.mark.gpu
@pytest.mark.parametrize("n", LEVEL_SIZES)
def test_frame_levels_bit_exact_against_the_model(n):
    """tsdrgpu_frame_levels at every frame base phase (0..3 floats past a 16-byte boundary), F = 1 / 17 / 64 (fewer for the
    largest frames), every ppm of the list, frames cycling through the adversarial distributions."""
    import torch
    ctx = _ctx()
    rng = np.random.default_rng(n)
    for phase in range(4):
        nf = (1, 17, 64, 17)[phase] if n < 500_000 else (1, 17, 3, 17)[phase]
        frames = [adversarial(n, (phase + k) % KINDS, rng) for k in range(nf)]
        sk = [valid_sorted_keys(f) for f in frames]
        buf = torch.full((phase + nf * n + 4,), float("nan"), device="cuda")
        buf[phase:phase + nf * n] = torch.from_numpy(np.concatenate(frames)).cuda()
        view = buf[phase:phase + nf * n]
        assert (view.data_ptr() - phase * 4) % 16 == 0
        for ppm in (0, 1, 3500, 10_000, 250_000):
            lo, hi, nv = ctx.frame_levels(view, n, ppm)
            for k in range(nf):
                wl, wh, wn = levels_from_sorted(sk[k], frames[k][0], ppm)
                assert int(nv[k]) == wn, (n, phase, ppm, k)
                assert lo[k].tobytes() == wl.tobytes() and hi[k].tobytes() == wh.tobytes(), (n, phase, ppm, k, lo[k], wl, hi[k], wh)


@pytest.mark.gpu
def test_frame_levels_refuses_bad_arguments():
    import torch
    ctx = _ctx()
    x = torch.zeros(64, device="cuda")
    lo, hi = (C.c_float * 1)(), (C.c_float * 1)()
    lib = _lib()
    assert lib.tsdrgpu_frame_levels(ctx._h, ctx.stream, x.data_ptr(), 64, 1, 250_001, lo, hi, None) == -3
    assert lib.tsdrgpu_frame_levels(ctx._h, ctx.stream, x.data_ptr(), 64, 1, -1, lo, hi, None) == -3
    pg = ctx.post_processor()
    assert lib.tsdrgpu_framestage_set_autogain(pg._h, 2, 0) == -3
    assert lib.tsdrgpu_framestage_set_autogain(pg._h, 1, 250_001) == -3


def _run_stage(ctx, pg, frames_np, w, h, mb, bits, F):
    """Batches of F frames through tsdrgpu_framestage_run_async; returns [(frames, results, reports)] after a join."""
    import torch
    from tests.test_production_batches import results_of, run_async
    keep = []
    for b in range(0, len(frames_np), F):
        x = torch.from_numpy(np.concatenate(frames_np[b:b + F])).cuda()
        out = torch.empty_like(x)
        flags = type("F", (), {"bits": lambda self: bits})()
        res, ag = run_async(ctx, pg, x, len(frames_np[b:b + F]), w, h, mb, flags, out)
        keep.append((x, out, res, ag, len(frames_np[b:b + F])))
    pg.join()
    torch.cuda.synchronize()
    got = []
    for x, out, res, ag, nf in keep:
        o = out.cpu().numpy().reshape(nf, -1)
        rs = [type(r).from_buffer_copy(r) for r in results_of(res, nf)]      # copies: the pinned buffer goes with `keep`
        got += [(o[i], rs[i], ag[i]) for i in range(nf)]
    return got


def _assert_stage(got, want, what, snr=False):
    assert len(got) == len(want)
    for k, ((gf, gr, ga), (wf, wr)) in enumerate(zip(got, want)):
        if snr and np.isfinite(wr["snr"]):
            assert abs(gr.snr - float(wr["snr"])) <= 1e-5 * abs(float(wr["snr"])), f"{what} snr {k}"    # 1e-5 relative (parallel double sums)
        assert np.array_equal(gf.view(np.uint32), wf.view(np.uint32)), f"{what} frame {k}"
        assert (gr.x_dx, gr.x_vx, gr.x_absvx, gr.x_stripsize) == wr["x"] and (gr.y_dx, gr.y_vx, gr.y_absvx, gr.y_stripsize) == wr["y"], f"{what} sync {k}"
        assert gr.avg_speed == wr["avg_speed"] and gr.pll_state == wr["pll_state"], f"{what} pll {k}"
        assert (np.float32(gr.lastmax), np.float32(gr.lastmin)) == (wr["lastmax"], wr["lastmin"]), f"{what} auto-gain state {k}"
        assert ga == wr["report"], f"{what} report {k}"


SMALL_CASES = [(a, l, g, F) for (a, l, g) in FLAGS for F in (1, 17, 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("autoshift,lpbs,aap,F", SMALL_CASES)
def test_frame_stage_clip_matches_the_restatement_small(autoshift, lpbs, aap, F):
    """Clip at 0.35 % through the GPU frame stage, every flag combination, two batches of F frames with spikes and motion
    blur 0.3: frames bit-exact, every result field exact."""
    from tempestsdr_b200 import _native as N
    O = orc.port()
    fs, h, fv = SMALL
    w, _, _ = O.geometry(fs, h, fv)
    frames = _synth_stream(w, h, 2 * F, 700)
    rng = np.random.default_rng(F)
    for f in frames:
        f[rng.integers(0, w * h, 5)] = 5.0
    pr = ClipPostProcessor(O, fs, h, fv, autoshift, 0, ppm=3500)
    want = [pr.run(f, w, h, 0.3, 0.1, lpbs, aap) for f in frames]
    ctx = _ctx()
    pg = ctx.post_processor()
    pg.set_autogain("clip:0.35")
    bits = N.FS_AUTOSHIFT * autoshift | N.FS_LOWPASS_BEFORE_SYNC * lpbs | N.FS_AUTOGAIN_AFTER_PROC * aap
    _assert_stage(_run_stage(ctx, pg, frames, w, h, 0.3, bits, F), want, f"flags {autoshift}{lpbs}{aap} F={F}")


@pytest.mark.gpu
@pytest.mark.parametrize("autoshift,lpbs,aap", [(1, 1, 0), (1, 0, 1), (0, 1, 1), (0, 0, 0)])
def test_frame_stage_clip_with_snr(autoshift, lpbs, aap):
    """Clip at 1 % with TSDRGPU_FS_COMPUTE_SNR: round 1's sum feeds the SNR's mean.  Frames and results bit-exact, SNR within
    1e-5 relative of the restatement (the tolerance of the min/max SNR tests), two batches of 17 frames with spikes."""
    from tempestsdr_b200 import _native as N
    O = orc.port()
    fs, h, fv = SMALL
    w, _, _ = O.geometry(fs, h, fv)
    frames = _synth_stream(w, h, 34, 1300)
    rng = np.random.default_rng(3)
    for f in frames:
        f[rng.integers(0, w * h, 5)] = 5.0
        f[rng.integers(0, w * h, 3)] = 512.0                 # markers: outside the sum, inside the deviations
    pr = ClipPostProcessor(O, fs, h, fv, autoshift, 0, ppm=10_000)
    want = [pr.run(f, w, h, 0.3, 0.1, lpbs, aap) for f in frames]
    ctx = _ctx()
    pg = ctx.post_processor()
    pg.set_autogain("clip:1")
    bits = N.FS_AUTOSHIFT * autoshift | N.FS_LOWPASS_BEFORE_SYNC * lpbs | N.FS_AUTOGAIN_AFTER_PROC * aap | N.FS_COMPUTE_SNR
    _assert_stage(_run_stage(ctx, pg, frames, w, h, 0.3, bits, 17), want, f"snr flags {autoshift}{lpbs}{aap}", snr=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg5", "cfg1"])
@pytest.mark.parametrize("mb", [0.0, 0.3])
def test_frame_stage_clip_at_bench_shapes(name, mb):
    """F = 64 at the benchmark's geometries with the side-stream overlap on, two batches, with and without motion blur."""
    from tempestsdr_b200 import _native as N
    from tests.test_gpu_parity import CFGS
    O = orc.port()
    fs, h, fv = CFGS[name]
    w, _, _ = O.geometry(fs, h, fv)
    frames = _synth_stream(w, h, 128, 900)
    pr = ClipPostProcessor(O, fs, h, fv, 1, 0, ppm=3500)
    want = [pr.run(f, w, h, mb, 0.1, 1, 0) for f in frames]
    ctx = _ctx()
    pg = ctx.post_processor()
    pg.set_overlap(True)
    pg.set_autogain("clip:0.35")
    _assert_stage(_run_stage(ctx, pg, frames, w, h, mb, N.FS_AUTOSHIFT | N.FS_LOWPASS_BEFORE_SYNC, 64), want, name)


@pytest.mark.gpu
def test_ppm0_stream_equals_min_max_and_a_switch_carries_the_iir():
    """ppm = 0 gives the min/max stream bit for bit; switching to clip in mid-stream (and back) keeps lastmin / lastmax going,
    also across tsdrgpu_framestage_reset, which keeps the mode."""
    from tempestsdr_b200 import _native as N
    O = orc.port()
    fs, h, fv = SMALL
    w, _, _ = O.geometry(fs, h, fv)
    frames = _synth_stream(w, h, 48, 1100)
    bits = N.FS_AUTOSHIFT | N.FS_LOWPASS_BEFORE_SYNC
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    b.set_autogain("clip:0")
    ga = _run_stage(ctx, a, frames, w, h, 0.0, bits, 16)
    gb = _run_stage(ctx, b, frames, w, h, 0.0, bits, 16)
    for k, (x, y) in enumerate(zip(ga, gb)):
        assert np.array_equal(x[0].view(np.uint32), y[0].view(np.uint32)) and (x[1].lastmin, x[1].lastmax) == (y[1].lastmin, y[1].lastmax), k
    # mid-stream switch: min/max for 16 frames, clip 1 % for 16, min/max again
    pr = ClipPostProcessor(O, fs, h, fv, 1, 0)
    pg = ctx.post_processor()
    got, want = [], []
    for i, spec in enumerate(("minmax", "clip:1", "minmax")):
        pg.set_autogain(spec)
        pr.ppm = None if spec == "minmax" else 10_000
        chunk = frames[16 * i:16 * (i + 1)]
        got += _run_stage(ctx, pg, chunk, w, h, 0.0, bits, 16)
        want += [pr.run(f, w, h, 0.0, 0.1, 1, 0) for f in chunk]
    _assert_stage(got, want, "switch")
    pg.reset()
    pr2 = ClipPostProcessor(O, fs, h, fv, 1, 0, ppm=10_000)
    pg.set_autogain("clip:1")
    pg.reset()                                          # the mode survives a reset
    _assert_stage(_run_stage(ctx, pg, frames[:16], w, h, 0.0, bits, 16), [pr2.run(f, w, h, 0.0, 0.1, 1, 0) for f in frames[:16]], "after reset")


# -------------------------------------------------------------------------------------------------- pipeline
def replay_box(O, iq_blocks, fs, h, fv, ppm, autoshift=1, pll=0, syncs=None):
    """The pipeline's work on one thread: the oracle's box resampler over every group of ten decimator blocks (cut with the live
    refresh rate), pixel-level drop compensation for tsdr_sync, and the clip-mode restatement one frame at a time."""
    w, _, _ = O.geometry(fs, h, fv)
    rs = O.resampler()
    pp = ClipPostProcessor(O, fs, h, fv, autoshift, pll, ppm=ppm)
    decim = np.zeros(0, np.float32); pix = np.zeros(0, np.float32)
    fv_live, w_live = fv, w
    frames, values, diff, pending = [], [], 0, 0
    for call, iq in enumerate(iq_blocks):
        decim = np.concatenate([decim, O.am_demod(iq)])
        while True:
            block = int(0.1 * fs / fv_live)
            if decim.size < 10 * block:
                break
            w_grp, fv_grp = w_live, fv_live
            n = w_grp * h
            px = np.concatenate([rs.run(decim[k * block:(k + 1) * block], float(w_grp * h) * fv_grp, float(fs)) for k in range(10)])
            decim = decim[10 * block:]
            diff, fwd, skip = O.dropcomp_add(diff, px.size, n, True)
            pix = np.concatenate([pix, px[skip:skip + fwd]])
            if pending:
                diff = O.dropcomp_shift_with(diff, n, -pending); pending = 0
            while pix.size >= n:
                out, res = pp.run(pix[:n], w_grp, h, 0.0, 0.1, 1, 0)
                frames.append((out, w_grp)); pix = pix[n:]
                if res["report"]:
                    values.append((float(res["lastmin"]), float(res["lastmax"])))
                if pll:
                    fv_live, w_live = res["refreshrate"], res["width"]
        if syncs and call in syncs:
            pending += syncs[call]
    return frames, values


def run_pipeline(fs, h, fv, blocks, autogain, params, batch=1, syncs=None, dropped=None):
    from tempestsdr_b200 import pipeline
    got, values = [], []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=batch, batch_blocks=10 * batch, block_when_busy=True,
                          params=params, on_frame=lambda f, ww, hh: got.append((f.copy(), ww)),
                          on_value=lambda vid, a, b: values.append((a, b)) if vid == 3 else None, autogain=autogain)
    for k, b in enumerate(blocks):
        p.process(b, (dropped or {}).get(k, 0))
        if syncs and k in syncs:
            p.sync(syncs[k])
    p.flush()
    p.close()
    return got, values


def _assert_frames(got, want):
    assert len(got) > 3 and len(got) == len(want)
    for k, ((g, gw), (wv, ww)) in enumerate(zip(got, want)):
        assert gw == ww and np.array_equal(g.view(np.uint32), wv.view(np.uint32)), f"frame {k}"


@pytest.mark.gpu
def test_pipeline_clip_matches_stagewise_replay():
    """Pipeline(autogain="clip:0.35") against the replay; value id 3 carries the clipped lastmin / lastmax."""
    O = orc.port()
    fs, h, fv = SMALL
    w, _, _ = O.geometry(fs, h, fv)
    nblk, items = 24, 65536
    iq_all = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=21)
    blocks = [iq_all[k * items:(k + 1) * items].copy() for k in range(nblk)]
    want, wvals = replay_box(O, blocks, fs, h, fv, 3500)
    got, gvals = run_pipeline(fs, h, fv, blocks, "clip:0.35", {"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1})
    _assert_frames(got, want)
    assert len(wvals) >= 2 and gvals == wvals


@pytest.mark.gpu
def test_pipeline_clip_with_the_pll_on():
    O = orc.port()
    fs, h, fv = SMALL
    w, _, _ = O.geometry(fs, h, fv)
    total, items = 24 * 65536, 65536
    iq_all = synth.video_like_iq(total // 2, fs, w, h, fv, seed=61, fv_ppm=2500.0)
    blocks = [iq_all[k:k + items].copy() for k in range(0, total, items)]
    want, _ = replay_box(O, blocks, fs, h, fv, 3500, pll=1)
    got, _ = run_pipeline(fs, h, fv, blocks, "clip:0.35", {"autoshift": 1, "framerate_pll": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1})
    _assert_frames(got, want)


@pytest.mark.gpu
def test_pipeline_clip_with_dropped_samples_and_manual_sync():
    O = orc.port()
    fs, h, fv = SMALL
    w, _, pt = O.geometry(fs, h, fv)
    items = 65536
    iq_all = synth.video_like_iq(30 * items // 2, fs, w, h, fv, seed=22)
    blocks = [iq_all[k * items:(k + 1) * items].copy() for k in range(30)]
    block = int(round(((w * h) << 1) * pt))
    dropped, diff, fed = 12345, 0, []
    for k, b in enumerate(blocks):
        diff = O.dropcomp_shift_with(diff, block, dropped if k == 7 else 0)
        diff, fwd, skip = O.dropcomp_add(diff, items // 2, block, True)
        fed.append(b[2 * skip:] if fwd else b[:0])
    syncs = {12: 37, 20: -5}
    want, _ = replay_box(O, fed, fs, h, fv, 3500, autoshift=0, syncs=syncs)
    got, _ = run_pipeline(fs, h, fv, blocks, "clip:0.35", {"autoshift": 0, "autocorr_plots_off": 1}, syncs=syncs, dropped={7: dropped})
    _assert_frames(got, want)


@pytest.mark.gpu
def test_host_library_with_clip_autogain_matches_the_pipeline(tmp_path, monkeypatch):
    """TSDR_AUTOGAIN=clip:0.35: tsdr_readasync driven by a RawFile plugin delivers the frames of the pipeline-level run."""
    from tests.test_host_library import FRAME_CB, MINE, PLOT_CB, VALUE_CB, bind
    fs, h, fv = SMALL
    O = orc.port()
    w, _, _ = O.geometry(fs, h, fv)
    items = 512 * 1024
    nblk = 6
    iq = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=31)
    raw = tmp_path / "iq.raw"
    iq.tofile(raw)
    want, _ = run_pipeline(fs, h, fv, [iq[k * items:(k + 1) * items].copy() for k in range(nblk)], "clip:0.35",
                           {"autoshift": 1, "framerate_pll": 0, "lowpass_before_sync": 1})
    if orc.have_ref():
        plugin, args = orc.REF_RAWFILE_SO, f'"{raw}" {fs} float'
    else:
        plugin, args = os.path.join(os.path.dirname(MINE), "TSDRPlugin_RawFileGPU.so"), f'"{raw}" {fs} float'
    monkeypatch.setenv("TSDR_NO_DROP", "1")
    monkeypatch.setenv("TSDR_AUTOGAIN", "clip:0.35")
    got = []
    lib = bind(MINE)
    t = C.c_void_p()
    nv, npl = VALUE_CB(lambda *a: None), PLOT_CB(lambda *a: None)
    fcb = FRAME_CB(lambda b, ww, hh, c: got.append(np.ctypeslib.as_array(b, shape=(ww * hh,)).copy()))
    lib.tsdr_init(C.byref(t), nv, npl, None)
    lib.tsdr_setresolution(t, h, fv); lib.tsdr_motionblur(t, 0.0); lib.tsdr_setgain(t, 0.5)
    for pid, v in ((0, 1), (1, 0), (6, 1)):
        lib.tsdr_setparameter_int(t, pid, v)
    assert lib.tsdr_loadplugin(t, plugin.encode(), args.encode()) == 0
    rc = []
    th = threading.Thread(target=lambda: rc.append(lib.tsdr_readasync(t, fcb, None)))
    th.start()
    deadline = time.time() + 60
    while len(got) < len(want) and time.time() < deadline:
        time.sleep(0.05)
    assert lib.tsdr_stop(t) == 0
    th.join(timeout=30)
    assert rc == [0]
    assert len(got) >= len(want) > 3
    for k, (wv, _) in enumerate(want):
        assert np.array_equal(got[k].view(np.uint32), wv.view(np.uint32)), f"frame {k}"
    lib.tsdr_free(C.byref(t))
