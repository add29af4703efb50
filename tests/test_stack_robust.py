"""The glitch-tolerant stack (TSDRGPU_STACK_ROBUST, include/tsdrgpu.h): the numpy model of tests/stack_robust_model.py checked
against the literal definition, against the track stack where nothing is held or gated, and for the quality it keeps through
one-frame disturbances (a frame of noise, a band of corrupted lines, a torn frame); then the GPU stage object, the frame stage,
the pipeline and the host library held bit for bit to (the same run without the stack) followed by the model.  The scenes are
synthetic: how often real captures hold such frames has not been measured."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from tests.stack_adapt_model import AdaptModel
from tests.stack_model import StackModel
from tests.stack_robust_model import GATED, RobustModel, robust_literal
from tests.stack_track_model import TrackModel
from tests.test_stack_adapt import _assert_same_adapt, _rec
from tests.test_stack_align import (ADVERSARIAL, STACK_SPECS_BAD, STACK_SPECS_OK, _ctx, _gpu_run, _picture, _pipeline, _psnr,
                                    _shift)
from tests.test_stack_track import _glyphs, _moving_frames, _scroll_frames, _scroll_scene, _vectors

F32 = np.float32


def _counts(m):
    return m.held, m.gated, m.hold


def _glitch(f, w, h, kind, rng):
    """One frame disturbed: "noise" replaces it by uniform noise, "band" the middle third of its lines, "torn" shifts the raster
    circularly by a third of the frame plus 137 pixels (not a multiple of W for any W > 137), "tear" by half a line."""
    f = f.copy()
    if kind == "noise":
        f[:] = rng.uniform(0, 1, f.size)
    elif kind == "band":
        f.reshape(h, w)[h // 3:max(h // 3 + 1, 2 * h // 3)] = rng.uniform(0, 1, (max(1, 2 * h // 3 - h // 3), w))
    elif kind == "torn":
        f = np.roll(f, f.size // 3 + 137)
    elif kind == "tear":
        f = np.roll(f, max(1, w // 2))
    return f.astype(F32)


def _glitched_frames(w, h, F, rng, events, drift=0.6, noise=0.03, adversarial=0):
    """A text patch over a blocky picture drifting along the raster, with {frame: kind} one-frame disturbances."""
    pic = _picture(w, h, rng).reshape(h, w)
    if w >= 16 and h >= 24:
        ph, pw = h // 2, w // 2
        pic[h // 4:h // 4 + ph, w // 4:w // 4 + pw] = _glyphs((ph + 11) // 12, (pw + 7) // 8, rng)[:ph, :pw]
    pic = pic.reshape(-1)
    out = []
    for k in range(F):
        f = (_shift(pic, drift * k) + rng.normal(0, noise, w * h)).astype(F32)
        if k in events:
            f = _glitch(f, w, h, events[k], rng)
        if adversarial:
            f[rng.integers(0, w * h, adversarial)] = rng.choice(ADVERSARIAL, adversarial)
        out.append(f)
    return out


# ============================================================================================================== CPU
@pytest.mark.parametrize("w,h,depth,rx,ry,scene", [
    (1, 1, 2, 1, 0, "glitch"),                 # smaller than a tile: a changed tile is the whole frame
    (7, 5, 3, 8, 2, "move"),
    (20, 12, 4, 3, 1, "glitch"),               # smaller than the search window, partial tiles
    (40, 24, 8, 8, 2, "flat"),                 # flat content: ties everywhere
    (37, 34, 8, 4, 1, "glitch"),               # a noise frame, a band and a torn frame
    (48, 40, 16, 8, 2, "move"),
])
def test_model_equals_the_literal_definition(w, h, depth, rx, ry, scene):
    """Markers, NaN, +-inf and out-of-range values in every case; per frame the outputs, the records, the vectors and the counts."""
    rng = np.random.default_rng(w * 31 + h * 7 + rx)
    if scene == "glitch":
        frames = _glitched_frames(w, h, 10, rng, {3: "noise", 6: "band", 8: "torn"}, adversarial=max(1, w * h // 60))
    else:
        frames = _moving_frames(w, h, 9, rng, (2, 1) if scene == "move" else (3, -2), 3, noise=0.0 if scene == "flat" else 0.02,
                                adversarial=max(1, w * h // 60), flat=scene == "flat")
    m = RobustModel(depth, rx, ry)
    outs, recs, vecs, cnts = [], [], [], []
    for f in frames:
        o, r = m.run(f, w, h)
        outs.append(o); recs.append(r); vecs.append(_vectors(m, w, h)); cnts.append(_counts(m))
    lo, lr, lv, lc = robust_literal(frames, w, h, depth, rx, ry)
    assert np.array_equal(np.stack(outs).view(np.uint32), lo.view(np.uint32))
    assert [_rec(r) for r in recs] == [_rec(r) for r in lr]
    assert vecs == lv
    assert cnts == lc
    if w * h > 1000:
        assert any(c[0] for c in cnts) and any(c[1] for c in cnts), cnts
    if scene == "glitch" and w * h > 100:
        assert any(c[2] for c in cnts), cnts


def _assert_equals_track(frames, w, h, depth=16):
    rm, tm = RobustModel(depth), TrackModel(depth)
    moved = 0
    for k, f in enumerate(frames):
        ro, rr = rm.run(f, w, h)
        to, tr = tm.run(f, w, h)
        assert _counts(rm) == (0, 0, False), (k, _counts(rm))
        assert np.array_equal(ro.view(np.uint32), to.view(np.uint32)) and _rec(rr) == _rec(tr), k
        assert np.array_equal(rm.vectors, tm.vectors) and rm.moved == tm.moved, k
        moved += tm.moved
    return moved


@pytest.mark.parametrize("w,h,drift", [(64, 48, 0.37), (100, 37, 5.3), (256, 128, 1.3), (17, 5, 0.6)])
def test_equals_track_on_static_frames(w, h, drift):
    """A blocky picture drifting by a band-limited sub-pixel shift at sigma = 0.01: nothing held or gated, and every frame,
    record and vector is track's bit for bit.  (One-pixel strokes under a sub-pixel drift, or sigma = 0.02 over enough
    pixel-frames, do gate a few pixels: DESIGN.md section 5.5.)"""
    rng = np.random.default_rng(int(w + 100 * drift))
    pic = _picture(w, h, rng, strokes=False)
    _assert_equals_track([(_shift(pic, drift * k) + rng.normal(0, 0.01, w * h)).astype(F32) for k in range(40)], w, h)


def test_equals_track_on_a_scroll_that_exposes_nothing_new():
    """Three rows of text with blank margins scrolling up a 12-line row every 4 frames (twice), drifting by 1 px/frame, at
    sigma = 0.01: every tile the scroll
    crosses finds its content and moves, nothing is held or gated, and frames, records and vectors are track's."""
    w, h = 128, 96
    rng = np.random.default_rng(21)
    page = np.full((h + 200, w), 0.1)
    page[40:76, 16:112] = _glyphs(3, 12, rng)
    frames = []
    for k in range(30):
        top = 0 if k < 6 else min((k - 6) // 4 + 1, 2) * 12
        frames.append((_shift(page[top:top + h].reshape(-1), 1.0 * k) + rng.normal(0, 0.01, w * h)).astype(F32))
    assert _assert_equals_track(frames, w, h, 32) > 0


def test_stack_robust_spec_parsing():
    """tsdrgpu_stack_parse with the robust: prefix: the same spellings as align: accepted and refused."""
    from tempestsdr_b200 import _native as N
    lib = N.lib()
    for spec, want in STACK_SPECS_OK.items():
        spec = spec.replace("align:", "robust:")
        assert N.stack_mode(spec) == ((N.STACK_ROBUST,) + want[1:] if want[0] else want), spec
    for spec in STACK_SPECS_BAD + ["robust:32:8x2,align:32", "robustalign:32", "Robust:32", "robusts:32", "robust32", "robust:"]:
        spec = spec.replace("align:", "robust:")
        out = [C.c_int(-7) for _ in range(4)]
        assert lib.tsdrgpu_stack_parse(spec.encode(), *[C.byref(o) for o in out]) == -3, spec
        assert [o.value for o in out] == [-7] * 4, spec
        with pytest.raises(ValueError):
            N.stack_mode(spec)
    assert N.stack_mode("track:32") == (N.STACK_TRACK, 32, 8, 2)
    assert N.STACK_ROBUST == 16


@pytest.mark.parametrize("value", ["robust:1", "robust:1025", "robust:32:33x2", "robust:32:8x9", "robust", "robust:+32", "robust:32:8x2 "])
def test_bogus_robust_setting_is_refused_by_the_host_library(tmp_path, monkeypatch, value):
    """TSDR_STACK=robust:... out of range or misspelt: tsdr_readasync fails with TSDR_INVALID_PARAMETER_VALUE."""
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
    monkeypatch.setenv("TSDR_STACK", value)
    assert lib.tsdr_readasync(t, FRAME_CB(lambda *a: None), None) == 9          # TSDR_INVALID_PARAMETER_VALUE
    assert b"TSDR_STACK" in lib.tsdr_getlasterrortext(t)
    assert b"robust" in lib.tsdr_getlasterrortext(t)
    assert lib.tsdr_isrunning(t) == 0
    lib.tsdr_free(C.byref(t))


# -------------------------------------------------------------------------------------------------- quality
W_Q, H_Q, F_Q, AT = 256, 128, 72, 32


def _terminal(rng):
    """The quality scenes' picture: a 192 x 96 region of terminal text at (32, 16) on a blocky picture with strokes."""
    pic = _picture(W_Q, H_Q, rng).reshape(H_Q, W_Q)
    pic[16:112, 32:224] = _glyphs(8, 24, rng)
    return pic.reshape(-1)


def _event_run(kind, sigma=0.05, drift=0.37, seed=1, models=(AdaptModel, TrackModel, RobustModel), pics=None):
    """The terminal drifting by `drift` px/frame with a one-row jump every 23 frames, sigma noise, frame AT disturbed by `kind`
    (or none), through the models at depth 32 -> per frame [PSNR of the whole output against the truth per model], the robust
    model's counts per frame, the records per model."""
    rng = np.random.default_rng(seed)
    pic = _terminal(rng)
    d = np.array([drift * k + W_Q * (k // 23) for k in range(F_Q)])
    ms = [M(32) for M in models]
    psnr, counts, recs = [], [], [[] for _ in ms]
    for k in range(F_Q):
        p = pic if pics is None else pics[k]
        f = (_shift(p, d[k]) + rng.normal(0, sigma, W_Q * H_Q)).astype(F32)
        if k == AT and kind:
            f = _glitch(f, W_Q, H_Q, kind, rng)
        row = []
        for i, m in enumerate(ms):
            o, r = m.run(f, W_Q, H_Q)
            R = math.floor(r["offset"] + 0.5)
            row.append(_psnr(o, _shift(p, d[0] + R)))
            recs[i].append(r)
        psnr.append(row)
        counts.append(_counts(ms[-1]))
    return np.array(psnr), counts, recs


@pytest.mark.parametrize("kind", ["noise", "band"])
def test_quality_through_a_one_frame_disturbance(kind):
    """A frame of noise, or a third of its lines corrupted, at frame 32 (sigma 0.05, 0.37 px/frame).  Robust delivers the
    average through the event, within 1.5 dB of the undisturbed run at every frame; adapt and track restart with the bad frame,
    fall below by more than 10 dB at the event and take about N = 32 frames to come back (DESIGN.md section 5.5 has both
    curves)."""
    ev, counts, _ = _event_run(kind)
    calm, _, _ = _event_run(None, models=(RobustModel,))
    rb, ad, tk = ev[:, 2], ev[:, 0], ev[:, 1]
    assert np.all(rb[AT:] >= calm[AT:, 0] - 1.5), (rb[AT:AT + 12], calm[AT:AT + 12, 0])
    assert counts[AT][0] > 0 and counts[AT][2] == (kind == "noise"), counts[AT]
    assert ad[AT] < calm[AT, 0] - 10 and tk[AT] < calm[AT, 0] - 10, (ad[AT], tk[AT])
    assert np.array_equal(ad, tk)
    assert ad[AT + 4] < calm[AT + 4, 0] - 3, ad[AT + 4]          # still rebuilding
    assert np.all(rb[AT:AT + 16] > ad[AT:AT + 16] + 0.5)


@pytest.mark.parametrize("kind", ["torn", "tear"])
def test_a_torn_frame_is_held_on_the_prediction(kind):
    """The raster shifted for one frame (a third of a frame, or half a line): robust holds the frame, the delivered offset stays
    on the constant-velocity prediction and the search after it is as if the frame had not been there; the output at the
    event is the average moved by R(b)."""
    ev, counts, recs = _event_run(kind)
    calm, _, crecs = _event_run(None, models=(RobustModel,))
    assert counts[AT][2], counts[AT]
    rr = recs[2]
    o1, o2 = rr[AT - 1]["offset"], rr[AT - 2]["offset"]
    b = math.floor(o1 + 0.5) * 2.0 - math.floor(o2 + 0.5)
    assert rr[AT]["offset"] == b and rr[AT]["changed"] == 0
    assert abs(rr[AT + 1]["offset"] - crecs[0][AT + 1]["offset"]) < 0.5
    assert np.all(ev[AT:, 2] >= calm[AT:, 0] - 1.5), (ev[AT:AT + 8, 2], calm[AT:AT + 8, 0])
    if kind == "torn":                                               # track and adapt lose the registration for good
        assert np.all(ev[AT + 8:, 1] < calm[AT + 8:, 0] - 10), ev[AT + 8:, 1]


def test_a_typed_word_appears_one_frame_later_and_stays():
    """New text in a 64 x 16 region at frame 32: track shows it from frame 32, robust holds the region one frame and shows it
    from frame 33, and keeps it: from frame 36 on robust reads within 4 dB of track over the region (it trails by 1.5-3.5 dB
    for about ten frames: DESIGN.md section 5.5)."""
    rng = np.random.default_rng(5)
    pic = _terminal(rng)
    region = np.zeros((H_Q, W_Q), bool)
    region[53:69, 37:101] = True
    pic2 = pic.copy().reshape(H_Q, W_Q)
    pic2[region] = np.where(rng.uniform(size=(16, 64)) < 0.3, 0.9, 0.1).reshape(-1)
    pics = [pic2.reshape(-1) if k >= AT else pic for k in range(F_Q)]
    rng = np.random.default_rng(6)
    d = np.array([0.37 * k + W_Q * (k // 23) for k in range(F_Q)])
    tm, rm = TrackModel(32), RobustModel(32)
    got = []
    for k in range(F_Q):
        f = (_shift(pics[k], d[k]) + rng.normal(0, 0.05, W_Q * H_Q)).astype(F32)
        row = []
        for m in (tm, rm):
            o, r = m.run(f, W_Q, H_Q)
            R = math.floor(r["offset"] + 0.5)
            mk = np.roll(region.reshape(-1), R)
            row.append((_psnr(o[mk], _shift(pics[k], d[0] + R)[mk]), r["changed"]))
        got.append(row)
        if k == AT:
            assert rm.held > 0 and not rm.hold
    (t32, tc32), (r32, rc32) = got[AT]
    (t33, _), (r33, rc33) = got[AT + 1]
    assert tc32 > 0 and rc32 == 0 and rc33 > 0
    assert r32 < t32 - 6, (r32, t32)                                  # still the old content
    assert r33 > r32 + 8, (r33, r32)                                  # the new word, a frame late
    for k in range(AT + 4, F_Q):
        assert got[k][1][0] >= got[k][0][0] - 4.0, (k, got[k])


def test_a_scroll_is_carried_as_in_track():
    """The track study's scrolling terminal (a new row appears at the bottom at every scroll): the moved text reads within
    0.5 dB of track 3-5 frames after each scroll, and robust carries as many tiles as track does."""
    rng = np.random.default_rng(7)
    pics, moved, _, _ = _scroll_scene(False, rng)
    d = np.array([0.37 * k + W_Q * (k // 23) for k in range(64)])
    tm, rm = TrackModel(32), RobustModel(32)
    diffs, carried = [], [0, 0]
    for k in range(64):
        f = (_shift(pics[k], d[k]) + rng.normal(0, 0.05, W_Q * H_Q)).astype(F32)
        row = []
        for i, m in enumerate((tm, rm)):
            o, r = m.run(f, W_Q, H_Q)
            R = math.floor(r["offset"] + 0.5)
            carried[i] += int(np.any(m.vectors != 0, axis=2).sum())
            if moved[k].any():
                mk = np.roll(moved[k], R)
                row.append(_psnr(o[mk], _shift(pics[k], d[0] + R)[mk]))
        if row and (k - 24) % 6 in (3, 4, 5):
            diffs.append(row[1] - row[0])
    assert np.mean(diffs) >= -0.5, diffs
    assert carried[1] >= 0.9 * carried[0] > 0, carried


def test_a_lone_pixel_that_persists_is_taken_on_its_second_frame():
    """A still picture at sigma = 0.01; from frame 12 one pixel of a flat block reads 0.16 higher (41 levels, too little for
    the tile to change).  Frame 12 gates it and keeps the average (bit 15 set), frame 13 gates it again and restarts it at the
    new value (count 1), frame 14 blends it normally."""
    w, h = 64, 48
    rng = np.random.default_rng(9)
    pic = _picture(w, h, rng, strokes=False)
    p = 20 * w + 30
    frames = []
    for k in range(18):
        f = pic.copy()
        if k >= 12:
            f[p] += 0.16
        frames.append((f + rng.normal(0, 0.01, w * h)).astype(F32))
    m = RobustModel(32)
    for k, f in enumerate(frames):
        o, r = m.run(f, w, h)
        assert abs(r["offset"]) < 0.5 and m.held == 0 and not m.hold
        if k < 12 or k >= 14:
            assert m.gated == 0, k
            assert m.c[p] & GATED == 0
        if k == 12:
            assert m.gated == 1 and m.c[p] & GATED and abs(o[p] - pic[p]) < 0.02, (m.gated, o[p], pic[p])
        if k == 13:
            assert m.gated == 1 and m.c[p] == 1 and abs(o[p] - pic[p] - 0.16) < 0.04, (m.gated, o[p], pic[p])
        if k == 14:
            assert m.c[p] == 2
    assert abs(o[p] - pic[p] - 0.16) < 0.02


# ============================================================================================================== GPU
SHAPES = [(1, 1), (3, 2), (7, 5), (16, 16), (31, 17), (507, 525), (740, 1125), (1481, 1125)]
SETTINGS = [(2, 1, 0), (32, 8, 2), (1024, 32, 8)]


def _gpu_robust(st, frames, w, h, pin, pout, cut, model, what):
    """frames through Stack.run in batches of `cut`: every frame and record against the model, and after every batch the
    vectors and counts of its last frame.  -> the (held, gated, glitch frames) the batches' last frames reported, summed."""
    seen = np.zeros(3, np.int64)
    for b in range(0, len(frames), cut):
        got, recs = _gpu_run(st, frames[b:b + cut], w, h, pin, pout, cut)
        want, wrecs = model.run_many(frames[b:b + cut], w, h)
        _assert_same_adapt(got, recs, want, wrecs, (what, b))
        assert np.array_equal(st.vectors(w, h), model.vectors), (what, b)
        c = st.robust_counts()
        assert c == _counts(model), (what, b, c, _counts(model))
        seen += np.array(c, np.int64)
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", SHAPES)
def test_robust_stage_bit_exact_against_the_model(w, h):
    """Each depth x window at this size, a text patch with a noise frame, a band and a torn frame, adversarial values, the
    16-byte phases of input and output cycling; frames, records, vectors and counts exact."""
    ctx = _ctx()
    big, huge = w * h > 100_000, w * h > 500_000              # the model searches every tile of a noise or torn frame
    rng = np.random.default_rng(w * 10007 + h + 5)
    for c, (depth, rx, ry) in enumerate(SETTINGS):
        F = 5 if huge else 8 if big else 14
        events = {2: "band"} if huge else {2: "band", 4: "noise", 6: "torn"} if big else {3: "noise", 6: "band", 7: "band", 10: "torn"}
        frames = _glitched_frames(w, h, F, rng, events, drift=(0.4, 2.6, 13.2)[c], adversarial=max(1, w * h // 5000))
        st = ctx.stack()
        st.set(f"robust:{depth}:{rx}x{ry}")
        k = c + w + h
        _gpu_robust(st, frames, w, h, k % 4, (k // 4) % 4, 1 if w * h > 1000 else (1, 5, F)[c], RobustModel(depth, rx, ry),
                    (w, h, depth, rx, ry))


@pytest.mark.gpu
def test_robust_stage_on_scrolling_and_typing():
    """The scrolling terminal and a moving text patch at 256 x 128, with disturbances: tiles are carried, held and gated, and
    the GPU follows the model bit for bit."""
    ctx = _ctx()
    rng = np.random.default_rng(12)
    scenes = [_scroll_frames(256, 128, 24, rng)]
    scenes[0][9] = _glitch(scenes[0][9], 256, 128, "band", rng)
    scenes[0][15] = _glitch(scenes[0][15], 256, 128, "noise", rng)
    scenes.append(_moving_frames(256, 128, 20, rng, (3, 2), 4, drift=0.6, noise=0.03))
    total = np.zeros(3, np.int64)
    for frames in scenes:
        st = ctx.stack()
        st.set("robust:32")
        total += _gpu_robust(st, frames, 256, 128, 1, 2, 1, RobustModel(32), "scene")
    assert np.all(total > 0), total


@pytest.mark.gpu
def test_robust_stage_every_16_byte_phase_pair():
    ctx = _ctx()
    w, h = 61, 37
    frames = _glitched_frames(w, h, 6, np.random.default_rng(5), {2: "noise", 4: "band"}, drift=1.7, adversarial=6)
    for pin in range(4):
        for pout in range(4):
            st = ctx.stack()
            st.set("robust:16")
            _gpu_robust(st, frames, w, h, pin, pout, 2, RobustModel(16), (pin, pout))


@pytest.mark.gpu
def test_robust_stage_batch_cuts_give_the_same_bits():
    """The same 64 frames of a scrolling terminal with disturbances as 64 x 1, 4 x 16 and 1 x 64."""
    ctx = _ctx()
    w, h = 507, 525
    rng = np.random.default_rng(6)
    frames = _scroll_frames(w, h, 64, rng)
    for k, kind in ((10, "noise"), (17, "band"), (30, "torn"), (45, "band"), (46, "band")):
        frames[k] = _glitch(frames[k], w, h, kind, rng)
    runs = []
    for cut in (1, 16, 64):
        st = ctx.stack()
        st.set("robust:32")
        runs.append(_gpu_run(st, frames, w, h, 0, 0, cut) + (st.vectors(w, h), st.robust_counts()))
    for got, recs, v, c in runs[1:]:
        _assert_same_adapt(got, recs, runs[0][0], runs[0][1], "cut")
        assert np.array_equal(v, runs[0][2]) and c == runs[0][3]
    m = RobustModel(32)
    want, wrecs = m.run_many(frames[:20], w, h)
    _assert_same_adapt(runs[0][0][:20], runs[0][1][:20], want, wrecs, "model")


@pytest.mark.gpu
def test_robust_stage_restarts_clear_pend_and_the_gate_bits():
    """A band at the last frame of a batch leaves tiles pending and pixels gated; a reset, a set that changes the settings
    (track to robust and back too) and a geometry change each restart them: the next band is held, not confirmed, exactly as
    the model restarted from scratch says.  The counts query refuses until a frame has been taken in robust mode."""
    ctx = _ctx()
    rng = np.random.default_rng(7)
    w, h = 96, 64
    a = _glitched_frames(w, h, 30, rng, {4: "band", 7: "band", 11: "band", 16: "noise", 23: "band", 28: "band"})
    b = _glitched_frames(w + 3, h, 6, rng, {1: "band", 2: "band"})
    st = ctx.stack()
    with pytest.raises(Exception):
        st.robust_counts()
    st.set("robust:8")
    m = RobustModel(8)
    _gpu_robust(st, a[:5], w, h, 0, 0, 5, m, "first")
    assert m.pend.any() and st.robust_counts()[0] > 0
    st.reset(); m.restart()
    with pytest.raises(Exception):
        st.robust_counts()
    _gpu_robust(st, a[5:8], w, h, 0, 0, 3, m, "after reset")
    st.set("robust:8")                                            # unchanged: carries on
    got, recs = _gpu_run(st, a[8:12], w, h, 0, 0, 4)
    assert recs[0].restarted == 0
    _assert_same_adapt(got, recs, *m.run_many(a[8:12], w, h), "same set")
    st.set("track:8")
    got, recs = _gpu_run(st, a[12:16], w, h, 0, 0, 4)
    assert recs[0].restarted == 1
    _assert_same_adapt(got, recs, *TrackModel(8).run_many(a[12:16], w, h), "track")
    with pytest.raises(Exception):
        st.robust_counts()
    st.set("robust:8:4x1")
    m = RobustModel(8, 4, 1)
    _gpu_robust(st, a[16:24], w, h, 0, 0, 8, m, "after set")
    _gpu_robust(st, a[24:30], w, h, 0, 0, 6, m, "carried on")
    got, recs = _gpu_run(st, b, w + 3, h, 0, 0, 6)
    assert recs[0].restarted == 1
    _assert_same_adapt(got, recs, *m.run_many(b, w + 3, h), "new geometry")
    assert st.robust_counts() == _counts(m)
    assert np.array_equal(st.vectors(w + 3, h), m.vectors)


@pytest.mark.gpu
def test_robust_stage_accepts_its_mode_and_refuses_bad_settings():
    """TSDRGPU_STACK_ROBUST with align's ranges; the values next to the modes are no modes."""
    from tempestsdr_b200 import _native as N
    ctx = _ctx()
    lib = N.lib()
    st = ctx.stack()
    R = N.STACK_ROBUST
    for args in ((2, 32, 8, 2), (3, 32, 8, 2), (5, 32, 8, 2), (12, 32, 8, 2), (15, 32, 8, 2), (17, 32, 8, 2), (32, 32, 8, 2),
                 (R, 1, 8, 2), (R, 1025, 8, 2), (R, 32, 0, 2), (R, 32, 33, 2), (R, 32, 8, -1), (R, 32, 8, 9)):
        assert lib.tsdrgpu_stack_set(st._h, *args) == -3, args
    assert lib.tsdrgpu_stack_set(st._h, R, 32, 8, 2) == 0
    pg = ctx.post_processor()
    assert lib.tsdrgpu_framestage_set_stack(pg._h, R, 32, 8, 2) == 0
    assert lib.tsdrgpu_framestage_set_stack(pg._h, R, 1, 8, 2) == -3
    assert lib.tsdrgpu_framestage_set_stack(pg._h, 5, 32, 8, 2) == -3


# -------------------------------------------------------------------------------------------------- frame stage
FLAGS = [(a, l, g, s) for a in (0, 1) for l in (0, 1) for g in (0, 1) for s in (0, 1)]   # autoshift, lp before sync, aap, super-res


@pytest.mark.gpu
@pytest.mark.parametrize("autoshift,lpbs,aap,superres", FLAGS)
@pytest.mark.parametrize("overlap", [0, 1])
def test_frame_stage_robust_is_the_plain_run_followed_by_the_model(autoshift, lpbs, aap, superres, overlap):
    """Every flag combination, motion blur 0.3, overlap off and on, two batches of 17 frames; deblur, NLM and CLAHE on as well
    in some cases: robust on equals the stack off followed by the model, then the deblur, NLM and CLAHE models; records of the
    last batch equal the model's; results unchanged."""
    from oracle import oracle as orc
    from tempestsdr_b200 import _native as N
    from tests.test_contrast_clahe import _run_stage, _stream
    from tests.test_stack_track import _assert_chain
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = orc.port().geometry(fs, h, fv)
    frames = _stream(w, h, 34, 7700 + 8 * autoshift + 4 * lpbs + 2 * aap + superres)
    bits = (N.FS_AUTOSHIFT * autoshift | N.FS_LOWPASS_BEFORE_SYNC * lpbs | N.FS_AUTOGAIN_AFTER_PROC * aap
            | N.FS_SUPERRESOLUTION * superres)
    k = autoshift + lpbs + aap + superres + overlap
    kw = {}
    if k % 4 == 1:
        kw = dict(db=(110, 12))
    elif k % 4 == 2:
        kw = dict(nl=(150, 2, 1))
    elif k % 4 == 3:
        kw = dict(db=(110, 12), nl=(150, 2, 1), ct=(250, 8, 8))
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    for pg in (a, b):
        pg.set_overlap(bool(overlap))
    b.set_stack("robust:16:8x2")
    if "db" in kw:
        b.set_deblur("rl:1.1:12")
    if "nl" in kw:
        b.set_denoise("nlm:0.15:2:1")
    if "ct" in kw:
        b.set_contrast("clahe:2.5:8x8")
    off = _run_stage(ctx, a, frames, w, h, 0.3, bits, 17)
    on = _run_stage(ctx, b, frames, w, h, 0.3, bits, 17)
    _assert_chain(on, off, w, h, RobustModel(16, 8, 2), f"flags {autoshift}{lpbs}{aap}{superres} overlap {overlap}", **kw)
    m2 = RobustModel(16, 8, 2)
    _, wrecs = m2.run_many([o[0] for o in off], w, h)
    assert [_rec(r) for r in b.stack_records(17)] == [_rec(r) for r in wrecs[17:]]


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [0, 1])
def test_switching_among_off_align_adapt_track_and_robust_batch_by_batch(overlap):
    """robust, off, align, adapt, track, robust, off, track, robust per batch of 8 (every switch restarts the stack), then a
    reset: each batch equals the plain run followed by its own model, the off batches equal a run that never switched."""
    from oracle import oracle as orc
    from tempestsdr_b200 import _native as N
    from tests.test_contrast_clahe import _run_stage, _stream
    from tests.test_stack_track import _assert_chain
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = orc.port().geometry(fs, h, fv)
    frames = _stream(w, h, 72, 8200)
    bits = N.FS_AUTOSHIFT | N.FS_LOWPASS_BEFORE_SYNC
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    for pg in (a, b):
        pg.set_overlap(bool(overlap))
    off = _run_stage(ctx, a, frames, w, h, 0.2, bits, 8)
    modes = ["robust:4:2x1", "off", "align:4:2x1", "adapt:4:2x1", "track:4:2x1", "robust:4:2x1", "off", "track:4:2x1",
             "robust:4:2x1"]
    models = {"align": StackModel, "adapt": AdaptModel, "track": TrackModel, "robust": RobustModel}
    got = []
    for i, spec in enumerate(modes):
        b.set_stack(spec)
        got += _run_stage(ctx, b, frames[8 * i:8 * (i + 1)], w, h, 0.2, bits, 8)
    for i, spec in enumerate(modes):
        g, o = got[8 * i:8 * (i + 1)], off[8 * i:8 * (i + 1)]
        if spec == "off":
            assert all(np.array_equal(x[0].view(np.uint32), y[0].view(np.uint32)) and x[1:] == y[1:] for x, y in zip(g, o)), i
        else:
            _assert_chain(g, o, w, h, models[spec.split(":")[0]](4, 2, 1), f"batch {i}")
    a.reset(); b.reset()
    _assert_chain(_run_stage(ctx, b, frames[:8], w, h, 0.2, bits, 8), _run_stage(ctx, a, frames[:8], w, h, 0.2, bits, 8),
                  w, h, RobustModel(4, 2, 1), "after reset")


# -------------------------------------------------------------------------------------------------- pipeline, host library
def _pipeline_model(off, depth, restarts=()):
    """The robust model over the plain pipeline's frames, restarting at the given frames -> (frames, value-101 sequence at the
    auto-gain report cadence: frames 6, 13, 20, ... of the frame stage)."""
    m = RobustModel(depth)
    outs, values = [], []
    ref, cnt = 0.0, 0
    for k, (o, ww, hh) in enumerate(off):
        if k in restarts:
            m.restart()
        f, r = m.run(o, ww, hh)
        outs.append(f)
        if r["restarted"]:
            ref, cnt = 0.0, 0
        else:
            cnt += 1
        if k % 7 == 6:
            values.append(((r["offset"] - ref) / cnt if cnt else 0.0, r["offset"] % (ww * hh)))
            ref, cnt = r["offset"], 0
    return outs, values


def _assert_pipeline(on, off, depth, restarts=()):
    (g, gv), (o, _) = on, off
    assert len(g) == len(o) > 3
    want, wv = _pipeline_model(o, depth, restarts)
    for k, ((gf, gw, gh), (_, ow, oh)) in enumerate(zip(g, o)):
        assert (gw, gh) == (ow, oh)
        assert np.array_equal(gf.view(np.uint32), want[k].view(np.uint32)), f"frame {k}"
    assert gv == wv


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 16])
def test_pipeline_robust_with_the_pll_on(batch):
    from tests.test_contrast_clahe import _iq_blocks
    blocks = _iq_blocks(40, 61, fv_ppm=2500.0)
    params = {"autoshift": 1, "framerate_pll": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1}
    _assert_pipeline(_pipeline(blocks, "robust:32", params, batch), _pipeline(blocks, "off", params, batch), 32)


@pytest.mark.gpu
def test_pipeline_robust_with_dropped_samples_and_manual_sync():
    """A drop does not restart the stack; tsdr_sync restarts it at the next frame-stage batch (found as the batch starts whose
    output is the plain frame bit for bit: exactly one per sync)."""
    from tests.test_contrast_clahe import _iq_blocks
    blocks = _iq_blocks(30, 22)
    params = {"autoshift": 0, "autocorr_plots_off": 1}
    kw = dict(syncs={12: 37, 20: -5}, dropped={7: 12345})
    on, off = _pipeline(blocks, "robust:8", params, **kw), _pipeline(blocks, "off", params, **kw)
    same = [k for k in range(4, len(on[0]), 4) if np.array_equal(on[0][k][0].view(np.uint32), off[0][k][0].view(np.uint32))]
    assert len(same) == 2, same
    _assert_pipeline(on, off, 8, restarts=same)


@pytest.mark.gpu
def test_pipeline_robust_in_argb_output_mode():
    from oracle import oracle as orc
    from tests.test_contrast_clahe import _iq_blocks
    P = orc.port()
    blocks = _iq_blocks(16, 91)
    params = {"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1}
    floats = _pipeline(blocks, "robust:16", params)
    _assert_pipeline(floats, _pipeline(blocks, "off", params), 16)
    argb, _ = _pipeline(blocks, "robust:16", params, argb=True)
    assert len(argb) == len(floats[0])
    for k, ((g, _, _), (f, _, _)) in enumerate(zip(argb, floats[0])):
        assert np.array_equal(g, P.pixels_argb(f, False)), f"frame {k}"


@pytest.mark.gpu
def test_host_library_with_robust_matches_the_pipeline(monkeypatch, tmp_path):
    """TSDR_STACK=robust:32: tsdr_readasync driven by a RawFile plugin delivers the pipeline's plain frames followed by the
    model, and announces value 101."""
    import threading
    import time
    from oracle import oracle as orc
    from tempestsdr_b200 import synth
    from tests.test_autogain_clip import run_pipeline
    from tests.test_contrast_clahe import SMALL
    from tests.test_host_library import FRAME_CB, MINE, PLOT_CB, VALUE_CB, bind
    fs, h, fv = SMALL
    w, _, _ = orc.port().geometry(fs, h, fv)
    items, nblk = 512 * 1024, 6
    iq = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=41)
    raw = tmp_path / "iq.raw"
    iq.tofile(raw)
    plain, _ = run_pipeline(fs, h, fv, [iq[k * items:(k + 1) * items].copy() for k in range(nblk)], "minmax",
                            {"autoshift": 1, "framerate_pll": 0, "lowpass_before_sync": 1})
    if orc.have_ref():
        plugin, args = orc.REF_RAWFILE_SO, f'"{raw}" {fs} float'
    else:
        plugin, args = os.path.join(os.path.dirname(MINE), "TSDRPlugin_RawFileGPU.so"), f'"{raw}" {fs} float'
    monkeypatch.setenv("TSDR_NO_DROP", "1")
    monkeypatch.setenv("TSDR_STACK", "robust:32")
    got, ids = [], []
    lib = bind(MINE)
    t = C.c_void_p()
    nv, npl = VALUE_CB(lambda vid, a, b, c: ids.append(vid)), PLOT_CB(lambda *a: None)
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
    while len(got) < len(plain) and time.time() < deadline:
        time.sleep(0.05)
    assert lib.tsdr_stop(t) == 0
    th.join(timeout=30)
    assert rc == [0]
    assert len(got) >= len(plain) > 3
    m = RobustModel(32)
    for k, (pv, pw) in enumerate(plain):
        want, _ = m.run(pv, pw, h)
        assert np.array_equal(got[k].view(np.uint32), want.view(np.uint32)), f"frame {k}"
    assert 101 in ids
    lib.tsdr_free(C.byref(t))
