"""Richardson-Lucy deconvolution along the lines, the deblur step (include/tsdrgpu.h): the numpy model of tests/deblur_model.py
checked against the literal definition and for the quality it buys on stacked frames, then the GPU stage, the frame stage, the
pipeline and the host library held bit for bit to (the same run without deblur) followed by the model."""
import ctypes as C
import math
import os
import threading
import time

import numpy as np
import pytest

from tests.deblur_model import deblur_frame, deblur_literal, deblur_taps, radius, taps_reference, valid_mask

F32 = np.float32
ADVERSARIAL = np.array((256.0, 512.0, 1024.0, -300.0, np.inf, -np.inf, np.nan, 0.0, -0.0, 1.0, 3.5, -1.5, 249.0), F32)
SPAN = 6144                     # enhance.cu's DB_SPAN: longer lines are cut into segments of SPAN - 4 R I with a halo of 2 R I


def _frame(w, h, rng, adversarial=True):
    """Blocky rows in [-0.2, 1.2] with one-pixel strokes and, optionally, markers, NaN, +-inf, +-0 and out-of-range values."""
    n = w * h
    f = np.repeat(rng.uniform(-0.2, 1.2, (n + 2) // 3), 3)[:n].astype(F32)
    f[rng.integers(0, n, max(1, n // 20))] = F32(1.0)
    if adversarial:
        k = max(1, n // 25)
        f[rng.integers(0, n, k)] = rng.choice(ADVERSARIAL, k)
    return f


# ============================================================================================================== CPU
def test_taps_match_an_independent_float64_gaussian():
    for sc in [25, 26, 33, 34, 50, 66, 67, 99, 100, 101, 125, 150, 200, 233, 333, 334, 399, 400]:
        k = deblur_taps(sc)
        r = radius(sc)
        assert r == math.ceil(3 * sc / 100 - 1e-12) and len(k) == 2 * r + 1, sc
        s = sc / 100.0
        e = np.array([math.exp(-(j * j) / (2 * s * s)) for j in range(-r, r + 1)])
        ref = e / e.sum()
        assert np.all(np.abs(k.astype(np.float64) - ref) <= 1e-7 * ref), sc
        assert np.array_equal(k, taps_reference(sc)), sc
        assert np.array_equal(k, k[::-1]), sc
    from tempestsdr_b200 import _native as N
    lib, r = N.lib(), C.c_int(-1)
    assert lib.tsdrgpu_deblur_taps(100, None, C.byref(r)) == 0 and r.value == 3
    for sc in (0, 24, 401, -100):
        assert lib.tsdrgpu_deblur_taps(sc, None, None) == -3, sc


SIZES = [(1, 1), (1, 5), (2, 3), (5, 2), (9, 2), (25, 2), (31, 1)]


@pytest.mark.parametrize("sc", [25, 100, 400])
@pytest.mark.parametrize("iters", [1, 20, 64])
def test_model_equals_the_literal_definition(sc, iters):
    """Lines shorter than the kernel, 1 x 1, W = 2R + 1, markers, NaN, +-inf and out-of-range values."""
    rng = np.random.default_rng(sc + iters)
    r = radius(sc)
    for w, h in SIZES + [(2 * r + 1, 2)]:
        f = _frame(w, h, rng)
        a, b = deblur_frame(f, w, h, sc, iters), deblur_literal(f, w, h, sc, iters)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (w, h)


def test_invalid_pixels_pass_through_and_valid_outputs_lie_in_0_1():
    rng = np.random.default_rng(2)
    w, h = 97, 13
    f = _frame(w, h, rng)
    f[:4] = np.array([256.0, np.nan, -np.inf, np.inf], F32)
    bad = ~valid_mask(f)
    for sc, it in ((25, 1), (100, 20), (400, 64), (150, 40)):
        g = deblur_frame(f, w, h, sc, it)
        assert np.array_equal(g.view(np.uint32)[bad], f.view(np.uint32)[bad]), (sc, it)
        assert np.all((g[~bad] >= 0) & (g[~bad] <= 1)), (sc, it)
        assert not np.any(np.signbit(g[~bad])), (sc, it)


def test_a_constant_line_stays_itself():
    """Constant valid lines, ends included: within 1e-5 relative of the constant after up to 64 iterations (float32 rounding
    only; the model shows at most 7.3e-6 relative here), and 0 stays 0."""
    for c in (0.0, 0.001, 0.25, 0.5, 0.9, 1.0):
        for sc, it in ((25, 64), (100, 20), (100, 64), (400, 64)):
            g = deblur_frame(np.full(3 * 40, F32(c)), 40, 3, sc, it)
            assert np.max(np.abs(g.astype(np.float64) - F32(c))) <= 1e-5 * c, (c, sc, it)


def test_pixels_beyond_the_reach_are_unaffected():
    """A valid pixel further than 2 R I from every invalid pixel and line end keeps its bits when they change."""
    rng = np.random.default_rng(4)
    for sc, it in ((50, 3), (100, 5), (125, 2)):
        reach = 2 * radius(sc) * it
        core = rng.uniform(0, 1, 2 * reach + 1).astype(F32)
        mid = reach
        base = deblur_frame(core, core.size, 1, sc, it)[mid]
        for left, right in ((5, 0), (0, 9), (17, 3)):
            line = np.concatenate([rng.uniform(-1, 2, left), core, rng.uniform(-1, 2, right)]).astype(F32)
            line[rng.integers(0, line.size, 4)] = F32(512.0)
            line[left:left + core.size] = core
            g = deblur_frame(line, line.size, 1, sc, it)
            assert g.view(np.uint32)[left + mid] == base.view(np.uint32), (sc, it, left, right)


DEBLUR_SPECS_OK = {"off": (0, 0, 0), "rl:1": (1, 100, 20), "rl:0.25": (1, 25, 20), "rl:4": (1, 400, 20), "rl:4.0": (1, 400, 20),
                   "rl:4.00": (1, 400, 20), "rl:1.5": (1, 150, 20), "rl:1.25:40": (1, 125, 40), "rl:0.3:1": (1, 30, 1),
                   "rl:2:64": (1, 200, 64), "rl:01.00:020": (1, 100, 20), "rl:0.82": (1, 82, 20)}
DEBLUR_SPECS_BAD = ["rl:0.24", "rl:0.2", "rl:4.01", "rl:5", "rl:0", "rl:1.255", "rl:1:0", "rl:1:65", "rl:1:", "rl:1:-1", "rl:+1",
                    "rl:-1", "rl: 1", "rl:1 ", " rl:1", "rl:", "rl", "rl:.5", "rl:1.", "rl:1e0", "rl:1,5", "RL:1", "OFF", "off ", "",
                    " ", "rl:1:20:1", "rl:1x20", "nlm:0.1", "rl:9999999", "rl:1:9999999", "rl:1.5:2.5"]


def test_deblur_spec_parsing():
    """tsdrgpu_deblur_parse, which the host library's TSDR_DEBLUR and Python's deblur= / set_deblur both use."""
    from tempestsdr_b200 import _native as N
    lib = N.lib()
    for spec, want in DEBLUR_SPECS_OK.items():
        assert N.deblur_mode(spec) == want, spec
        out = [C.c_int(-7) for _ in range(3)]
        assert lib.tsdrgpu_deblur_parse(spec.encode(), *[C.byref(o) for o in out]) == 0, spec
        assert tuple(o.value for o in out) == want, spec
    for spec in DEBLUR_SPECS_BAD:
        out = [C.c_int(-7) for _ in range(3)]
        assert lib.tsdrgpu_deblur_parse(spec.encode(), *[C.byref(o) for o in out]) == -3, spec
        assert [o.value for o in out] == [-7] * 3, spec
        with pytest.raises(ValueError):
            N.deblur_mode(spec)


@pytest.mark.parametrize("value", ["rl:0.2", "rl:1:65", "on", "rl:+1", ""])
def test_bogus_deblur_setting_is_refused_by_the_host_library(tmp_path, monkeypatch, value):
    """TSDR_DEBLUR other than "off" / "rl:<sigma>[:<I>]": tsdr_readasync fails with TSDR_INVALID_PARAMETER_VALUE before touching
    the GPU, and the error text names the variable."""
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
    monkeypatch.setenv("TSDR_DEBLUR", value)
    assert lib.tsdr_readasync(t, FRAME_CB(lambda *a: None), None) == 9          # TSDR_INVALID_PARAMETER_VALUE
    assert b"TSDR_DEBLUR" in lib.tsdr_getlasterrortext(t)
    assert lib.tsdr_isrunning(t) == 0
    lib.tsdr_free(C.byref(t))


# -------------------------------------------------------------------------------------------------- quality
def _picture(w, h, rng):
    """The stack's quality picture: blocky in [0.1, 0.9] with one-pixel strokes (w x h, float64, flattened)."""
    ty, tx = (h + 3) // 4, (w + 3) // 4
    img = np.kron(rng.uniform(0.1, 0.9, size=(ty, tx)), np.ones((4, 4)))[:h, :w]
    img[:, rng.integers(0, w, max(1, w // 12))] = 1.0
    return img.reshape(-1)


def _front_end(pic, d, r, phi):
    """The truth moved by d px along the raster, seen through a front end that blurs: each sample integrates it over its period
    of r px (sample s covers [phi + s r, phi + (s + 1) r)) and the box resampler holds the sample on the pixels whose centres
    fall in that period."""
    n = pic.size
    cs = np.concatenate([[0.0], np.cumsum(pic)])

    def integral(t):                                     # of the periodic, pixel-wise constant truth from 0 to t
        return np.floor(t / n) * cs[-1] + np.interp(np.mod(t, n), np.arange(n + 1), cs)

    a = np.floor((np.arange(n) + 0.5 - phi) / r) * r + phi
    return (integral(a + r - d) - integral(a - d)) / r


def _psnr(x, ref):
    return 10.0 * np.log10(1.0 / np.mean((np.asarray(x, np.float64) - ref) ** 2))


def test_deblur_gain_on_stacked_frames():
    """256 x 128 frames of the stack's quality picture through a blurring front end (r = 1.998, sampling phase drawn anew per
    frame), drifting 0.37 px/frame, sigma = 0.2 noise; the stack at depth 32, then rl:1 (the defaults, I = 20).  PSNR against the
    truth at the integer position the stack delivers.  Measured with the model at frame 63: stacked 18.3 dB, deblurred +1.21 dB
    (seed 1) and +1.11 dB (seed 2); rl:0.75 gives +0.87.  On a single frame deblur loses: 12.2 dB, -1.4 dB at rl:1:10 and
    -2.2 dB at rl:1."""
    from tests.stack_model import StackModel
    w, h, F, r = 256, 128, 64, 1.998
    for seed in (1, 2):
        rng = np.random.default_rng(seed)
        pic = _picture(w, h, rng)
        phis = rng.uniform(0, r, F)
        frames = [(_front_end(pic, 0.37 * k, r, phis[k]) + rng.normal(0, 0.2, w * h)).astype(F32) for k in range(F)]
        outs, recs = StackModel(32).run_many(frames, w, h)
        k = F - 1
        target = np.roll(pic, int(math.floor(recs[k]["offset"] + 0.5)))
        stacked = _psnr(outs[k], target)
        gain = _psnr(deblur_frame(outs[k], w, h, 100, 20), target) - stacked
        assert gain >= 0.8, (seed, stacked, gain)
        single = _psnr(frames[k], np.roll(pic, int(math.floor(0.37 * k + 0.5))))
        sgain = _psnr(deblur_frame(frames[k], w, h, 100, 20), np.roll(pic, int(math.floor(0.37 * k + 0.5)))) - single
        assert sgain < 0 < gain, (seed, single, sgain)


# ============================================================================================================== GPU
def _ctx():
    from tempestsdr_b200 import api
    return api.Context(0)


def _gpu_case(ctx, distinct, w, h, sc, it, F, pin, pout, c=0, want1=None):
    """F frames cycled from `distinct` through Context.deblur, input at 16-byte phase pin, output at pout; compared to the model."""
    import torch
    nd = len(distinct)
    want1 = want1 or [deblur_frame(f, w, h, sc, it) for f in distinct]
    src = np.concatenate([distinct[(k + c) % nd] for k in range(F)])
    want = np.concatenate([want1[(k + c) % nd] for k in range(F)])
    buf = torch.full((pin + src.size + 4,), float("nan"), device="cuda")
    buf[pin:pin + src.size] = torch.from_numpy(src).cuda()
    view = buf[pin:pin + src.size]
    obuf = torch.zeros(pout + src.size + 4, device="cuda")
    assert (view.data_ptr() - 4 * pin) % 16 == 0 and obuf.data_ptr() % 16 == 0
    g = ctx.deblur(view, w, h, f"rl:{sc // 100}.{sc % 100:02d}:{it}", out=obuf[pout:pout + src.size]).cpu().numpy()
    assert obuf[:pout].abs().sum().item() == 0 and obuf[pout + src.size:].abs().sum().item() == 0
    assert np.array_equal(view.cpu().numpy().view(np.uint32), src.view(np.uint32)), "input untouched"
    bad = np.flatnonzero(g.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (w, h, sc, it, F, pin, pout, bad[:5], g[bad[:5]], want[bad[:5]])


SETTINGS = [(25, 1), (100, 20), (400, 64), (82, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(1, 1), (7, 1125), (3, 2), (13, 9), (507, 525), (740, 1125), (1481, 1125)])
def test_tsdrgpu_deblur_bit_exact_against_the_model(w, h):
    """Every setting of SETTINGS at this size, F cycling through 1 / 17 / 64 (fewer at the large sizes) and the 16-byte phases."""
    ctx = _ctx()
    rng = np.random.default_rng(w * 10007 + h)
    big = w * h > 100000
    distinct = [_frame(w, h, rng) for _ in range(2 if big else 3)]
    for c, (sc, it) in enumerate(SETTINGS):
        F = (1, 2, 3, 2)[c] if big else (1, 17, 64, 5)[c]
        _gpu_case(ctx, distinct, w, h, sc, it, F, (c + w) % 4, (c + h) % 4, c)


@pytest.mark.gpu
def test_tsdrgpu_deblur_all_phase_pairs():
    ctx = _ctx()
    rng = np.random.default_rng(9)
    w, h = 37, 11
    distinct = [_frame(w, h, rng) for _ in range(3)]
    want1 = [deblur_frame(f, w, h, 100, 20) for f in distinct]
    for pin in range(4):
        for pout in range(4):
            _gpu_case(ctx, distinct, w, h, 100, 20, 17, pin, pout, pin + pout, want1)


@pytest.mark.gpu
@pytest.mark.parametrize("sc,it", [(100, 20), (400, 64)])
def test_tsdrgpu_deblur_around_the_segment_length(sc, it):
    """Lines of SPAN - 1, SPAN (whole) and SPAN + 1 (cut), and 2 seg + 2 halo + 1, seg = SPAN - 4 R I, so that a middle segment
    has its full halo on both sides; markers near the cuts."""
    ctx = _ctx()
    r = radius(sc)
    halo, seg = 2 * r * it, SPAN - 4 * r * it
    rng = np.random.default_rng(sc + it)
    for c, w in enumerate((SPAN - 1, SPAN, SPAN + 1, 2 * seg + 2 * halo + 1, 3 * seg + 5)):
        h = 3
        f = _frame(w, h, rng)
        for cut in (seg, 2 * seg):
            if cut < w:
                f[cut - 1:cut + 2] = F32(512.0) if c % 2 else f[cut - 1:cut + 2]
        _gpu_case(ctx, [f], w, h, sc, it, 2, c % 4, (c + 1) % 4)


@pytest.mark.gpu
def test_tsdrgpu_deblur_wide_frames():
    """16666 x 525, 4000 x 4000 and one 16 000 000 x 1 line, a few frames, small sigma and I to keep the model quick."""
    ctx = _ctx()
    rng = np.random.default_rng(16666)
    _gpu_case(ctx, [_frame(16666, 525, rng)], 16666, 525, 100, 4, 2, 1, 2)
    _gpu_case(ctx, [_frame(4000, 4000, rng)], 4000, 4000, 50, 2, 2, 3, 0)
    _gpu_case(ctx, [_frame(16_000_000, 1, rng)], 16_000_000, 1, 25, 2, 1, 2, 1)


@pytest.mark.gpu
def test_tsdrgpu_deblur_refuses_overlap_and_bad_arguments():
    import torch
    from tempestsdr_b200 import _native as N
    ctx = _ctx()
    lib = N.lib()
    w, h, F = 33, 29, 3
    n = w * h * F
    x = torch.zeros(2 * n + 64, device="cuda")
    p0 = x.data_ptr()
    for src, dst in ((p0, p0), (p0, p0 + 4), (p0, p0 + 4 * (n - 1)), (p0 + 4 * (n - 1), p0), (p0 + 4 * 32, p0 + 4 * 31)):
        assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, src, dst, w, h, F, 100, 20) == -3, (src - p0, dst - p0)
    assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, p0, p0 + 4 * n, w, h, F, 100, 20) == 0          # adjacent, no overlap
    assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, p0 + 4 * n, p0, w, h, F, 100, 20) == 0
    out = torch.zeros(n, device="cuda")
    for args in ((w, h, F, 24, 20), (w, h, F, 401, 20), (w, h, F, 100, 0), (w, h, F, 100, 65), (0, h, F, 100, 20),
                 (w, 0, F, 100, 20), (w, h, -1, 100, 20), (4001, 4000, 1, 100, 20), (16_000_001, 1, 1, 100, 20)):
        assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, p0, out.data_ptr(), *args) == -3, args
    assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, p0 + 2, out.data_ptr(), w, h, 1, 100, 20) == -3
    assert lib.tsdrgpu_deblur(ctx._h, ctx.stream, p0, out.data_ptr(), w, h, F, 100, 20) == 0
    pg = ctx.post_processor()
    assert lib.tsdrgpu_framestage_set_deblur(pg._h, 2, 100, 20) == -3
    assert lib.tsdrgpu_framestage_set_deblur(pg._h, 1, 401, 20) == -3
    assert lib.tsdrgpu_framestage_set_deblur(pg._h, 1, 100, 65) == -3
    assert lib.tsdrgpu_framestage_set_deblur(pg._h, 0, 0, 0) == 0
    with pytest.raises(ValueError):
        ctx.deblur(x, w, h, "off")


# -------------------------------------------------------------------------------------------------- frame stage
def _chain(off, w, h, db, stack=None, nl=None, ct=None):
    """The models in the enhancement chain's order: stack -> deblur -> NLM -> CLAHE, over the plain frames in order."""
    from tests.clahe_model import clahe_frame
    from tests.nlm_model import nlm_frame
    out = []
    for f in off:
        x = stack.run(f, w, h)[0] if stack else f
        x = deblur_frame(x, w, h, *db)
        if nl:
            x = nlm_frame(x, w, h, *nl)
        if ct:
            x = clahe_frame(x, w, h, *ct)
        out.append(x)
    return out


def _assert_chain(on, off, w, h, db, what, **kw):
    """on == off followed by the chain of models: frames bit for bit, result structs and reports identical."""
    assert len(on) == len(off) > 0
    want = _chain([o[0] for o in off], w, h, db, **kw)
    for k, ((gf, gr, ga), (_, orr, oa), wf) in enumerate(zip(on, off, want)):
        assert np.array_equal(gf.view(np.uint32), wf.view(np.uint32)), f"{what} frame {k}"
        assert gr == orr and ga == oa, f"{what} results {k}"


FLAGS = [(a, l, g, s) for a in (0, 1) for l in (0, 1) for g in (0, 1) for s in (0, 1)]   # autoshift, lp before sync, aap, super-res


@pytest.mark.gpu
@pytest.mark.parametrize("autoshift,lpbs,aap,superres", FLAGS)
@pytest.mark.parametrize("overlap", [0, 1])
def test_frame_stage_deblur_is_the_plain_run_followed_by_the_model(autoshift, lpbs, aap, superres, overlap):
    """Every flag combination, motion blur 0.3, overlap off and on, two batches of 17 frames; in every other case the stack,
    NLM and CLAHE are on as well, and the result is the chain of their models in the order stack -> deblur -> NLM -> CLAHE."""
    from oracle import oracle as orc
    from tempestsdr_b200 import _native as N
    from tests.stack_model import StackModel
    from tests.test_contrast_clahe import _run_stage, _stream
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = orc.port().geometry(fs, h, fv)
    frames = _stream(w, h, 34, 2300 + 8 * autoshift + 4 * lpbs + 2 * aap + superres)
    bits = (N.FS_AUTOSHIFT * autoshift | N.FS_LOWPASS_BEFORE_SYNC * lpbs | N.FS_AUTOGAIN_AFTER_PROC * aap
            | N.FS_SUPERRESOLUTION * superres)
    full = (autoshift + lpbs + aap + superres + overlap) % 2 == 1
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    for pg in (a, b):
        pg.set_overlap(bool(overlap))
    b.set_deblur("rl:1.1:12")
    if full:
        b.set_stack("align:8")
        b.set_denoise("nlm:0.15:3:1")
        b.set_contrast("clahe:2.5:8x8")
    off = _run_stage(ctx, a, frames, w, h, 0.3, bits, 17)
    on = _run_stage(ctx, b, frames, w, h, 0.3, bits, 17)
    kw = dict(stack=StackModel(8), nl=(150, 3, 1), ct=(250, 8, 8)) if full else {}
    _assert_chain(on, off, w, h, (110, 12), f"flags {autoshift}{lpbs}{aap}{superres} overlap {overlap}", **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg5", "cfg1"])
def test_frame_stage_deblur_at_bench_shapes(name):
    """F = 64 at the benchmark's geometries and default flags with the side-stream overlap on, two batches, the defaults."""
    from oracle import oracle as orc
    from tempestsdr_b200 import _native as N
    from tests.test_contrast_clahe import _run_stage, _stream
    from tests.test_gpu_parity import CFGS
    fs, h, fv = CFGS[name]
    w, _, _ = orc.port().geometry(fs, h, fv)
    frames = _stream(w, h, 128, 2500)
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    for pg in (a, b):
        pg.set_overlap(True)
    b.set_deblur("rl:1")
    bits = N.FS_AUTOSHIFT | N.FS_LOWPASS_BEFORE_SYNC
    off = _run_stage(ctx, a, frames, w, h, 0.0, bits, 64)
    on = _run_stage(ctx, b, frames, w, h, 0.0, bits, 64)
    sel = [0, 37, 63, 64, 127]
    _assert_chain([on[k] for k in sel], [off[k] for k in sel], w, h, (100, 20), name)
    assert all(on[k][1] == off[k][1] and on[k][2] == off[k][2] for k in range(128))


@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [0, 1])
def test_switching_deblur_batch_by_batch_leaves_the_off_batches_alone(overlap):
    """Deblur on, off, on, off, ... per batch of 8 (and a reset in between, which keeps the mode): the off batches equal a run
    that never switched, the on batches equal that run followed by the model."""
    from oracle import oracle as orc
    from tempestsdr_b200 import _native as N
    from tests.test_contrast_clahe import _run_stage, _stream
    fs, h, fv = 2_000_000, 125, 60.0
    w, _, _ = orc.port().geometry(fs, h, fv)
    frames = _stream(w, h, 48, 2700)
    bits = N.FS_AUTOSHIFT | N.FS_LOWPASS_BEFORE_SYNC
    ctx = _ctx()
    a, b = ctx.post_processor(), ctx.post_processor()
    for pg in (a, b):
        pg.set_overlap(bool(overlap))
    off = _run_stage(ctx, a, frames, w, h, 0.2, bits, 8)
    got = []
    for i in range(6):
        b.set_deblur("rl:0.9:15" if i % 2 == 0 else "off")
        got += _run_stage(ctx, b, frames[8 * i:8 * (i + 1)], w, h, 0.2, bits, 8)
    for i in range(6):
        g, o = got[8 * i:8 * (i + 1)], off[8 * i:8 * (i + 1)]
        if i % 2 == 0:
            _assert_chain(g, o, w, h, (90, 15), f"batch {i}")
        else:
            assert all(np.array_equal(x[0].view(np.uint32), y[0].view(np.uint32)) and x[1:] == y[1:] for x, y in zip(g, o)), i
    b.set_deblur("rl:2:3")
    a.reset(); b.reset()
    _assert_chain(_run_stage(ctx, b, frames[:8], w, h, 0.2, bits, 8), _run_stage(ctx, a, frames[:8], w, h, 0.2, bits, 8),
                  w, h, (200, 3), "after reset")


# -------------------------------------------------------------------------------------------------- pipeline, host library
def _pipeline(blocks, deblur, params, stack="off", syncs=None, dropped=None, argb=False, batch_frames=4):
    from tempestsdr_b200 import pipeline
    from tests.test_contrast_clahe import SMALL
    fs, h, fv = SMALL
    got = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=batch_frames, batch_blocks=40,
                          block_when_busy=True, params=params, deblur=deblur, stack=stack,
                          on_frame=lambda f, ww, hh: got.append((f.view(np.int32 if argb else np.float32).copy(), ww, hh)))
    if argb:
        p.set_output_argb(True, False)
    for k, b in enumerate(blocks):
        p.process(b, (dropped or {}).get(k, 0))
        if syncs and k in syncs:
            p.sync(syncs[k])
    p.flush()
    p.close()
    return got


def _assert_pipeline(on, off, db):
    assert len(on) == len(off) > 3
    for k, ((g, gw, gh), (o, ow, oh)) in enumerate(zip(on, off)):
        assert (gw, gh) == (ow, oh)
        want = deblur_frame(o, ow, oh, *db)
        assert np.array_equal(g.view(np.uint32), want.view(np.uint32)), f"frame {k}"


@pytest.mark.gpu
@pytest.mark.parametrize("batch_frames", [1, 16])
def test_pipeline_deblur_with_the_pll_on(batch_frames):
    from tests.test_contrast_clahe import _iq_blocks
    blocks = _iq_blocks(24, 63, fv_ppm=2500.0)
    params = {"autoshift": 1, "framerate_pll": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1}
    _assert_pipeline(_pipeline(blocks, "rl:1", params, batch_frames=batch_frames),
                     _pipeline(blocks, "off", params, batch_frames=batch_frames), (100, 20))


@pytest.mark.gpu
def test_pipeline_stack_and_deblur_with_dropped_samples_and_manual_sync():
    """The stack on and restarted by tsdr_sync, with drops: deblur on equals the same run with deblur off followed by the
    model, since deblur comes after the stack and feeds nothing back."""
    from tests.test_contrast_clahe import _iq_blocks
    blocks = _iq_blocks(30, 24)
    params = {"autoshift": 0, "autocorr_plots_off": 1}
    kw = dict(syncs={12: 37, 20: -5}, dropped={7: 12345})
    stacked = _pipeline(blocks, "off", params, stack="align:8", **kw)
    both = _pipeline(blocks, "rl:1.25:10", params, stack="align:8", **kw)
    _assert_pipeline(both, stacked, (125, 10))


@pytest.mark.gpu
def test_pipeline_deblur_in_argb_output_mode():
    """ARGB pixels of the deblurred frames: the glue's pixel rule (oracle port) applied to the float run with deblur on."""
    from oracle import oracle as orc
    from tests.test_contrast_clahe import _iq_blocks
    P = orc.port()
    blocks = _iq_blocks(16, 93)
    params = {"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1}
    floats = _pipeline(blocks, "rl:1", params)
    _assert_pipeline(floats, _pipeline(blocks, "off", params), (100, 20))
    argb = _pipeline(blocks, "rl:1", params, argb=True)
    assert len(argb) == len(floats)
    for k, ((g, _, _), (f, _, _)) in enumerate(zip(argb, floats)):
        assert np.array_equal(g, P.pixels_argb(f, False)), f"frame {k}"


@pytest.mark.gpu
def test_host_library_with_deblur_matches_the_pipeline(tmp_path, monkeypatch):
    """TSDR_DEBLUR=rl:1: tsdr_readasync driven by a RawFile plugin delivers the pipeline's plain frames followed by the model."""
    from oracle import oracle as orc
    from tempestsdr_b200 import synth
    from tests.test_autogain_clip import run_pipeline
    from tests.test_contrast_clahe import SMALL
    from tests.test_host_library import FRAME_CB, MINE, PLOT_CB, VALUE_CB, bind
    fs, h, fv = SMALL
    w, _, _ = orc.port().geometry(fs, h, fv)
    items, nblk = 512 * 1024, 6
    iq = synth.video_like_iq(nblk * items // 2, fs, w, h, fv, seed=33)
    raw = tmp_path / "iq.raw"
    iq.tofile(raw)
    plain, _ = run_pipeline(fs, h, fv, [iq[k * items:(k + 1) * items].copy() for k in range(nblk)], "minmax",
                            {"autoshift": 1, "framerate_pll": 0, "lowpass_before_sync": 1})
    if orc.have_ref():
        plugin, args = orc.REF_RAWFILE_SO, f'"{raw}" {fs} float'
    else:
        plugin, args = os.path.join(os.path.dirname(MINE), "TSDRPlugin_RawFileGPU.so"), f'"{raw}" {fs} float'
    monkeypatch.setenv("TSDR_NO_DROP", "1")
    monkeypatch.setenv("TSDR_DEBLUR", "rl:1")
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
    while len(got) < len(plain) and time.time() < deadline:
        time.sleep(0.05)
    assert lib.tsdr_stop(t) == 0
    th.join(timeout=30)
    assert rc == [0]
    assert len(got) >= len(plain) > 3
    for k, (pv, pw) in enumerate(plain):
        want = deblur_frame(pv, pw, h, 100, 20)
        assert np.array_equal(got[k].view(np.uint32), want.view(np.uint32)), f"frame {k}"
    lib.tsdr_free(C.byref(t))
