"""The two opt-in FIRs of the sample path, swept over the shapes that change their code paths.

rs_sinc (csrc/resample.cu) cuts every block into tiles of pt pixels (4096, fewer below r = 0.9927), stages each tile's samples
in a shared array of SINC_SCAP floats, reads the history for samples before the run and writes each magnitude from the one tile
that owns it.  The CPU tests restate that geometry (tests/sinc_tiles_model.py) and check its unchecked bounds over a dense grid
of ratios; the GPU tests run the kernel bit for bit against SincModel at every ratio class, at the ratios where those bounds are
tightest, and at block shapes that end a tile short, exactly or one pixel long.

cf_fir (csrc/channel.cu) runs the taps in chunks of CF_K = 9 and a tail chunk of (T - 2) mod 9 + 1 taps whose last tap loads no
sample.  The GPU tests run every tap count from 9 to 257 against tests/channel_filter_model.py bit for bit, every tail length
with signed zeros, subnormals, overflowing products and NaN, and one run past 2^31 floats.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from tempestsdr_b200 import _native as N
from tests import resample_model as rm
from tests import sinc_tiles_model as M
from tests.channel_filter_model import ChannelModel, fir, taps
from tests.test_channel_filter import FOUR_STOPS, gpu_runs, spec_with
from tests.test_sinc_resampler import SincModel, mags

CF_K, CF_P = 9, 2304                       # channel.cu: outputs per thread, per CTA
CF_FS = 2_000_000


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ============================================================================================================== CPU: sinc tiles
def test_tile_size_is_the_library_s():
    """The restated sinc_pixels_per_tile equals the one the resampler launches with, at every grid ratio and either side of
    the lowest accepted ratio."""
    up, down = M.grid()
    r = up / down
    lib = np.array([N.lib().tsdrgpu_sinc_tile_pixels(float(x)) for x in r], np.int64)
    mine = M.pixels_per_tile(r)
    bad = np.flatnonzero(lib != mine)
    assert bad.size == 0, [(float(r[i]), int(mine[i]), int(lib[i])) for i in bad[:5]]
    assert N.lib().tsdrgpu_sinc_tile_pixels(np.nextafter(M.MIN_RATIO, 0.0)) == 0
    assert mine.min() == 256 and mine.max() == M.PT_MAX and M.pixels_per_tile(np.nextafter(M.CAP_RATIO, 0.0)) == M.PT_MAX - 1


def test_sweep_blocks_are_the_host_plan():
    """The vectorised recurrence of sweep_blocks equals tests/resample_model.plan and tsdrgpu_plan_resample, run after run."""
    up, down = M.grid()
    pick = np.unique(np.concatenate([np.arange(0, up.size, 97), [up.size - 1, up.size - 2, up.size - 3]]))
    b = M.sweep_blocks(up[pick], down[pick])
    for k, i in enumerate(pick):
        off, coff = 0.0, C.c_double(0.0)
        for run in range(len(M.RECIPE)):
            sel = (b["ratio"] == k) & (b["run"] == run)
            sizes = b["size"][sel]
            plan, off = rm.plan(off, sizes.tolist(), up[i], down[i])
            assert [p[1] for p in plan] == b["n_out"][sel].tolist()
            assert np.array_equal(np.array([p[3] for p in plan]).view(np.uint64), b["phase"][sel].view(np.uint64))
            assert b["in_start"][sel].tolist() == np.concatenate([[0], np.cumsum(sizes)[:-1]]).tolist()
            desc = (C.c_uint64 * (5 * sizes.size))()
            s32 = sizes.astype(np.uint32)
            N.lib().tsdrgpu_plan_resample(C.byref(coff), s32.ctypes.data_as(C.c_void_p), 0, s32.size, up[i], down[i],
                                          C.cast(desc, C.c_void_p))
            assert [desc[5 * j + 2] >> 32 for j in range(sizes.size)] == b["n_out"][sel].tolist()
            assert coff.value == off


def test_sinc_tile_invariants_hold_over_the_ratio_grid(capsys):
    """For every tile of the sweep: the staged span fits SINC_SCAP, the oldest staged sample lies within the H carried ones,
    the newest tap lies inside the block, the host reserves a descriptor for every tile, and the owned ranges of a block's
    tiles partition [0, size).  Prints the smallest margin of each and where it occurs."""
    up, down = M.grid()
    b, t, margins = M.sweep()
    r = up / down
    lines = [f"sinc tile sweep: {r.size} ratios, {b['size'].size} blocks, {t['n_st'].size} tiles"]
    for name, what in (("scap", "SINC_SCAP - staged span"), ("hist", "in_start + st_lo + H"),
                       ("inside", "size - 1 - newest tap"), ("desc", "descriptors reserved - tiles")):
        i = int(np.argmin(margins[name]))
        lines.append(f"  {what:>28}: smallest {int(margins[name][i]):3d} at r = {float(r[i])!r}")
    with capsys.disabled():
        print("\n" + "\n".join(lines))
    for name in margins:
        assert margins[name].min() >= 0, (name, [float(x) for x in r[margins[name] < 0][:5]])
    # partition: each block's first tile from 0, its last to size, consecutive tiles meeting, none reversed
    blk = t["block"]
    first, last = t["p_lo"] == 0, t["p_hi"] == b["n_out"][blk]
    assert np.all(t["own_lo"][first] == 0) and np.all(t["own_hi"][last] == b["size"][blk[last]])
    same = blk[1:] == blk[:-1]
    assert np.array_equal(first[1:], ~same) and np.all(t["own_hi"][:-1][same] == t["own_lo"][1:][same])
    assert np.all(t["own_lo"] <= t["own_hi"])
    assert np.all(t["st_lo"] <= t["own_lo"]) and np.all(t["own_hi"] <= t["st_hi"])


def test_every_pixel_reads_inside_its_tile():
    """Pixel by pixel at the tightest ratios, 1/16, the cap crossing and every 50th grid ratio: the taps k0 - 7 ... k0 + 8 of
    every pixel lie in its tile's staged span [st_lo, st_hi), and k0 never decreases along a block (which is what lets the
    grid sweep check tiles by their end pixels)."""
    up, down = M.grid()
    r = up / down
    want = [M.MIN_RATIO, M.CAP_RATIO, np.nextafter(M.CAP_RATIO, 0.0)]
    want += [u / d for name in ("scap", "hist", "inside") for u, d in M.tightest(name)]
    pick = np.unique(np.concatenate([np.arange(0, r.size, 50), [int(np.flatnonzero(r == x)[0]) for x in want]]))
    b = M.sweep_blocks(up[pick], down[pick])
    pt = M.pixels_per_tile(b["r"])
    t = M.tiles(b["in_start"], b["size"], b["n_out"], b["r"], b["phase"], pt)
    npx = t["p_hi"] - t["p_lo"]
    tile = np.repeat(np.arange(npx.size), npx)
    p = np.arange(tile.size) - np.repeat(np.cumsum(npx) - npx, npx) + t["p_lo"][tile]
    blk = t["block"][tile]
    k0, j = M.sinc_pos(p, b["phase"][blk], 1.0 / b["r"][blk])
    assert np.all((j >= 0) & (j < M.L))
    assert np.all(k0 - (M.T // 2 - 1) >= t["st_lo"][tile]) and np.all(k0 + M.T // 2 < t["st_hi"][tile])
    along = blk[1:] == blk[:-1]
    assert np.all(np.diff(k0)[along] >= 0)


# ============================================================================================================== GPU
@pytest.fixture(scope="module")
def ctx():
    from tempestsdr_b200 import api
    return api.Context(0)


PAD = 256                                   # NaN floats past every output and magnitude range, zero floats past the input


def sinc_classes():
    """(name, up, down) of every ratio class of the sinc sweep."""
    out = [("1/16", M.MIN_RATIO, 1.0), ("0.1", 0.1, 1.0), ("0.2718", 0.2718, 1.0)]
    out += [(f"scap{k}", u, d) for k, (u, d) in enumerate(M.tightest("scap"))]
    out += [(f"hist{k}", u, d) for k, (u, d) in enumerate(M.tightest("hist"))]
    out += [("cap-1ulp", float(np.nextafter(M.CAP_RATIO, 0.0)), 1.0), ("cap", M.CAP_RATIO, 1.0),
            ("cfg2", 1.99631, 1.0), ("5.3171", 5.3171, 1.0)]
    return out


def _plan_one(off, s, up, down):
    blocks, new = rm.plan(off, [s], up, down)
    return (blocks[0][1] if blocks else 0), new


def exact_blocks(targets, up, down, off, pt):
    """Block sizes whose n_out are exactly `targets` from offset `off`; where no size hits a target, a shim block of 1 ... 1000
    samples first moves the offset to one from which a size does.  Above r = 2 a block yields one of only two pixel counts
    around size * r, so a target may be out of reach at every offset: then the first of target + pt, target + 2 pt, ... that is
    reachable, which ends the block's last tile the same way.  Returns (sizes, offset after them)."""
    r = up / down
    sizes = []
    for n in targets:
        done = False
        for want in range(n, n + 8 * pt, pt):
            for shim in range(0, 1001):
                o = off
                if shim:
                    k, o = _plan_one(off, shim, up, down)
                    if k == 0:
                        continue
                s = int(M._size_for(np.array([float(want)]), np.array([o]), np.array([r]), "lo")[0])
                k, o2 = _plan_one(o, s, up, down)
                if k == want:
                    sizes += ([shim] if shim else []) + [s]
                    off, done = o2, True
                    break
            if done:
                break
        assert done, f"no block of {n} (mod {pt}) pixels at r = {r!r}"
    return sizes, off


def sinc_runs(up, down):
    """The sweep's three runs from offset 0 (the tightest tiles of the grid are among them); then a run of blocks of pt - 1, pt,
    pt + 1, 2 pt and 2 pt + 1 pixels with blocks of 1 sample (or the fewest that yield a pixel) and shorter than H between them;
    then a run shorter than H in total, so the history it carries out mixes the one it read and its own samples; then the
    shaped run again."""
    runs = M.sweep_runs(up, down)
    off = 0.0
    for sizes in runs:
        off = rm.plan(off, sizes, up, down)[1]
    pt = int(M.pixels_per_tile(up / down))
    shaped, off = exact_blocks([pt - 1, pt], up, down, off, pt)
    short = rm.sizes_with_pixels([1, 5, 17, 31], up, down, off)
    off = rm.plan(off, short, up, down)[1]
    more, off = exact_blocks([pt + 1, 2 * pt, 2 * pt + 1], up, down, off, pt)
    runs.append(shaped + short + more)
    tiny = rm.sizes_with_pixels([1, 2, 3], up, down, off)
    while sum(tiny) >= M.H:
        tiny.pop()
    assert tiny and all(s < M.H for s in tiny)
    off = rm.plan(off, tiny, up, down)[1]
    runs.append(tiny)
    again, off = exact_blocks([pt - 1, pt, pt + 1, 2 * pt, 2 * pt + 1], up, down, off, pt)
    runs.append(again)
    return runs


def run_sinc(ctx, x, runs, up, down, iq, offset):
    """Feed the runs to a fresh sinc resampler: input at `offset` floats past a 256-byte boundary, each run's output into a
    NaN-filled buffer, the magnitudes (IQ input) into one NaN-filled buffer for the stream.  Checks that nothing is written past
    a run's pixels or the stream's magnitudes, and returns (pixels per run, magnitudes or None)."""
    import torch
    e = 2 if iq else 1
    dev = torch.zeros(x.size + offset + PAD, dtype=torch.float32, device="cuda")
    dev[offset:offset + x.size] = torch.from_numpy(x)
    total = x.size // e
    mag = torch.full((total + PAD,), float("nan"), dtype=torch.float32, device="cuda") if iq else None
    rs = ctx.resampler()
    rs.set_kernel("sinc")
    outs, pos = [], 0
    for sizes in runs:
        n = int(sum(sizes))
        need = rs.plan(sizes, up, down)
        out = torch.full((need + PAD,), float("nan"), dtype=torch.float32, device="cuda")
        got = rs.process(dev[offset + e * pos: offset + e * (pos + n)], sizes, up, down, in_is_iq=iq, out=out,
                         mag_out=mag[pos:pos + n] if iq else None)
        assert got.numel() == need
        o = out.cpu().numpy()
        assert np.all(np.isnan(o[need:])), "written past the run's pixels"
        outs.append(o[:need])
        pos += n
    m = None
    if iq:
        m = mag.cpu().numpy()
        assert np.all(np.isnan(m[total:])), "written past the stream's magnitudes"
        m = m[:total]
    return outs, m


@pytest.mark.gpu
@pytest.mark.parametrize("name,up,down", sinc_classes(), ids=[c[0] for c in sinc_classes()])
def test_sinc_kernel_matches_the_model_by_ratio_class(ctx, name, up, down):
    import torch
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    runs = sinc_runs(up, down)
    n = sum(sum(s) for s in runs)
    for iq, offset in ((True, 0), (True, 2), (False, 0), (False, 1), (False, 2), (False, 3)):
        x = (rng.standard_normal(2 * n if iq else n) * 3 + (0 if iq else 5)).astype(np.float32)
        got, mag = run_sinc(ctx, x, runs, up, down, iq, offset)
        model, pos = SincModel(), 0
        mg = mags(x) if iq else x
        for k, sizes in enumerate(runs):
            m = int(sum(sizes))
            want = model.run(mg[pos:pos + m], sizes, up, down)
            pos += m
            g = got[k]
            assert g.size == want.size and np.array_equal(_bits(g), _bits(want)), \
                (name, iq, offset, k, int(np.flatnonzero(_bits(g) != _bits(want))[0]) if g.size == want.size else None)
        if iq:
            ref = ctx.am_demod(torch.from_numpy(x).cuda()).cpu().numpy()
            assert not np.any(np.isnan(mag)), (name, offset, "magnitudes never written", np.flatnonzero(np.isnan(mag))[:8])
            assert np.array_equal(_bits(mag), _bits(ref)), (name, offset)


def test_sinc_classes_reach_every_block_shape():
    """The runs of every class contain blocks of pt - 1, pt, pt + 1, 2 pt and 2 pt + 1 pixels (above r = 2 blocks whose last
    tile is one short, exact or one pixel long), blocks of one sample where the ratio allows it, blocks shorter than H and a
    run shorter than H."""
    for name, up, down in sinc_classes():
        runs = sinc_runs(up, down)
        pt = int(M.pixels_per_tile(up / down))
        off, n_outs, sizes = 0.0, [], []
        for s in runs:
            plan, off = rm.plan(off, s, up, down)
            n_outs += [p[1] for p in plan]
            sizes += s
        ends = {n % pt for n in n_outs if n >= pt - 1}
        assert {pt - 1, 0, 1} <= ends, name
        if up / down <= 2.0:
            assert {pt - 1, pt, pt + 1, 2 * pt, 2 * pt + 1} <= set(n_outs), name
        assert min(sizes) < M.H and sum(runs[4]) < M.H, name
        if up / down >= 1.0:
            assert 1 in sizes, name


# ============================================================================================================== GPU: cf_fir
def cf_tail(T):
    """Taps in cf_fir's tail chunk: the whole chunks run while t0 + CF_K < T, from t0 = 1."""
    t0 = 1
    while t0 + CF_K < T:
        t0 += CF_K
    return T - t0


TAIL_TS = sorted({min(T for T in range(9, 258, 2) if cf_tail(T) == k) for k in range(1, CF_K + 1)} |
                 {max(T for T in range(9, 258, 2) if cf_tail(T) == k) for k in range(1, CF_K + 1)})


def _cf(ctx, T):
    cf = ctx.channel_filter()
    cf.set(spec_with(FOUR_STOPS, T), CF_FS)
    m = ChannelModel()
    m.set(spec_with(FOUR_STOPS, T), CF_FS)
    return cf, m


@pytest.mark.gpu
@pytest.mark.parametrize("T", list(range(9, 258, 2)))
def test_cf_fir_matches_the_model_at_every_tap_count(ctx, T):
    """Runs of 1, H - 1, H, H + 1, CF_P - 1, CF_P, CF_P + 1, CF_P + H and 3 CF_P + 7 pairs (H = T - 1), in order with the
    history carried."""
    H = T - 1
    runs = [1, H - 1, H, H + 1, CF_P - 1, CF_P, CF_P + 1, CF_P + H, 3 * CF_P + 7]
    rng = np.random.default_rng(T)
    x = (rng.standard_normal(2 * sum(runs)) * 3).astype(np.float32)
    x[rng.random(x.size) < 0.01] = 0.0
    cf, m = _cf(ctx, T)
    got = gpu_runs(cf, x, runs)
    pos = 0
    for k, n in enumerate(runs):
        want = m.run(x[2 * pos:2 * (pos + n)])
        pos += n
        assert np.array_equal(_bits(got[k]), _bits(want)), (T, cf_tail(T), k, n)


def _same(g, w):
    """Bit for bit, except that a NaN need only be a NaN (x86 and the GPU make different NaN payloads)."""
    gn, wn = np.isnan(g), np.isnan(w)
    return np.array_equal(gn, wn) and np.array_equal(_bits(g)[~gn], _bits(w)[~wn])


def special_parts(T):
    """The special-value runs for T taps: (runs as interleaved float32, outputs of run 0 that must be -0 as (pair, 0 = I /
    1 = Q), NaN input pairs of run 2).  In run 0 every sample is +-0, and before each listed output its T samples carry the
    signs that make every one of its T products -0 in that component (I: sign(I) = not sign(hr_t), sign(Q) = sign(hi_t);
    Q: sign(I) = not sign(hi_t), sign(Q) = not sign(hr_t)), so the output is -0 only if the sum starts from the first product."""
    h = taps(spec_with(FOUR_STOPS, T), CF_FS)
    shr, shi = np.signbit(h.real), np.signbit(h.imag)
    rng = np.random.default_rng(1000 + T)
    n0 = CF_P + 3 * T + 5
    sa, sb = rng.random(n0) < 0.5, rng.random(n0) < 0.5
    neg = []
    for k, n in enumerate(range(T - 1, n0, T)):
        w = n - np.arange(T)
        if k % 2 == 0:
            sa[w], sb[w] = ~shr, shi
        else:
            sa[w], sb[w] = ~shi, ~shr
        neg.append((n, k % 2))
    zeros = np.zeros(2 * n0, np.float32)
    zeros[0::2][sa] = -0.0
    zeros[1::2][sb] = -0.0
    sub = (rng.integers(1, 1 << 23, 2 * n0, dtype=np.uint32) | (rng.integers(0, 2, 2 * n0, dtype=np.uint32) << 31)).view(np.float32)
    nan_run = (rng.standard_normal(2 * (2 * CF_P + 11)) * 3).astype(np.float32)
    nan_at = [CF_P - 3, nan_run.size // 2 - 1]
    nan_run[2 * nan_at[0]] = np.nan
    nan_run[2 * nan_at[1] + 1] = np.nan
    after = (rng.standard_normal(2 * (CF_P + 3)) * 3).astype(np.float32)
    huge = (np.float32(3.4e38) * rng.uniform(0.9, 1.0, 2 * n0) * np.where(rng.random(2 * n0) < 0.5, -1, 1)).astype(np.float32)
    return [zeros, sub, nan_run, after, huge], neg, nan_at


@pytest.mark.gpu
@pytest.mark.parametrize("T", TAIL_TS)
def test_cf_fir_special_values_at_every_tail_length(ctx, T):
    """In order, history carried: all +-0, with outputs whose every product is -0 (the t = 0 step sets the sums, so they
    stay -0); subnormal samples; ordinary samples with a NaN pair straddling a tile edge and a NaN as the last pair (it reaches
    the next run through the history); ordinary samples; samples near FLT_MAX whose sums overflow.  A NaN input shows up in
    exactly the T outputs that read it."""
    H = T - 1
    parts, neg, nan_at = special_parts(T)
    x = np.concatenate(parts)
    runs = [p.size // 2 for p in parts]
    cf, m = _cf(ctx, T)
    got = gpu_runs(cf, x, runs)
    want = [m.run(p) for p in parts]
    for k, (g, w) in enumerate(zip(got, want)):
        assert _same(g, w), (T, cf_tail(T), k)
    assert all(_bits(got[0])[2 * n + c] == 0x80000000 for n, c in neg), T
    sb = _bits(got[1])
    assert np.any(((sb & 0x7F800000) == 0) & ((sb & 0x7FFFFF) != 0)) and np.any(np.isinf(got[4]))      # subnormal out, overflow
    # the NaNs: outputs nan_at[0] .. nan_at[0] + T - 1 of the run, its last output, and the first T - 1 outputs of the next
    bad = np.isnan(got[2][0::2]) | np.isnan(got[2][1::2])
    expect = np.zeros(bad.size, bool)
    expect[nan_at[0]:nan_at[0] + T] = True
    expect[nan_at[1]] = True
    assert np.array_equal(bad, expect), T
    assert np.all(np.isnan(got[2][0::2]) == bad) and np.all(np.isnan(got[2][1::2]) == bad)
    bad = np.isnan(got[3][0::2]) | np.isnan(got[3][1::2])
    assert np.array_equal(np.flatnonzero(bad), np.arange(H)), T


@pytest.mark.gpu
def test_cf_fir_run_past_2_31_floats(ctx):
    """One run of 2^30 + 5 pairs at T = 257, so the float index passes 2^31: the CTA tile that holds pair 2^30 - 1 and the last
    10 000 pairs against the model over their own windows (fed the T - 1 pairs before them as history), then a short run that
    reads its history from the end of the long one."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip(f"needs 24 GB of free device memory, {free / 2**30:.1f} GB free")
    T, n = 257, (1 << 30) + 5
    H = T - 1
    cf, _ = _cf(ctx, T)
    h = taps(spec_with(FOUR_STOPS, T), CF_FS)
    g = torch.Generator(device="cuda")
    g.manual_seed(257)
    x = torch.randn(2 * n, generator=g, dtype=torch.float32, device="cuda")
    out = torch.full((2 * n,), float("nan"), dtype=torch.float32, device="cuda")
    cf.run(x, out=out)
    torch.cuda.synchronize()
    tile0 = ((1 << 30) - 1) // CF_P * CF_P
    w0 = min(tile0, n - 10_000)
    xs = x[2 * (w0 - H):].cpu().numpy()
    got = out[2 * w0:].cpu().numpy()
    tail = torch.randn(2 * 7, generator=g, dtype=torch.float32, device="cuda")
    tail_out = cf.run(tail)
    torch.cuda.synchronize()
    tail_got, tail_x = tail_out.cpu().numpy(), tail.cpu().numpy()
    del x, out
    torch.cuda.empty_cache()
    want, hist = fir(xs[2 * H:], h, xs[:2 * H].view(np.complex64))
    assert np.array_equal(_bits(got), _bits(want))
    assert np.array_equal(_bits(tail_got), _bits(fir(tail_x, h, hist)[0]))
