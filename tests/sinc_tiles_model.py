"""rs_sinc's tile geometry (tempestsdr_b200/csrc/resample.cu) restated in float64 numpy.  TEST INFRASTRUCTURE ONLY.

A sinc run cuts every block into tiles of `pt` consecutive pixels, one CTA each.  A tile stages the magnitudes its taps read in a
shared array of SINC_SCAP floats, reading the carried history where the sample index is negative, and writes the magnitudes it
owns to `mag_out`.  Nothing in the kernel checks that the staged span fits the array, that the history holds the oldest tap, or
that the owned ranges of a block's tiles partition its samples: those hold by the arithmetic restated here, which the CPU tests
check over a dense grid of ratios and many block phases.  Every step is the kernel's IEEE double operation in the kernel's order
(numpy does not contract), so the indices land where the kernel's land.  No pixel values: tests/test_sinc_resampler.py's
SincModel computes those.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

T, L, D, H = 16, 256, 8, 32                 # TSDRGPU_SINC_TAPS / _PHASES / _DELAY / _HISTORY (tsdrgpu.h)
SCAP = 4096 + 64                            # SINC_SCAP: staged samples per CTA (resample.cu:474)
PT_MAX = 4096                               # SINC_PT_MAX: pixels per CTA (resample.cu:475)
MIN_RATIO = 0.0625                          # TSDRGPU_SINC_MIN_RATIO
CAP_RATIO = 4098.0 / 4128.0                 # the first ratio whose tile is capped at PT_MAX pixels


def pixels_per_tile(r):
    """sinc_pixels_per_tile (resample.cu:480-483), elementwise."""
    pt = np.floor(float(SCAP - T - 16) * np.asarray(r, np.float64) - 2.0)
    return np.where(pt >= PT_MAX, PT_MAX, pt).astype(np.int64)


def sinc_pos(p, phase, rinv):
    """sinc_pos (resample.cu:485-492): (k0, j) of pixels p of blocks with `phase`, rinv = __drcp_rn(r) = 1/r."""
    q = ((np.asarray(p, np.int64).astype(np.float64) + 0.5) - phase) * rinv - (0.5 + D)
    k0 = np.floor(q)
    j = ((q - k0) * L + 0.5).astype(np.int64)          # (int): truncation of a value >= 0.5
    wrap = j == L
    return np.where(wrap, k0 + 1.0, k0).astype(np.int64), np.where(wrap, 0, j)


def tiles(in_start, size, n_out, r, phase, pt):
    """The host's tile list (resample.cu:725-726: p0 = 0, pt, 2 pt, ... below n_out) and each tile's staging geometry
    (resample.cu:503-512).  Arguments are per-block arrays (pt per block too); returns a dict of per-tile arrays, `block` the
    index of the tile's block."""
    in_start, size, n_out, pt = (np.asarray(a, np.int64) for a in (in_start, size, n_out, pt))
    r, phase = np.asarray(r, np.float64), np.asarray(phase, np.float64)
    ntiles = -(-n_out // pt)
    blk = np.repeat(np.arange(n_out.size), ntiles)
    first = np.concatenate([[0], np.cumsum(ntiles)[:-1]])
    p_lo = (np.arange(blk.size) - first[blk]) * pt[blk]
    bn, bs, bph, rinv = n_out[blk], size[blk], phase[blk], 1.0 / r[blk]
    p_hi = np.minimum(p_lo + pt[blk], bn)
    first_lo = sinc_pos(p_lo, bph, rinv)[0] - (T // 2 - 1)                       # oldest tap of the first pixel
    newest_hi = sinc_pos(p_hi - 1, bph, rinv)[0] + T // 2                        # newest tap of the last pixel
    own_lo = np.where(p_lo == 0, 0, np.maximum(0, first_lo + (T - 1)))
    own_hi = np.where(p_hi == bn, bs, np.maximum(0, sinc_pos(p_hi, bph, rinv)[0] + T // 2))
    st_lo, st_hi = np.minimum(own_lo, first_lo), np.maximum(own_hi, newest_hi + 1)
    return dict(block=blk, p_lo=p_lo, p_hi=p_hi, first_lo=first_lo, newest_hi=newest_hi, own_lo=own_lo, own_hi=own_hi,
                st_lo=st_lo, st_hi=st_hi, n_st=st_hi - st_lo, base=in_start[blk] + st_lo)


# ------------------------------------------------------------------------------------------------------ block sweep
# The blocks the sweep feeds at every ratio, as n_out targets a*pt + b: "lo" is the shortest block that yields at least that
# many pixels, "hi" the longest that yields at most that many (at r > 1 a target may fall between two block sizes).  Three runs
# from offset 0, so each block starts at the phase the recurrence left; long "hi" blocks end their last tile the most samples
# past its last pixel, short first blocks of a run reach furthest into the history.
RECIPE = (
    ((0, 1, "lo"), (1, 0, "hi"), (1, -1, "hi"), (1, 1, "lo"), (2, 0, "hi"), (0, 1, "hi"), (2, 1, "lo"), (3, 0, "hi"), (1, 0, "lo")),
    ((1, 0, "hi"), (0, 1, "hi"), (3, 1, "lo"), (0, 2, "lo"), (2, 0, "lo"), (1, -1, "lo"), (2, -1, "hi")),
    ((0, 1, "lo"), (0, 1, "lo"), (1, 0, "hi"), (3, 0, "hi"), (0, 7, "hi"), (1, 1, "hi")),
)


def _n(s, off, r):
    """n_out of a block of s samples: (uint32_t) (int) ((size - off) * r) (host_plan.c:17)."""
    return np.trunc((s - off) * r)


def _size_for(N, off, r, side):
    """Block sizes (float64 arrays of integers) for n_out target N at the current offsets: see RECIPE."""
    if side == "hi":
        s = _size_for(N + 1, off, r, "lo") - 1.0
        return np.where((s >= 1) & (_n(np.maximum(s, 1.0), off, r) >= 1), s, _size_for(np.ones_like(N), off, r, "lo"))
    s = np.maximum(1.0, np.ceil(N / r + off))
    for _ in range(4):                       # the estimate is off by at most one sample either way
        s = np.where((s > 1) & (_n(s - 1.0, off, r) >= N), s - 1.0, s)
        s = np.where(_n(s, off, r) < N, s + 1.0, s)
    return s


def sweep_blocks(up, down):
    """The recipe's block descriptors at every ratio r = up/down (arrays), via the host recurrence of tsdrgpu_plan_resample
    (host_plan.c:9-29, as tests/resample_model.plan).  Returns per-block arrays (ratio index, run, in_start, size, n_out, r,
    phase), ordered by ratio, run and block."""
    up, down = np.asarray(up, np.float64), np.asarray(down, np.float64)
    r, rinv = up / down, down / up
    pt = pixels_per_tile(r).astype(np.float64)
    off = np.zeros_like(r)
    cols = []
    for run, steps in enumerate(RECIPE):
        in_start = np.zeros_like(r)
        for a, b, side in steps:
            s = _size_for(a * pt + b, off, r, side)
            n = _n(s, off, r)
            assert np.all(n >= 1)
            cols.append((run, in_start.copy(), s, n, -off * r))
            off = off + (n * rinv - s)
            in_start = in_start + s
    nb = len(cols)
    idx = np.repeat(np.arange(r.size), nb)
    run = np.tile([c[0] for c in cols], r.size)
    get = lambda k: np.stack([c[k] for c in cols], axis=1).reshape(-1)
    return dict(ratio=idx, run=run, in_start=get(1).astype(np.int64), size=get(2).astype(np.int64), n_out=get(3).astype(np.int64),
                r=np.repeat(r, nb), phase=get(4), up=np.repeat(up, nb), down=np.repeat(down, nb))


def sweep_runs(up, down):
    """The recipe's runs at one ratio, as lists of block sizes (what the GPU tests feed a resampler from offset 0)."""
    b = sweep_blocks(np.array([up]), np.array([down]))
    return [b["size"][b["run"] == k].tolist() for k in range(len(RECIPE))]


# ------------------------------------------------------------------------------------------------------ ratio grid
def _pt_steps():
    """For every tile size n the tiling takes below the cap, the smallest double r with pixels_per_tile(r) = n."""
    n = np.arange(int(pixels_per_tile(MIN_RATIO)), PT_MAX + 1)
    r = (n + 2.0) / float(SCAP - T - 16)
    for _ in range(8):
        down = np.nextafter(r, 0.0)
        r = np.where(pixels_per_tile(down) >= n, down, r)
        r = np.where(pixels_per_tile(r) < n, np.nextafter(r, np.inf), r)
    assert np.array_equal(pixels_per_tile(r), n) and np.all(pixels_per_tile(np.nextafter(r, 0.0)) == n - 1)
    return r


def production_ratios():
    """(up, down) of the benchmark's front ends as the pipeline plans them: up = w h fv, down = fs."""
    from tempestsdr_b200 import _native as N
    out = []
    for fs, h, fv in ((8_000_000, 525, 60.0), (25_000_000, 1125, 60.0), (50_000_000, 1125, 60.0)):
        w, pr, ptime = C.c_int(0), C.c_double(0), C.c_double(0)
        N.lib().tsdrgpu_geometry(fs, h, fv, C.byref(w), C.byref(pr), C.byref(ptime))
        out.append((float(w.value * h) * fv, float(fs)))
    return out


@functools.lru_cache(maxsize=None)
def grid():
    """(up, down) arrays of the sweep: 3000 log-spaced ratios in [1/16, 16]; every ratio where the tile size steps, one ulp
    either side and 1e-9 relative either side; 1/16; the cap crossing; the sinc tests' RATIOS; the production ratios."""
    steps = _pt_steps()
    r = np.concatenate([np.geomspace(MIN_RATIO, 16.0, 3000), steps, np.nextafter(steps, 0.0), np.nextafter(steps, np.inf),
                        steps * (1 + 1e-9), steps * (1 - 1e-9),
                        [MIN_RATIO, CAP_RATIO, 0.37, 0.5, 0.8, 1.0, 1.5, 1.99631, 1.998, 1.99935, 2.0, 3.7, 7.5]])
    r = np.unique(r[(r >= MIN_RATIO) & (r <= 16.0)])
    prod = np.array(production_ratios())
    return np.concatenate([r, prod[:, 0]]), np.concatenate([np.ones_like(r), prod[:, 1]])


@functools.lru_cache(maxsize=None)
def sweep():
    """Every tile of the recipe's blocks at every grid ratio, with the per-ratio smallest margin of each invariant:
    scap = SCAP - n_st, hist = in_start + st_lo + H, inside = size - 1 - newest_hi, desc = the tiles the host reserves for a
    block (resample.cu:698) minus the tiles it emits.  Returns (blocks, tiles, {name: per-ratio margin})."""
    up, down = grid()
    b = sweep_blocks(up, down)
    pt = pixels_per_tile(b["r"])
    t = tiles(b["in_start"], b["size"], b["n_out"], b["r"], b["phase"], pt)
    tr = b["ratio"][t["block"]]
    R = up.size
    margins = {}
    for name, v, idx in (("scap", SCAP - t["n_st"], tr), ("hist", t["base"] + H, tr),
                         ("inside", b["size"][t["block"]] - 1 - t["newest_hi"], tr)):
        m = np.full(R, np.iinfo(np.int64).max)
        np.minimum.at(m, idx, v)
        margins[name] = m
    reserved = (np.floor(b["size"] * b["r"] + 2.0).astype(np.int64) // pt) + 2
    margins["desc"] = np.full(R, np.iinfo(np.int64).max)
    np.minimum.at(margins["desc"], b["ratio"], reserved - (-(-b["n_out"] // pt)))
    return b, t, margins


def tightest(name, k=3):
    """(up, down) of the k grid ratios with the smallest margin `name` (smallest first)."""
    up, down = grid()
    m = sweep()[2][name]
    order = np.lexsort((up / down, m))[:k]
    return [(float(up[i]), float(down[i])) for i in order]
