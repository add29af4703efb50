"""CPU classifier of the box resampler's geometry (tempestsdr_b200/csrc/resample.cu, header comment).  TEST INFRASTRUCTURE ONLY.

Sample k of a block covers lo_k = fl(fl(k r) + phase), hi_k = fl(lo_k + r), c_k = fl(hi_k - 1) on the pixel axis; after it the
reference's `pid` is P(k) = max(0, ceil(c_k)), so it emits pixels P(k-1) .. P(k)-1, the first of them an A pixel iff
P(k-1) < lo_k and P(k-1) < c_k.  Everything here is float64 elementwise numpy, one IEEE operation per step (numpy does not
contract), so it lands where the reference and the kernels land.  No pixel VALUES: the oracle computes those.

What it classifies is where the kernels take their rare paths: bank walks (an A sample whose predecessor was not A), walks that
reach back across a tile start or past the block start (left to rs_fixup), blocks without any A sample (rs_fixup's serial
branch), stale slots (the reference sizes a block for one pixel more than its loop writes), samples that emit three or more
pixels, and rs_main's tiles whose pixels do or do not fit its shared-memory staging.
"""
from __future__ import annotations

from collections import Counter

import numpy as np

RS_TILE = 2048                      # samples per CTA tile (resample.cu)
RS_OUT_CAP = 3 * RS_TILE + 16       # pixels rs_main stages per tile; a tile with more stores directly


def plan(offset: float, sizes, up: float, down: float):
    """tsdrgpu_plan_resample (dsp.c:258-262,272,306) for consecutive blocks: ([(size, n_out, r, phase)], new offset), or
    (None, offset) when a block would yield no pixel (the reference asserts there)."""
    r = up / down
    rinv = down / up
    off = float(offset)
    blocks = []
    for s in sizes:
        n = int((s - off) * r) & 0xFFFFFFFF          # (uint32_t) (int) ((size - off) * r)
        if n == 0:
            return None, offset
        blocks.append((int(s), n, r, -off * r))
        off = off + (n * rinv - s)
    return blocks, off


def sizes_with_pixels(sizes, up: float, down: float, offset: float = 0.0):
    """`sizes`, each block grown by the fewest samples that make it yield a pixel where it would yield none."""
    r = up / down
    out = []
    off = float(offset)
    for s in sizes:
        s = int(s)
        while int((s - off) * r) & 0xFFFFFFFF == 0:
            s += 1
        n = int((s - off) * r) & 0xFFFFFFFF
        out.append(s)
        off = off + (n * (down / up) - s)
    return out


def geometry(blocks):
    """Per sample of the blocks laid end to end: local index k, lo, c, P(k-1), P(k), A; and the blocks' sample starts."""
    sizes = np.array([b[0] for b in blocks], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    k = np.arange(int(sizes.sum()), dtype=np.int64) - np.repeat(starts, sizes)
    r = np.repeat(np.array([b[2] for b in blocks], dtype=np.float64), sizes)
    phase = np.repeat(np.array([b[3] for b in blocks], dtype=np.float64), sizes)
    lo = np.add(np.multiply(k.astype(np.float64), r), phase)
    hi = np.add(lo, r)
    c = np.add(hi, -1.0)
    P = np.where(c > 0.0, np.ceil(c), 0.0)
    Pm = np.concatenate([[0.0], P[:-1]])
    Pm[starts] = 0.0                                  # pid starts every block at 0
    A = (Pm < lo) & (Pm < c)
    return dict(k=k, lo=lo, hi=hi, c=c, Pm=Pm, P=P, A=A, starts=starts, sizes=sizes)


def classify(blocks, leads=None):
    """Counts for one run of consecutive blocks (plan()'s list).  `leads[b]`: samples block b's input start lies past a
    16-byte boundary (rs_main4 cuts its first tile short by that many; 0 for rs_main).  Returns (Counter, emitted) where
    emitted[b] = P(size_b - 1), the pixels the reference's loop writes for block b."""
    g = geometry(blocks)
    k, P, Pm, A, starts, sizes = g["k"], g["P"], g["Pm"], g["A"], g["starts"], g["sizes"]
    nb = len(blocks)
    ends = starts + sizes - 1
    n_out = np.array([b[1] for b in blocks], dtype=np.int64)
    r = np.array([b[2] for b in blocks], dtype=np.float64)
    idx = np.arange(k.size, dtype=np.int64)
    blk = np.repeat(np.arange(nb), sizes)
    cnt = (P - Pm).astype(np.int64)
    emitted = P[ends].astype(np.int64)
    C = Counter()
    C["samples"] = int(k.size)
    C["blocks"] = nb
    C["A_pixels"] = int(A.sum())
    C["B_pixels"] = int(cnt.sum() - A.sum())
    C["ge3_samples"] = int((cnt >= 3).sum())
    # the bank rule's `P(k) < hi_k` (dsp.c:299) at an A sample, the only samples whose bank the next sample takes as it is
    C["A_with_P_ge_hi"] = int((A & (P >= g["hi"])).sum())
    # latest A sample strictly before each sample, within its block (-1: none)
    lastA = np.maximum.accumulate(np.where(A, idx, -1))
    prevA_at = np.concatenate([[-1], lastA[:-1]])
    prevA_at = np.where(prevA_at >= np.repeat(starts, sizes), prevA_at, -1)
    Aprev = np.concatenate([[False], A[:-1]])
    Aprev[starts] = False
    walk = A & (k > 0) & ~Aprev
    walk_r_gt_1 = walk & (np.repeat(r, sizes) > 1.0)
    C["walks"] = int(walk.sum())
    C["walks_r_gt_1"] = int(walk_r_gt_1.sum())
    past = walk & (prevA_at < 0)
    C["walks_past_block_start"] = int(past.sum())
    # rs_main4's tiles: the first one cut short by `lead`, every later one RS_TILE long
    lead = np.zeros(nb, dtype=np.int64) if leads is None else np.asarray(leads, dtype=np.int64)
    first_end = np.repeat(RS_TILE - lead, sizes)
    tile0 = np.where(k < first_end, 0, first_end + ((k - first_end) // RS_TILE) * RS_TILE)
    tile_start = np.repeat(starts, sizes) + tile0
    cross = walk & (prevA_at >= 0) & (prevA_at < tile_start)
    C["walks_cross_tile"] = int(cross.sum())
    C["no_A_blocks"] = int(np.count_nonzero(np.bincount(blk, weights=A, minlength=nb) == 0))
    C["no_A_blocks_with_pixels"] = int(np.count_nonzero((np.bincount(blk, weights=A, minlength=nb) == 0) & (n_out >= 1)))
    C["stale_slots"] = int(np.maximum(n_out - emitted, 0).sum())
    C["pixels_past_n_out"] = int(np.maximum(emitted - n_out, 0).sum())
    # rs_main's tiles (RS_TILE from each block start): staged in shared memory while the tile's pixels fit RS_OUT_CAP
    ts = np.flatnonzero(k % RS_TILE == 0)
    te = np.concatenate([ts[1:], [k.size]]) - 1
    tile_px = P[te] - Pm[ts]
    C["tiles_staged"] = int((tile_px <= RS_OUT_CAP).sum())
    C["tiles_unstaged"] = int((tile_px > RS_OUT_CAP).sum())
    return C, emitted


def stale_slots(blocks, emitted):
    """Output indices (over the run) of the slots the reference sizes but does not write; the library writes 0.0f there."""
    out, base = [], 0
    for (s, n, _, _), e in zip(blocks, emitted):
        out.extend(range(base + int(e), base + n))
        base += n
    return out
