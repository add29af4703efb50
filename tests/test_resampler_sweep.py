"""The box resampler (tsdrgpu_resampler_run, csrc/resample.cu) bit for bit against the oracle through every kernel it can launch.

In box mode a run launches one main kernel and then rs_fixup:
  * rs_main4<true, MINB> (IQ in, demodulation fused) or rs_main4<false, 5> (magnitudes) for r <= 2 -- every ratio a front end
    gives; MINB is 4 unless TSDRGPU_RS_MINB (read once per process) asks for 3, 5 or 6;
  * rs_main<IQ> for r > 2 and whenever TSDRGPU_RS_V1 is set (read on every run): the cross-check of rs_main4.  It stages a
    tile's pixels in shared memory while they fit RS_OUT_CAP and stores them directly beyond;
  * rs_fixup: one CTA striding over the blocks by 256, which writes each block's first A pixel (its bank reaches into the
    previous block), passes the bank through blocks without an A sample, zeroes stale slots and leaves the new `contrib`.
Every case here runs with the default dispatch and again with TSDRGPU_RS_V1=1, with magnitude and IQ input (IQ also writing the
magnitudes, with guard floats around them), at every input, output and magnitude address phase.  The oracle is the compiled
reference where it travelled with the tree, else the pinned restatement; slots the reference leaves stale are 0.0f here
(DESIGN.md §2) and are found with tests/resample_model.py, which these CPU tests first hold to the restatement.

Axes: the ten front-end geometries the project meets (and two PLL-moved refresh rates each), general ratios from 1/16 to 16
(either side of 1, 2 and the staging capacity), block sizes 1..8, around RS_TILE and 2 RS_TILE, runs of 1 ... 4000 blocks and one
of 65 535, streams cut into calls at different places, resumed from set_state and with the ratio changing between calls, the
nearest-neighbour mode, and refusals, which must change nothing.  The coverage certificate checks that the cases reach every
rare path of the kernels (tests/resample_model.py names them), so trimming the case list cannot drop one unnoticed.
"""
import ctypes as C
import functools
import os
import subprocess
import sys
import zlib
from collections import Counter

import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import _native as N
from tests import resample_model as rm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RS_TILE, RS_OUT_CAP = rm.RS_TILE, rm.RS_OUT_CAP
EINVAL, ECAPACITY = -3, -5                 # TSDRGPU_EINVAL, TSDRGPU_ECAPACITY (include/tsdrgpu.h)

# (samplerate, lines, refresh rate): the front ends of the README and the geometry sweep's 7-, 71- and 16666-column frames
PRODUCTION = {
    "8M_525": (8_000_000, 525, 60.0),
    "25M_1125": (25_000_000, 1125, 60.0),
    "50M_1125": (50_000_000, 1125, 60.0),
    "2048k_525": (2_048_000, 525, 60.0),
    "2400k_313": (2_400_000, 313, 59.94),
    "1M_100_exact2": (1_000_000, 100, 50.0),            # r = 2.0 exactly
    "10M_625_exact2": (10_000_000, 625, 50.0),          # r = 2.0 exactly
    "2400k_1125_w71": (2_400_000, 1125, 60.0),          # r = 639/320
    "250k_1125_w7": (250_000, 1125, 60.0),
    "50M_100_w16666": (50_000_000, 100, 60.0),
}
PLL_STEP = 3e-5           # the PLL-moved refresh rates: fv -+ 3 * 1e-5
# general ratios (C-ABI), as (upsample_by, downsample_by) so that r = up/down is the intended double
GENERAL = {
    "1/16": (1.0, 16.0), "0.1": (0.1, 1.0), "1/3": (1.0, 3.0), "0.37": (0.37, 1.0), "0.5": (0.5, 1.0), "0.9999": (0.9999, 1.0),
    "1": (1.0, 1.0), "1+2^-40": (1.0 + 2.0 ** -40, 1.0), "1.0001": (1.0001, 1.0), "4/3": (4.0, 3.0), "1.5": (1.5, 1.0),
    "1.996875": (1.996875, 1.0), "1.998": (1.998, 1.0), "2-2^-51": (2.0 - 2.0 ** -51, 1.0), "2": (2.0, 1.0),
    "2+2^-51": (2.0 + 2.0 ** -51, 1.0), "2.5": (2.5, 1.0), "3": (3.0, 1.0),
    # a full tile of RS_TILE samples yields RS_OUT_CAP pixels (staged) / RS_OUT_CAP + 1 (stored directly)
    "cap": (float(RS_OUT_CAP), float(RS_TILE)), "cap+1": (float(RS_OUT_CAP + 1), float(RS_TILE)),
    "3.25": (3.25, 1.0), "7.5": (7.5, 1.0), "16": (16.0, 1.0),
}
MIXED = [1000 + 37 * j for j in range(9)] + [7, 11, 4100, RS_TILE - 1, RS_TILE + 1, 2 * RS_TILE + 1, 1, 2, 3, 5000]
SHAPES = (list(range(1, 9)) + list(range(RS_TILE - 4, RS_TILE + 5)) + [2 * RS_TILE - 1, 2 * RS_TILE + 1, 4100]
          + [int(s) for s in np.random.default_rng(20).integers(1, 5000, 12)])
SHAPE_RATIOS = ["1M_100_exact2", "2400k_1125_w71", "25M_1125", "1/16", "0.37", "1", "1.5", "2+2^-51", "cap+1", "3.25", "16"]
RUN_COUNTS = [1, 255, 256, 257, 4000]
COUNT_RATIOS = ["1M_100_exact2", "2400k_1125_w71", "0.5"]
# (input phase, output phase, magnitude phase), floats past a 16-byte boundary (IQ input: input phase mod 2, in pairs)
PHASES = [(0, 1, 2), (1, 2, 3), (2, 3, 0), (3, 0, 1)]


def geometry(fs, h, fv):
    w, pr, pt = C.c_int(0), C.c_double(0), C.c_double(0)
    N.lib().tsdrgpu_geometry(fs, h, fv, C.byref(w), C.byref(pr), C.byref(pt))
    return w.value


def production_rate(fs, h, fv):
    """(upsample_by, downsample_by, block) as the pipeline plans them (pipeline.cu: block, up = w h fv)."""
    w = geometry(fs, h, fv)
    return float(w * h) * fv, float(fs), int(0.1 * fs / fv)


def ratio(name):
    """(upsample_by, downsample_by, production block or None) of a named ratio: NAME, NAME+pll or NAME-pll, or a GENERAL key."""
    if name in GENERAL:
        return GENERAL[name] + (None,)
    base, _, moved = name.partition("@")
    fs, h, fv = PRODUCTION[base]
    fv = fv + PLL_STEP if moved == "+pll" else fv - PLL_STEP if moved == "-pll" else fv
    return production_rate(fs, h, fv)


SWEEP_RATIOS = [n for b in PRODUCTION for n in (b, b + "@+pll", b + "@-pll")] + list(GENERAL)


def sweep_calls(name):
    """The ratio sweep's stream for a ratio: one call of production blocks (enough for 300 000 samples, 4 to 300 blocks), or
    MIXED grown where a block would yield no pixel."""
    up, down, block = ratio(name)
    sizes = [block] * min(300, max(4, 300_000 // block)) if block else rm.sizes_with_pixels(MIXED, up, down)
    return [(sizes, up, down)]


def shape_calls(name):
    up, down, _ = ratio(name)
    return [(rm.sizes_with_pixels(SHAPES, up, down), up, down)]


def count_calls(name, nblocks):
    up, down, _ = ratio(name)
    sizes = np.random.default_rng(nblocks).integers(1, 700, nblocks)
    return [(rm.sizes_with_pixels(sizes, up, down), up, down)]


def small_blocks_calls():
    """65 535 blocks of 1 to 8 samples at r = 2: the largest run, rs_fixup over 256 strides, most blocks without an A sample."""
    sizes = np.random.default_rng(65535).integers(1, 9, 65535)
    return [(rm.sizes_with_pixels(sizes, 2.0, 1.0), 2.0, 1.0)]


def all_cases():
    cases = {f"sweep[{n}]": sweep_calls(n) for n in SWEEP_RATIOS}
    cases.update({f"shapes[{n}]": shape_calls(n) for n in SHAPE_RATIOS})
    cases.update({f"count[{n},{c}]": count_calls(n, c) for n in COUNT_RATIOS for c in RUN_COUNTS})
    cases["65535_blocks"] = small_blocks_calls()
    return cases


def plan_calls(calls, offset=0.0):
    """Per call the model's blocks; the offset after the last call."""
    out = []
    for sizes, up, down in calls:
        blocks, offset = rm.plan(offset, sizes, up, down)
        assert blocks is not None
        out.append(blocks)
    return out, offset


# ------------------------------------------------------------------------------------------------ CPU: the model
def _ref_written(R, block, up, down, state):
    """Pixels the compiled reference's loop writes for one block, from state: from that state first run a block long enough
    to write NaN over every slot this one is sized for, then the block itself over zeros; the slots still NaN were not written
    (the output buffer is the reference's own, kept between calls; realloc keeps its content)."""
    R.state = state
    R.run(np.full(2 * block + int(2 * down / up) + 2, np.nan, np.float32), up, down)
    R.state = state
    o = R.run(np.zeros(block, np.float32), up, down)
    nan = np.flatnonzero(np.isnan(o))
    return int(nan[0]) if nan.size else o.size


def test_classifier_emitted_counts_match_the_restatement_and_the_reference():
    """For every case of the GPU sweep, block by block: the model's emitted count P(size-1) equals the restatement's
    `last_emitted`, and, where the compiled reference is present, the slots its loop writes."""
    P = orc.port()
    R = orc.ref().resampler() if orc.have_ref() else None
    for name, calls in all_cases().items():
        rs = P.resampler()
        zero = np.zeros(max(max(s) for s, _, _ in calls), np.float32)
        blocks_per_call, _ = plan_calls(calls)
        checked_stale = 0
        for (sizes, up, down), blocks in zip(calls, blocks_per_call):
            _, emitted = rm.classify(blocks)
            for b, ((s, n, _, _), e) in enumerate(zip(blocks, emitted)):
                before = rs.state
                assert rs.run(zero[:s], up, down).size == n, (name, b)
                assert rs.last_emitted == e, (name, b, rs.last_emitted, int(e))
                if R is not None and (b < 64 or (e < n and checked_stale < 2000)):   # the start of every stream, stale slots
                    assert _ref_written(R, s, up, down, before) == min(int(e), n), (name, b)
                    checked_stale += e < n
        assert rs.state[1] == plan_calls(calls)[1], name


RS_BLOCK = np.dtype([("in_start", "<u8"), ("out_start", "<u8"), ("size", "<u4"), ("n_out", "<u4"), ("r", "<f8"), ("phase", "<f8")])
PLAN_RATIOS = list(PRODUCTION) + ["1/16", "0.37", "1", "3.25"]


@pytest.mark.parametrize("name", PLAN_RATIOS)
def test_plan_resample_matches_the_reference_recurrence(name):
    """tsdrgpu_plan_resample over 100 000 consecutive blocks (one call) against the reference's recurrence (dsp.c:258-262,272,306)
    restated in Python, every field of every block and the final offset bit for bit; and against the oracle's resampler (the
    compiled reference where present), block by block in nearest-neighbour mode, over the first blocks up to 5e7 pixels."""
    up, down, block = ratio(name)
    block = block or 4099
    nb = 100_000
    lib = N.lib()
    off = C.c_double(0.0)
    arr = np.zeros(nb, RS_BLOCK)
    total = lib.tsdrgpu_plan_resample(C.byref(off), None, block, nb, up, down, arr.ctypes.data_as(C.c_void_p))
    want, want_off = rm.plan(0.0, [block] * nb, up, down)
    n_out = np.array([b[1] for b in want], np.uint64)
    assert total == int(n_out.sum())
    assert np.array_equal(arr["n_out"], n_out.astype(np.uint32))
    assert np.array_equal(arr["size"], np.full(nb, block, np.uint32))
    assert np.array_equal(arr["out_start"], np.concatenate([[0], np.cumsum(n_out)[:-1]]).astype(np.uint64))
    assert np.array_equal(arr["in_start"], np.arange(nb, dtype=np.uint64) * block)
    assert np.array_equal(arr["r"].view(np.uint64), np.full(nb, up / down).view(np.uint64))
    assert np.array_equal(arr["phase"].view(np.uint64), np.array([b[3] for b in want]).view(np.uint64))
    assert off.value == want_off
    O = orc.best()
    rs = O.resampler()
    x = np.zeros(block, np.float32)
    limit = 0
    for b in range(nb):
        if limit > 50_000_000:
            break
        assert rs.run(x, up, down, nearest=True).size == want[b][1], b
        limit += want[b][1]
        if b + 1 < nb:
            assert arr["phase"][b + 1] == -rs.state[1] * (up / down), b
    assert b >= 200


@functools.lru_cache(maxsize=1)
def certificate():
    """The model's counts summed over every case of the sweep, at every input phase the GPU runs use."""
    total = Counter()
    for name, calls in all_cases().items():
        blocks_per_call, _ = plan_calls(calls)
        for blocks in blocks_per_call:
            starts = np.concatenate([[0], np.cumsum([b[0] for b in blocks])[:-1]])
            C0, _ = rm.classify(blocks)
            total.update(C0)
            for ph in range(4):                              # magnitude input: rs_main4 cuts the first tile by (phase + start) mod 4
                Cp, _ = rm.classify(blocks, leads=(ph + starts) % 4)
                total["walks_cross_tile_main4"] += Cp["walks_cross_tile"]
    return total


RARE = ["ge3_samples", "walks_r_gt_1", "walks_cross_tile", "walks_cross_tile_main4", "walks_past_block_start", "no_A_blocks_with_pixels", "stale_slots", "tiles_staged",
        "tiles_unstaged", "A_pixels", "B_pixels"]


def test_coverage_certificate():
    """Every rare path of the box kernels is reached somewhere in the sweep: samples emitting three or more pixels (rs_main4's
    third predicated store), bank walks at r > 1 (rs_bank_walk, rs_main's general case), walks across a tile start (for
    rs_main's tiles and for rs_main4's address-cut ones), walks past the block start (left to rs_fixup), blocks with pixels
    but no A sample (rs_fixup's serial branch), stale slots, and rs_main tiles on both sides of RS_OUT_CAP."""
    total = certificate()
    print("\nbox resampler coverage certificate:", {k: total[k] for k in ["samples", "blocks"] + RARE})
    missing = [k for k in RARE if total[k] == 0]
    assert not missing, f"the sweep no longer reaches {missing}"
    # An A sample has c > 0, so P = ceil(c) < c + 1 = hi (hi - 1 is exact): the bank rule's `P < hi` cannot fail where its
    # result is used unwalked, and `<` and `<=` there give the same pixels.
    assert total["A_with_P_ge_hi"] == 0


def test_blocks_without_an_A_sample_are_reachable():
    """A block can yield pixels without any sample emitting an A pixel, so rs_fixup's serial branch (which passes the bank
    through such a block) is live code: at r = 2 a one-sample block from offset 0 writes one B pixel and is sized for two, and
    at r = 1/2 a two-sample block is sized for one pixel it never writes.  Checked against the restatement."""
    P = orc.port()
    for sizes, up, down in [([1, 1, 3], 2.0, 1.0), ([2, 2, 5], 0.5, 1.0), ([16, 16, 40], 1.0, 16.0)]:
        blocks, _ = rm.plan(0.0, sizes, up, down)
        g = rm.geometry(blocks[:1])
        assert not g["A"].any() and blocks[0][1] >= 1
        Cn, emitted = rm.classify(blocks)
        assert Cn["no_A_blocks_with_pixels"] >= 2 and Cn["stale_slots"] >= 2
        rs = P.resampler()
        for (s, n, _, _), e in zip(blocks, emitted):
            assert rs.run(np.ones(s, np.float32), up, down).size == n and rs.last_emitted == e


# ------------------------------------------------------------------------------------------------ GPU
def noise_iq(n_pairs, seed):
    """Seeded noise IQ with a few exact specials: magnitudes 0, |-0|, 1e-30 and 3e38."""
    rng = np.random.default_rng(seed)
    iq = rng.standard_normal(2 * n_pairs).astype(np.float32)
    specials = [(0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (1e-30, 0.0), (0.0, 1e-30), (3e38, 0.0), (-3e38, 0.0)]
    at = np.linspace(0, n_pairs - 1, min(n_pairs, 3 * len(specials))).astype(np.int64)
    for j, p in enumerate(at):
        iq[2 * p], iq[2 * p + 1] = specials[j % len(specials)]
    return iq


def oracle_stream(O, mag, calls, state=(0.0, 0.0), nearest=False):
    """The oracle block by block over the calls from `state`; stale slots 0.0f (found by the model).  (pixels, state)."""
    rs = O.resampler()
    rs.state = state
    out, pos, off = [], 0, state[1]
    for sizes, up, down in calls:
        blocks, off = rm.plan(off, sizes, up, down)
        _, emitted = rm.classify(blocks)
        for (s, n, _, _), e in zip(blocks, emitted):
            o = rs.run(mag[pos:pos + s], up, down, nearest)
            assert o.size == n
            if not nearest and e < n:
                o = o.copy()
                o[e:] = 0.0
            out.append(o)
            pos += s
        assert rs.state[1] == off
    return np.concatenate(out), rs.state


GUARD = -7.0


class Gpu:
    """Runs calls through one tsdrgpu resampler with input, output and magnitude views at chosen address phases."""

    def __init__(self, ctx):
        import torch
        self.torch, self.ctx = torch, ctx

    def view(self, host, phase, fill=None, n=None):
        t = self.torch
        n = host.size if n is None else n
        buf = t.full((n + 8,), GUARD if fill is None else fill, dtype=t.float32, device="cuda")
        assert buf.data_ptr() % 16 == 0
        if host is not None and fill is None:
            buf[4 + phase:4 + phase + n] = t.from_numpy(host)
        return buf, buf[4 + phase:4 + phase + n]

    def run(self, iq, mag, calls, is_iq, phases, nearest=False, with_mag=True, state=None, r=None):
        """(pixels, state, magnitudes or None, guards intact) of the calls, each its own tsdrgpu_resampler_run."""
        t = self.torch
        in_ph, out_ph, mag_ph = phases
        src = iq if is_iq else mag
        fl = 2 if is_iq else 1
        _, x = self.view(src, 2 * (in_ph % 2) if is_iq else in_ph)
        want_mag = is_iq and with_mag and not nearest
        if want_mag:
            mbuf, mview = self.view(None, mag_ph, fill=GUARD, n=mag.size)
        r = r or self.ctx.resampler()
        if state is not None:
            r.state = state
        total = sum(int(sum(s)) for s, _, _ in calls)
        need, off = 0, r.state[1]
        for sizes, up, down in calls:
            blocks, off = rm.plan(off, sizes, up, down)
            need += sum(b[1] for b in blocks)
        obuf, oview = self.view(None, out_ph, fill=GUARD, n=need)
        pos = opos = 0
        for sizes, up, down in calls:
            bs = (sizes[0], len(sizes)) if len(set(sizes)) == 1 else sizes
            n = int(sum(sizes))
            got = r.process(x[fl * pos:fl * (pos + n)], bs, up, down, nearest, in_is_iq=is_iq, out=oview[opos:],
                            mag_out=mview[pos:pos + n] if want_mag else None)
            pos += n
            opos += got.numel()
        assert pos == total and opos == need
        t.cuda.synchronize()
        ob = obuf.cpu().numpy()
        guards = np.all(ob[:4 + out_ph] == GUARD) and np.all(ob[4 + out_ph + need:] == GUARD)
        m = None
        if want_mag:
            mb = mbuf.cpu().numpy()
            guards = guards and np.all(mb[:4 + mag_ph] == GUARD) and np.all(mb[4 + mag_ph + mag.size:] == GUARD)
            m = mb[4 + mag_ph:4 + mag_ph + mag.size]
        return ob[4 + out_ph:4 + out_ph + need], r.state, m, guards


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_same(got, want, what):
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    bad = np.flatnonzero(bits(got) != bits(want))
    assert bad.size == 0, f"{what}: {bad.size} of {got.size} pixels differ, first at {bad[:5]}: {got[bad[:5]]} vs {want[bad[:5]]}"


@pytest.fixture(scope="module")
def ctx():
    from tempestsdr_b200 import api
    return api.Context(0)


@pytest.fixture(scope="module")
def O():
    return orc.best()


def stream(calls, seed):
    n = sum(int(sum(s)) for s, _, _ in calls)
    iq = noise_iq(n, seed)
    return iq, orc.best().am_demod(iq)


def check_all_paths(ctx, O, calls, monkeypatch, seed, phases=PHASES, state=(0.0, 0.0), what=""):
    """The calls from `state`, against the oracle: magnitude and IQ input, each phase triple, default dispatch and TSDRGPU_RS_V1."""
    iq, mag = stream(calls, seed)
    want, want_state = oracle_stream(O, mag, calls, state)
    g = Gpu(ctx)
    for v1 in (False, True):
        if v1:
            monkeypatch.setenv("TSDRGPU_RS_V1", "1")
        else:
            monkeypatch.delenv("TSDRGPU_RS_V1", raising=False)
        for is_iq in (False, True):
            for ph in phases:
                label = f"{what} v1={v1} iq={is_iq} phases={ph}"
                got, st, m, guards = g.run(iq, mag, calls, is_iq, ph, state=state)
                assert_same(got, want, label)
                assert st == want_state, (label, st, want_state)
                assert guards, f"{label}: a write outside the output or magnitude view"
                if m is not None:
                    assert_same(m, mag, label + " magnitudes")
    monkeypatch.delenv("TSDRGPU_RS_V1", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SWEEP_RATIOS)
def test_ratio_sweep(ctx, O, name, monkeypatch):
    check_all_paths(ctx, O, sweep_calls(name), monkeypatch, seed=zlib.crc32(name.encode()), what=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SHAPE_RATIOS)
def test_block_shapes(ctx, O, name, monkeypatch):
    """Blocks of 1 to 8 samples, RS_TILE - 4 ... RS_TILE + 4, 2 RS_TILE -+ 1, 4100 and a seeded mix, back to back in one run."""
    check_all_paths(ctx, O, shape_calls(name), monkeypatch, seed=5, what=name)


@pytest.mark.gpu
@pytest.mark.parametrize("nblocks", RUN_COUNTS)
@pytest.mark.parametrize("name", COUNT_RATIOS)
def test_run_counts(ctx, O, name, nblocks, monkeypatch):
    """1 to 4000 blocks in one run: rs_fixup strides over the blocks by 256."""
    check_all_paths(ctx, O, count_calls(name, nblocks), monkeypatch, seed=nblocks, phases=PHASES[:2], what=f"{name} x{nblocks}")


@pytest.mark.gpu
def test_65535_small_blocks(ctx, O, monkeypatch):
    """The largest run a call takes, of blocks of 1 to 8 samples at r = 2 (most of them without an A sample)."""
    check_all_paths(ctx, O, small_blocks_calls(), monkeypatch, seed=65535, phases=PHASES[1:2], what="65535 blocks")


@pytest.mark.gpu
def test_stream_cut_into_calls_anywhere(ctx, O, monkeypatch):
    """One stream, cut into calls at three different places (and into four calls), gives the same pixels and state as the
    oracle's block-by-block run and so as one call."""
    up, down, block = ratio("2400k_313")
    sizes = [block] * 6 + [5, 1, 2, RS_TILE + 3, block, 7, block]
    sizes = rm.sizes_with_pixels(sizes, up, down)
    for cuts in ([1], [6], [9], [2, 8, 11]):
        edges = [0] + cuts + [len(sizes)]
        calls = [(sizes[a:b], up, down) for a, b in zip(edges[:-1], edges[1:])]
        check_all_paths(ctx, O, calls, monkeypatch, seed=3, phases=PHASES[:2], what=f"cuts {cuts}")


@pytest.mark.gpu
@pytest.mark.parametrize("state", [(0.125, -0.25), (1e30, 0.3), (-3.5, -0.75), (0.0, 0.999)])
@pytest.mark.parametrize("name", ["25M_1125", "1M_100_exact2", "0.37", "3.25"])
def test_resume_from_set_state(ctx, O, name, state, monkeypatch):
    """set_state from an arbitrary (contrib, offset), given to the oracle too: a negative offset, a contrib of 1e30."""
    up, down, block = ratio(name)
    sizes = rm.sizes_with_pixels(([block] * 3 if block else []) + [1, 2, 3, 4100, RS_TILE + 1], up, down, state[1])
    check_all_paths(ctx, O, [(sizes, up, down)], monkeypatch, seed=17, phases=PHASES[:2], state=state, what=f"{name} {state}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["8M_525", "2400k_1125_w71", "1M_100_exact2"])
def test_ratio_changes_between_calls(ctx, O, name, monkeypatch):
    """As the PLL moves the refresh rate: every call its own geometry and block, the state carried across."""
    fs, h, fv = PRODUCTION[name]
    calls = []
    for step in (0, 1, 3, -2, -7, 0, 11):
        up, down, block = production_rate(fs, h, fv + step * 1e-5)
        calls.append(([block] * 2, up, down))
    check_all_paths(ctx, O, calls, monkeypatch, seed=23, phases=PHASES[:2], what=name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", SWEEP_RATIOS[::2] + SHAPE_RATIOS[:1])
def test_nearest_neighbour(ctx, O, name):
    """Nearest-neighbour mode at the sweep's ratios, phases and shapes; it leaves `contrib` alone."""
    up, down, _ = ratio(name)
    calls = [(rm.sizes_with_pixels(sweep_calls(name)[0][0] + SHAPES, up, down), up, down)]
    iq, mag = stream(calls, 31)
    state = (0.625, 0.0)
    want, want_state = oracle_stream(O, mag, calls, state, nearest=True)
    g = Gpu(ctx)
    for is_iq in (False, True):
        for ph in PHASES:
            got, st, _, guards = g.run(iq, mag, calls, is_iq, ph, nearest=True, state=state)
            assert_same(got, want, f"{name} nearest iq={is_iq} {ph}")
            assert st == (state[0], want_state[1]) and guards


@pytest.mark.gpu
def test_refusals_change_nothing(ctx, O):
    """A block with no pixel (EINVAL), a too-small output (ECAPACITY), more than 65 535 blocks (EINVAL), and magnitudes asked
    of magnitude input or of the nearest-neighbour mode (EINVAL) are refused; a refused call leaves the state, the armed
    magnitude output and the next run's pixels exactly as they were."""
    import torch
    lib = N.lib()
    up, down, block = ratio("2400k_1125_w71")
    sizes = [block] * 3
    calls = [(sizes, up, down)]
    iq, mag = stream(calls, 41)
    want, want_state = oracle_stream(O, mag, calls, (0.25, -0.125))
    n = int(sum(sizes))
    need = int(sum(b[1] for b in rm.plan(-0.125, sizes, up, down)[0]))
    x_iq = torch.from_numpy(iq).cuda()
    x_mag = torch.from_numpy(mag).cuda()
    out = torch.full((need + 4,), GUARD, device="cuda")
    arr = np.array(sizes, np.uint32)
    sz = arr.ctypes.data_as(C.c_void_p)
    one = np.array([1], np.uint32)
    big = np.full(65536, block, np.uint32)

    def raw(x, is_iq, p, u, nb, up_, down_, nearest, o, cap):
        n_out = C.c_uint64(123)
        rc = lib.tsdrgpu_resampler_run(r._h, ctx.stream, x.data_ptr(), is_iq, p, u, nb, up_, down_, nearest, o.data_ptr(), cap,
                                       C.byref(n_out))
        return rc, n_out.value

    refusals = [
        ("no pixel", lambda: raw(x_mag, 0, one.ctypes.data_as(C.c_void_p), 0, 1, 0.1, 1.0, 0, out, need), EINVAL),
        ("capacity", lambda: raw(x_iq, 1, sz, 0, 3, up, down, 0, out, need - 1), ECAPACITY),
        ("65536 blocks", lambda: raw(x_mag, 0, big.ctypes.data_as(C.c_void_p), 0, 65536, up, down, 0, out, 1 << 40), EINVAL),
        ("65536 uniform", lambda: raw(x_mag, 0, None, block, 65536, up, down, 0, out, 1 << 40), EINVAL),
        ("mag of magnitudes", lambda: raw(x_mag, 0, sz, 0, 3, up, down, 0, out, need), EINVAL),
        ("mag of nearest", lambda: raw(x_iq, 1, sz, 0, 3, up, down, 1, out, need), EINVAL),
    ]
    for what, call, code in refusals:
        for armed in ((True,) if what.startswith("mag") else (False, True)):   # magnitudes are refused only when asked for
            r = ctx.resampler()
            r.state = (0.25, -0.125)
            mbuf = torch.full((n + 8,), GUARD, device="cuda")
            if armed:
                assert lib.tsdrgpu_resampler_set_mag_out(r._h, mbuf[4:].data_ptr()) == N.OK
            for _ in range(5):                                # more refusals than descriptor slots
                rc, n_out = call()
                assert (rc, n_out) == (code, 0), (what, rc, n_out)
            assert r.state == (0.25, -0.125), what
            torch.cuda.synchronize()
            assert torch.all(out == GUARD) and torch.all(mbuf == GUARD), f"{what}: a refused call wrote"
            rc, n_out = raw(x_iq, 1, sz, 0, 3, up, down, 0, out, need)
            assert (rc, n_out) == (N.OK, need), what
            got = out[:need].cpu().numpy()
            assert_same(got, want, f"the run after '{what}' (mag armed: {armed})")
            assert r.state == want_state, what
            m = mbuf.cpu().numpy()
            if armed:                                         # still armed: the run after the refusal writes the magnitudes
                assert_same(m[4:4 + n], mag, f"magnitudes after '{what}'")
                assert np.all(m[:4] == GUARD) and np.all(m[4 + n:] == GUARD)
            else:
                assert np.all(m == GUARD)
            out.fill_(GUARD)
            del r


# ---- TSDRGPU_RS_MINB: read once per process, so each value in a process of its own
MINB_RATIOS = ["25M_1125", "1M_100_exact2", "2400k_1125_w71", "250k_1125_w7", "50M_100_w16666"]


def minb_case(path):
    """Production ratios, IQ input with magnitudes, every phase triple: pixels, states and magnitudes to `path`."""
    from tempestsdr_b200 import api
    g = Gpu(api.Context(0))
    res = {}
    for name in MINB_RATIOS:
        calls = sweep_calls(name)
        iq, mag = stream(calls, 7)
        for j, ph in enumerate(PHASES):
            got, st, m, guards = g.run(iq, mag, calls, True, ph)
            res[f"{name}_{j}_px"], res[f"{name}_{j}_mag"] = got, m
            res[f"{name}_{j}_state"] = np.array([st[0], st[1], float(guards)])
    np.savez(path, **res)


@pytest.mark.gpu
@pytest.mark.parametrize("minb", ["3", "5", "6"])
def test_rs_main4_register_targets(O, tmp_path, minb):
    """rs_main4<true, 3/5/6> (TSDRGPU_RS_MINB) give the oracle's bits at the production ratios, with magnitudes, at every phase."""
    path = str(tmp_path / "minb.npz")
    env = dict(os.environ, TSDRGPU_RS_MINB=minb)
    env.pop("TSDRGPU_RS_V1", None)
    p = subprocess.run([sys.executable, "-c", f"from tests.test_resampler_sweep import minb_case; minb_case({path!r}); print('case ok')"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert p.returncode == 0 and "case ok" in p.stdout, (p.stdout[-1500:], p.stderr[-2500:])
    got = np.load(path)
    for name in MINB_RATIOS:
        calls = sweep_calls(name)
        _, mag = stream(calls, 7)
        want, want_state = oracle_stream(O, mag, calls)
        for j in range(len(PHASES)):
            assert_same(got[f"{name}_{j}_px"], want, f"MINB={minb} {name} phases {PHASES[j]}")
            assert_same(got[f"{name}_{j}_mag"], mag, f"MINB={minb} {name} magnitudes")
            assert tuple(got[f"{name}_{j}_state"]) == (want_state[0], want_state[1], 1.0)
