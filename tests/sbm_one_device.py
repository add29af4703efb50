"""All H ranks of a superbandwidth group on ONE device, through a list of stitches (tests/test_superb_sweep.py).

    python -m tests.sbm_one_device H            the sweep's cases for H ranks
    python -m tests.sbm_one_device 4 full       BASELINE configs[3]'s hop size: 4 x 2^21

Every rank has a context and a stream of its own; the process is started with CUDA_DEVICE_MAX_CONNECTIONS=32 so that every
rank's stream gets a hardware queue of its own.  For every stitch:
  * the lags equal the compiled reference's (superb_ondataready), the one-GPU path's (tsdrgpu_superb_stitch) and round 1's
    (tsdrgpu_superb_lags) on the same hops;
  * the magnitudes are within C_OWN_MAX / C_OWN_RMS units of the model of the sharded dataflow (superb_model.stitch_sharded) and
    within that plus the pinned deviation of |superb_model.stitch_reference| (SHARDED_DEVIATION).
Units: fft_model.rounding_units over the H N points.  The measured units of every case are printed.

With TSDRGPU_FFT_TRUE_DFT=1 (exact stage angles) both models are taken with exact angles, and the reference model with the
reference's angles must be missed: that is the difference the bound has to see at 2^23 points."""
import ctypes as C
import os
import sys

import numpy as np
import torch

from oracle import oracle as orc
from tempestsdr_b200 import api, superband
from tests import fft_model as fm
from tests import superb_model as sm


TRUE_DFT = os.environ.get("TSDRGPU_FFT_TRUE_DFT") is not None


def case(pairs, sif, lags, seed, hop0="copy", in_place=False):
    """One stitch: hop q's correlation peak at lags[q] (in the nd-point correlation this pairs / sif give)."""
    return dict(pairs=pairs, sif=sif, lags=lags, seed=seed, hop0=hop0, in_place=in_place)


def sweep_cases(H):
    """Per root (0, H/2, H - 1): three stitches in a row, N = 2^16, 2^12, 2^16 (re-prepared, epochs stepped), both hop-0 modes,
    copy-out and in-place window, nd = N/2 (sif 8000, 700) and nd = N (sif 2^11, 2^15), the last hop longer than a power of two.
    Lags from every class: 0, 1, nd/2 - 1, nd/2, nd/2 + 1, nd - 2, nd - 1, spread over the ranks."""
    out = []
    for k, root in enumerate(sorted({0, H // 2, H - 1})):
        def spread(nd, j):
            cls = [1, nd - 1, nd // 2, nd // 2 - 1, nd // 2 + 1, nd - 2, 0, 3]
            return [0] + [cls[(j + q) % len(cls)] for q in range(H - 1)]
        out.append((root, [
            case(1 << 16, 8000, spread(1 << 15, k), seed=10 * k + 1, hop0="copy", in_place=False),
            case(1 << 12, 1 << 11, spread(1 << 12, k + 2), seed=10 * k + 2, hop0="pull", in_place=True),
            case((1 << 16) + 777, 1 << 15, spread(1 << 16, k + 4), seed=10 * k + 3, hop0="pull" if k % 2 == 0 else "copy",
                 in_place=k % 2 == 1),
        ]))
    return out


FULL_CASES = [(0, [case(4_166_660, 416_666, [0, 1234, (1 << 20) - 77, (1 << 19) + 1], seed=19)])]


def refusals(groups, d_hop, sif):
    """One rank called with arguments every rank refuses (N < 64; N > the window's n_max): an error before anything is enqueued."""
    g = groups[-1]
    for pairs in (32, 63, 2 * groups[0].n_max_pairs):
        hn = C.c_uint32(0)
        rc = g.ctx._lib.tsdrgpu_superb_mgpu_stitch(g._h, g.ctx.stream, d_hop.data_ptr(), None, pairs, sif, None, C.byref(hn))
        assert rc != 0, f"a stitch of {pairs} pairs was accepted"


def run(H: int, cases, max_pairs: int) -> None:
    O = orc.best()
    ctxs = [api.Context(0) for _ in range(H)]
    streams = [torch.cuda.Stream() for _ in range(H)]
    worst = [0.0, 0.0, 0.0, 0.0]
    for root, stitches in cases:
        groups = superband.SuperbGroup.local(ctxs, max_pairs, root=root)
        for g in groups:
            g.n_max_pairs = max_pairs
        for i, c in enumerate(stitches):
            pairs, sif = c["pairs"], c["sif"]
            n = fm.getrealsize(pairs)
            nd = sm.correlation_pairs(2 * n, sif)
            hops = sm.shifted_hops(pairs, [sm.shift_for_lag(l, nd) for l in c["lags"]], seed=c["seed"])
            want_iq, offs = O.superb_ondataready(hops, sif)
            assert [int(o) // 2 for o in offs] == c["lags"], (list(offs), c["lags"])
            d_hops = [torch.from_numpy(h).cuda() for h in hops]
            torch.cuda.synchronize()
            if i == len(stitches) - 1 and root == cases[-1][0]:
                refusals(groups, d_hops[-1], sif)
            out = None
            for r in range(H):
                with torch.cuda.stream(streams[r]):
                    res = groups[r].stitch(d_hops[r], sif, hop0=d_hops[0] if c["hop0"] == "copy" else None, in_place=c["in_place"])
                    out = res if res is not None else out
            torch.cuda.synchronize()
            lags = groups[0].lags()
            assert all(g.lags() == lags for g in groups), [g.lags() for g in groups]
            assert [2 * l for l in lags] == [int(o) for o in offs], (lags, list(offs))
            got = out.cpu().numpy().astype(np.float64)
            # the one-GPU path and round 1's lag search on the same hops
            _, one = ctxs[0].superb_stitch(d_hops, sif)
            blocks = [superband.local_block(ctxs[0], h, sif) for h in d_hops]
            r1 = superband.lags_from_gathered(ctxs[0], torch.cat([b[0] for b in blocks]), H, blocks[0][1], blocks[0][2])
            assert one == [int(o) for o in offs] and r1 == lags, (one, r1, lags)
            own = sm.stitch_sharded(hops, lags, true_dft=TRUE_DFT)
            ref, _ = sm.stitch_reference(hops, sif, offsets=[int(o) for o in offs], true_dft=TRUE_DFT)
            ref = np.abs(ref)
            if TRUE_DFT:
                angles = np.abs(sm.stitch_reference(hops, sif, offsets=[int(o) for o in offs])[0])
                ua, dv = sm.units(got, angles, H * n), sm.sharded_deviation(H, n)
                print(f"exact angles vs the reference's angles: max {ua[0]:.3f} rms {ua[1]:.3f}")
                assert ua[0] > sm.C_OWN_MAX + dv[0], "exact stage angles within the bound of the reference's"
            assert got.shape == own.shape, (got.shape, own.shape)
            u_own, u_ref = sm.units(got, own, H * n), sm.units(got, ref, H * n)
            dev = (0.7, 0.7) if TRUE_DFT else sm.sharded_deviation(H, n)     # exact angles: the float32 twiddle tables only
            print(f"H={H} root={root} N=2^{fm.log2_of(n)} nd=2^{fm.log2_of(nd)} hop0={c['hop0']} in_place={c['in_place']} lags={lags}: "
                  f"vs own model max {u_own[0]:.3f} rms {u_own[1]:.3f}; vs reference model max {u_ref[0]:.3f} rms {u_ref[1]:.3f} "
                  f"(pinned deviation {dev[0]:.3f} / {dev[1]:.3f})")
            worst = [max(worst[0], u_own[0]), max(worst[1], u_own[1]), max(worst[2], u_ref[0] - dev[0]), max(worst[3], u_ref[1] - dev[1])]
            assert u_own[0] <= sm.C_OWN_MAX and u_own[1] <= sm.C_OWN_RMS, u_own
            assert u_ref[0] <= sm.C_OWN_MAX + dev[0] and u_ref[1] <= sm.C_OWN_RMS + dev[1], (u_ref, dev)
        for g in groups:
            g.close()
    print(f"worst H={H}: own model max {worst[0]:.3f} rms {worst[1]:.3f}; reference model beyond the pinned deviation max {worst[2]:.3f} rms {worst[3]:.3f}")
    print("sbm ok")


if __name__ == "__main__":
    H = int(sys.argv[1])
    full = len(sys.argv) > 2 and sys.argv[2] == "full"
    cases = FULL_CASES if full else sweep_cases(H)
    run(H, cases, max(c["pairs"] for _, cs in cases for c in cs))
