"""GPU: the frame stage's row/column collapse and re-centring on 16-byte rows against the oracle, bit for bit.

When a frame's rows start on 16-byte boundaries (w % 4 == 0, aligned base) the collapse streams 2-D boxes through tensor-map
copies (column CTAs: 128 columns x 16 rows; row CTAs: 32 columns x 128 rows, 128-byte swizzle) and the re-centring copies whole
float4s, selecting between two aligned source float4s by dx mod 4.  These tests cover what those paths do differently from the
scalar ones: widths and heights that leave ragged boxes (the tensor map's zero fill must never enter a sum), every residue of
dx mod 4, the vertical wrap and dy = 0, and the fall-back to the scalar kernels when a base is not 16-byte aligned.
"""
import numpy as np
import pytest
import torch

from tempestsdr_b200 import synth
from tests.test_gpu_parity import CFGS, assert_same_bits, dev
from tests.test_production_batches import O, assert_same_result, gpu, results_of, run_async  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _frame(w, h, seed):
    if w > 8 and h > 8:
        f = synth.video_like_frame(w, h, seed=seed).reshape(h, w)
    else:
        f = np.random.default_rng(seed).uniform(-1, 1, (h, w)).astype(np.float32)
    f = f.copy()
    f[:, w // 2] = -0.0                                   # a column and a row of negative zeros
    f[h // 2, :] = -0.0
    return np.ascontiguousarray(f.reshape(-1))


@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "base+4B"])
@pytest.mark.parametrize("w", [740, 36, 4])
@pytest.mark.parametrize("h", [1125, 17, 1])
def test_average_v_h_ragged_boxes(gpu, O, w, h, offset):
    """dsp_average_v_h at aligned widths that are not multiples of the boxes' 32 / 128 columns and heights that are not
    multiples of their 16 / 128 rows; offset by one float the same frame takes the scalar cp.async kernel."""
    g = _frame(w, h, seed=w * 7 + h)
    buf = torch.zeros(w * h + 4, dtype=torch.float32, device="cuda")
    buf[offset:offset + w * h] = dev(g)
    wb, hb = gpu.dsp_average_v_h(buf[offset:offset + w * h], w, h)
    wr, hr = O.average_v_h(g, w, h)
    assert_same_bits(wb, wr, f"colsum {w}x{h}")
    assert_same_bits(hb, hr, f"rowsum {w}x{h}")


NF = 64


def _batch(O):
    """64 frames of 740x1125 whose detected x_dx moves by ~5 per frame (every residue mod 4) and whose vertical offset starts at
    small values: dy = 0 on one frame, rows wrapping at the bottom on the others."""
    fs, hgt, fv = CFGS["cfg2"]
    w, _, _ = O.geometry(fs, hgt, fv)
    frames = [synth.video_like_frame(w, hgt, seed=500 + k, shift_x=(60 + 5 * k) % w, shift_y=20) for k in range(NF)]
    po = O.postprocessor(fs, hgt, fv, 1, 0)
    want = [po.run(f, w, hgt, 0.0, 0.1, 1, 0) for f in frames]
    return w, hgt, frames, want


@pytest.fixture(scope="module")
def batch(O):
    return _batch(O)


def _run(gpu, w, h, frames, offset):
    from tempestsdr_b200.api import PostProcessFlags
    n = w * h
    src = torch.zeros(NF * n + 4, dtype=torch.float32, device="cuda")
    dst = torch.zeros(NF * n + 4, dtype=torch.float32, device="cuda")
    x = src[offset:offset + NF * n]
    x.copy_(dev(np.concatenate(frames)))
    out = dst[offset:offset + NF * n]
    pg = gpu.post_processor()
    pg.set_overlap(True)
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True)
    res, _ = run_async(gpu, pg, x, NF, w, h, 0.0, flags, out)
    pg.join(); torch.cuda.synchronize()
    return out.cpu().numpy().reshape(NF, -1), results_of(res, NF)


@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "base+4B"])
def test_64_frame_batch_every_dx_residue(gpu, batch, offset):
    """tsdrgpu_framestage_run_async over 64 cfg2 frames (what the benchmark runs), default stage order with the side stream:
    every frame and every sync result bit-exact.  Aligned, the batch takes fs_collapse_tiles and fs_shift4; with input and
    output one float off their 16-byte boundary, the re-centring falls back to the scalar kernel (and the fused
    normalise/low-pass to its scalar path) with identical results."""
    w, h, frames, want = batch
    got, rs = _run(gpu, w, h, frames, offset)
    for k in range(NF):
        wf, wr = want[k]
        assert_same_bits(got[k], wf, f"frame {k}")
        assert_same_result(rs[k], wr, f"frame {k}")
    xs = [r.x_dx for r in rs]
    ys = [r.y_dx for r in rs]
    assert {x % 4 for x in xs} == {0, 1, 2, 3}, xs
    assert 0 in ys and any(y > 0 for y in ys), ys
