"""GPU: the default-order frame stage with motion blur 0, where the collapse normalises the raw frames on load and a certificate
decides on the device whether the batch is redone literally (DESIGN 5.2).

Every case runs 64-frame batches through tsdrgpu_framestage_run_async with the side-stream overlap on, at cfg2 with the input
16-byte aligned (fs_collapse_tiles) and one float off (fs_collapse), and at cfg1 (odd width: fs_collapse).  The same batches run
once more with TSDRGPU_NO_FUSE=1, which takes the separate auto-gain, low-pass and collapse kernels; every delivered frame and
every frame result must have the same bits (NaN payloads included).  The cases are the values of v for which the identity
fails and the screen states that must carry across paths:
  * negzero: a first batch with minimum 0 and raw -0.0f pixels, so v == -0.0f and the literal screen value is +0.0f;
  * tiny:    pixel 0 a huge marker, so the span is huge and small negative x - lastmin underflow to -0.0f;
  * nan0 / nan31 / nan63: a NaN pixel in frame 0, 31 or 63, then a clean batch (the NaN stays in the screen);
  * inf:     +inf in pixel 0 of every frame (infinite span);
  * blur:    clean batches at motion blur 0, 0.3, 0 (the screen stays continuous across paths);
  * clean:   two clean batches.
The negzero case is also checked frame by frame against the oracle.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NF = 64
CASES = ["negzero", "tiny", "nan0", "nan31", "nan63", "inf", "blur", "clean"]
LAYOUTS = [("cfg2", 0), ("cfg2", 1), ("cfg1", 0)]           # (shape, offset of the input in floats)


def geometry(name):
    from tests.test_gpu_parity import CFGS
    fs, h, fv = CFGS[name]
    return int(2 * (fs / (fv * h))), h


def case_batches(case, w, h):
    """[(frames (NF, w*h) float32, motion blur)] of one case."""
    from tempestsdr_b200 import synth

    def frames(seed):
        return np.stack([synth.video_like_frame(w, h, seed=seed + k, shift_x=(60 + 3 * k) % w, shift_y=(20 + k) % h).ravel()
                         for k in range(NF)]).astype(np.float32)
    a, b = frames(1000), frames(2000)
    if case == "negzero":
        a -= a.min(axis=1, keepdims=True)                     # minimum exactly +0.0f, lastmin stays +0.0f
        a[:, 7::97] = np.float32(-0.0)
        return [(a, 0.0), (b, 0.0)]
    if case == "tiny":
        a[:, 0] = np.float32(3e38)                            # a marker: seeds max, span ~3e37
        a[:, 11::53] = np.float32(-1e-9)                      # minimum; (x - lastmin) / span underflows to -0.0f
        return [(a, 0.0), (b, 0.0)]
    if case.startswith("nan"):
        a[int(case[3:]), 5000] = np.float32("nan")
        return [(a, 0.0), (b, 0.0)]
    if case == "inf":
        a[:, 0] = np.float32("inf")
        return [(a, 0.0), (b, 0.0)]
    if case == "blur":
        return [(a, 0.0), (b, 0.3), (frames(3000), 0.0)]
    return [(a, 0.0), (b, 0.0)]


def run_all(out_path):
    """Runs every case and layout in this process; writes {case/shape/offset: [[sha of frames, sha of results] per batch]}."""
    import torch
    from tempestsdr_b200 import api
    from tempestsdr_b200.api import PostProcessFlags
    from tests.test_production_batches import run_async
    gpu = api.Context(0)
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True)
    digests = {}
    for shape, off in LAYOUTS:
        w, h = geometry(shape)
        for case in CASES:
            pg = gpu.post_processor()
            pg.set_overlap(True)
            keep = []
            for frames, mb in case_batches(case, w, h):
                buf = torch.empty(frames.size + 4, dtype=torch.float32, device="cuda")
                x = buf[off:off + frames.size]
                x.copy_(torch.from_numpy(frames.ravel()))
                out = torch.empty(frames.size, dtype=torch.float32, device="cuda")
                keep.append((buf, out) + run_async(gpu, pg, x, NF, w, h, mb, flags, out))
            pg.join(); torch.cuda.synchronize()
            digests[f"{case}/{shape}/{off}"] = [[hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest(),
                                                 hashlib.sha256(res.numpy().tobytes()).hexdigest(), list(ag)] for _, out, res, ag in keep]
            if case == "negzero" and off == 0:
                np.save(out_path + f".{shape}.negzero.npy", keep[0][1].cpu().numpy())
            del keep, pg
    json.dump(digests, open(out_path, "w"))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("norm_in_collapse")
    got = {}
    for mode in ("fast", "literal"):
        env = dict(os.environ)
        env.pop("TSDRGPU_NO_FUSE", None)
        if mode == "literal":
            env["TSDRGPU_NO_FUSE"] = "1"
        path = str(d / f"{mode}.json")
        r = subprocess.run([sys.executable, os.path.abspath(__file__), path], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0, r.stderr[-3000:]
        got[mode] = (path, json.load(open(path)))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("shape,off", LAYOUTS, ids=[f"{s}-off{o}" for s, o in LAYOUTS])
@pytest.mark.parametrize("case", CASES)
def test_same_bits_as_the_separate_kernels(runs, case, shape, off):
    key = f"{case}/{shape}/{off}"
    fast, literal = runs["fast"][1][key], runs["literal"][1][key]
    assert len(fast) == len(literal)
    for b, (f, l) in enumerate(zip(fast, literal)):
        assert f[0] == l[0], f"{key}: frames of batch {b} differ"
        assert f[1] == l[1], f"{key}: frame results of batch {b} differ"
        assert f[2] == l[2], f"{key}: auto-gain reports of batch {b} differ"


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["cfg2", "cfg1"])
def test_negative_zero_batch_against_the_oracle(runs, shape):
    """The first negzero batch, frame by frame against the oracle: the literal screen is +0.0f where v is -0.0f."""
    from oracle import oracle as orc
    from tests.test_gpu_parity import CFGS, assert_same_bits
    O = orc.best()
    fs, h, fv = CFGS[shape]
    w, _, _ = O.geometry(fs, h, fv)
    assert (w, h) == geometry(shape)
    po = O.postprocessor(fs, h, fv, 1, 0)
    frames, mb = case_batches("negzero", w, h)[0]
    got = np.load(runs["fast"][0] + f".{shape}.negzero.npy").reshape(NF, -1)
    for k in range(NF):
        wf, _ = po.run(frames[k], w, h, mb, 0.1, 1, 0)
        assert_same_bits(got[k], wf, f"{shape} negzero frame {k}")


if __name__ == "__main__":
    run_all(sys.argv[1])
