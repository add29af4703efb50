"""Kernel time of the frame stage's low-pass and collapse with motion blur 0 (the collapse normalises the raw frames on load, then
the two gated launches fs_redo_lowpass / fs_redo_collapse) against motion blur 1e-6 (the separate fs_norm_lowpass and fs_collapse),
one process.

Prints one JSON line with
  * the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after the timed work;
  * per shape (cfg2 740x1125, cfg5 1481x1125, cfg1 507x525) and motion blur, 64-frame batches of drifting video-like frames through
    the frame stage in the benchmark's flags (autoshift, low-pass before sync; side stream off so that every kernel's event pair
    times that kernel alone): after warm-up, ROUNDS rounds of LAUNCHES batches each, the library's per-kernel profile -> ms per
    launch of every kernel of the low-pass and collapse, and their sum.
GPU only:  python profiles/studies/norm_in_collapse_timing.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from collapse_shift_timing import SHAPES, gpu_info, profile  # noqa: E402

NFRAMES = 64
WARMUP = 5
ROUNDS = 3
LAUNCHES = 20
KERNELS = ["fs_norm_lowpass", "fs_collapse", "fs_redo_lowpass", "fs_redo_collapse"]
BLURS = {"blur0": 0.0, "blur1e-6": 1e-6}


def shape_run(gpu, name, mb):
    import torch
    from tempestsdr_b200 import synth
    from tempestsdr_b200.api import PostProcessFlags
    fs, h = SHAPES[name]
    w = int(2 * (fs / (60.0 * h)))
    frames = np.concatenate([synth.video_like_frame(w, h, seed=k, shift_x=(60 + 5 * k) % w, shift_y=(20 + k) % h) for k in range(NFRAMES)])
    x = torch.from_numpy(frames).cuda()
    out = torch.empty_like(x)
    pg = gpu.post_processor()
    pg.set_overlap(False)
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True)

    def batches(k):
        for _ in range(k):
            pg.process(x, w, h, mb, 0.1, flags, out=out, want_results=False)
        torch.cuda.synchronize()

    batches(WARMUP)
    res = {"width": w, "height": h, "frames": NFRAMES, "motionblur": mb, "ms": {}}
    for _ in range(ROUNDS):
        prof = profile(gpu, lambda: batches(LAUNCHES))
        for k in KERNELS:
            if prof.get(k, (0.0, 0))[1]:                 # names of the other motion blur's kernels stay listed with no launches
                tot, cnt = prof[k]
                assert cnt == LAUNCHES, (k, cnt)
                res["ms"].setdefault(k, []).append(tot / cnt)
    res["sum_ms"] = [sum(v[r] for v in res["ms"].values()) for r in range(ROUNDS)]
    return res


def main():
    from tempestsdr_b200 import api
    result = {"hardware": gpu_info(), "shapes": {}}
    gpu = api.Context(0)
    for name in SHAPES:
        result["shapes"][name] = {b: shape_run(gpu, name, mb) for b, mb in BLURS.items()}
    result["hardware_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
