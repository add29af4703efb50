"""Kernel time of the frame stage's row/column collapse (fs_collapse) and re-centring (fs_shift), one process.

Prints one JSON line with
  * the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after the timed work;
  * per shape (cfg2 740x1125, cfg5 1481x1125, cfg1 507x525), 64-frame batches of drifting video-like frames through the frame
    stage in the benchmark's flags (autoshift, low-pass before sync; side stream off so that every kernel's event pair times that
    kernel alone): after warm-up, ROUNDS rounds of LAUNCHES batches each, the library's per-kernel profile (CUDA events around
    every launch, as bench.py's per-kernel pass) -> ms per launch and GB/s against 4 B per pixel (collapse: one read of the
    frame) and 8 B per pixel (shift: one read, one write), the bytes bench.py's roofline counts for these kernels.
GPU only:  python profiles/studies/collapse_shift_timing.py
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

SHAPES = {"cfg2": (25_000_000, 1125), "cfg5": (50_000_000, 1125), "cfg1": (8_000_000, 525)}
NFRAMES = 64
WARMUP = 5
ROUNDS = 3
LAUNCHES = 20
KERNELS = {"fs_collapse": 4, "fs_shift": 8}          # algorithmic bytes per pixel


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def profile(gpu, fn):
    lib = gpu._lib
    gpu.chk(lib.tsdrgpu_profile_enable(gpu._h, 1))
    fn()
    cap = 64
    names = C.create_string_buffer(48 * cap)
    ms = (C.c_double * cap)()
    cnt = (C.c_uint64 * cap)()
    n = C.c_int(0)
    gpu.chk(lib.tsdrgpu_profile_collect(gpu._h, names, ms, cnt, cap, C.byref(n)))
    gpu.chk(lib.tsdrgpu_profile_enable(gpu._h, 0))
    return {names.raw[48 * i: 48 * (i + 1)].split(b"\0")[0].decode(): (ms[i], cnt[i]) for i in range(n.value)}


def shape_run(gpu, name):
    import torch
    from tempestsdr_b200 import synth
    from tempestsdr_b200.api import PostProcessFlags
    fs, h = SHAPES[name]
    w = int(2 * (fs / (60.0 * h)))                     # the frame width bench.py derives (TSDRLibrary.c:540-550)
    frames = np.concatenate([synth.video_like_frame(w, h, seed=k, shift_x=(60 + 5 * k) % w, shift_y=(20 + k) % h) for k in range(NFRAMES)])
    x = torch.from_numpy(frames).cuda()
    out = torch.empty_like(x)
    pg = gpu.post_processor()
    pg.set_overlap(False)
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True)

    def batches(k):
        for _ in range(k):
            pg.process(x, w, h, 0.0, 0.1, flags, out=out, want_results=False)
        torch.cuda.synchronize()

    batches(WARMUP)
    res = {"width": w, "height": h, "frames": NFRAMES, "ms": {k: [] for k in KERNELS}}
    for _ in range(ROUNDS):
        prof = profile(gpu, lambda: batches(LAUNCHES))
        for k in KERNELS:
            tot, cnt = prof[k]
            assert cnt == LAUNCHES, (k, cnt)
            res["ms"][k].append(tot / cnt)
    npix = w * h * NFRAMES
    res["gbps"] = {k: [round(b * npix / (ms * 1e6), 1) for ms in res["ms"][k]] for k, b in KERNELS.items()}
    return res


def main():
    from tempestsdr_b200 import api
    result = {"hardware": gpu_info(), "shapes": {}}
    gpu = api.Context(0)
    for name in SHAPES:
        result["shapes"][name] = shape_run(gpu, name)
    result["hardware_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
