"""Stitch time of the coherent superbandwidth stitch beside the reference's one-GPU stitch (tsdrgpu_superb_stitch), on the H100.

Shapes: 4 hops of 2^22 and of 2^21 pairs (25 MS/s at 60 Hz records 10 frames of 416 666 pairs, 2^21 used per hop; 2^22 is the
next power of two).  CUDA events around each call, the L2 flushed (a 256 MB write) before every repetition, the two stitches
alternated.  Prints the card's name and power limit from the same run.  Run: python profiles/studies/superband_coherent_timing.py
"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tempestsdr_b200 import api, synth  # noqa: E402
from tests import superband_coherent_model as sm  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main(reps=20):
    ctx = api.Context(0)
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    print(f"card: {card()}")
    for log2n in (21, 22):
        n, H, o = 1 << log2n, 4, 25
        d = sm.spacing(n, o)
        hops = [torch.from_numpy(synth.noise_iq(n, seed=10 + i)).cuda() for i in range(H)]
        sif = 416_666
        times = {"coherent": [], "reference": []}
        out = torch.empty(2 * H * n, dtype=torch.float32, device="cuda")
        for name in times:                                                   # warm-up: tables, scratch
            (ctx.superband_stitch_coherent(hops, d, out=out) if name == "coherent" else ctx.superb_stitch(hops, sif))
        torch.cuda.synchronize()
        for _ in range(reps):
            for name in times:
                flush.fill_(1.0)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                if name == "coherent":
                    ctx.superband_stitch_coherent(hops, d, out=out)
                else:
                    ctx.superb_stitch(hops, sif)                             # synchronises at its end (reads the lags back)
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        for name, t in times.items():
            t = np.array(t)
            print(f"H={H} N=2^{log2n} {name:9s}: median {np.median(t):8.3f} ms  min {t.min():8.3f}  max {t.max():8.3f}  ({reps} reps)")
    ctx.close()


if __name__ == "__main__":
    main()
