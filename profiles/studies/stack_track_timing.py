"""The motion-tracking stack ("track:32") against "adapt:32" at cfg2's 740 x 1125: what one frame costs when no tile changed,
when a region scrolls, and when every tile changed.

Each case is one 9-frame batch run after tsdrgpu_stack_reset: a restart frame, 7 frames of a static picture
(synth.video_like_frame, shifted by 1 px per frame, noise sigma 0.1) that settle every tile's level, and a last frame that is
  * "static": the same picture again (no tile changed);
  * "scroll": the picture with a 512 x 384 text region at (100, 300) moved up by one 12-line row, a new row at its bottom;
  * "cut": an unrelated picture (every tile changed: about 3 300 tiles x 2 145 candidates x 64 words of search).
CUDA events around BATCHES batches (reset + run), the cases and modes alternating, ROUNDS rounds -> ms per batch.  The cost of
the last frame over a static one is (case - static) + static / 9; the records give the restarted tiles of the last frame and
the vectors the tiles carried.  Prints one JSON line with the GPU's name and power limit, read (read-only nvidia-smi queries) in
the same call.
GPU only:  python profiles/studies/stack_track_timing.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

ROUNDS = 5
BATCHES = 10
MODES = ("adapt:32", "track:32")
CASES = ("static", "scroll", "cut")


def smi(fields):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]


def frames_of(case, w, h):
    import numpy as np
    from tempestsdr_b200 import synth
    rng = np.random.default_rng(2)
    base = synth.video_like_frame(w, h, seed=1, noise=0.0).reshape(h, w)
    text = np.full((384 + 12, 512), 0.1, np.float32)
    for r in range(33):
        for c in range(64):
            g = rng.uniform(size=(8, 5)) < 0.3
            text[12 * r + 2:12 * r + 10, 8 * c + 1:8 * c + 6][g] = 0.9
    pic = base.copy()
    pic[300:684, 100:612] = text[:384]
    last = pic
    if case == "scroll":
        last = pic.copy()
        last[300:684, 100:612] = text[12:396]
    elif case == "cut":
        last = synth.video_like_frame(w, h, seed=5, noise=0.0).reshape(h, w)
    seq = [pic] * 8 + [last]
    return np.concatenate([np.roll(p.reshape(-1), k) + rng.normal(0, 0.1, w * h).astype(np.float32)
                           for k, p in enumerate(seq)]).astype(np.float32)


def main():
    import numpy as np
    import torch
    os.environ["BENCH_SHAPE"] = "cfg2"
    import bench
    from tempestsdr_b200 import api
    name, power, sm_max = smi("name,power.limit,clocks.max.sm")
    gpu = api.Context(0)
    w, h = bench.geometry(), bench.HEIGHT
    data = {c: torch.from_numpy(frames_of(c, w, h)).cuda() for c in CASES}
    out = torch.empty_like(data["static"])
    stacks, last = {}, {}
    for spec in MODES:
        stacks[spec] = gpu.stack()
        stacks[spec].set(spec)
        for c in CASES:
            stacks[spec].reset()
            _, recs = stacks[spec].run(data[c], w, h, out=out)
            carried = int(np.any(stacks[spec].vectors(w, h) != 0, axis=2).sum()) if spec.startswith("track") else 0
            last[f"{spec} {c}"] = {"restarted_tiles": recs[-1].changed, "carried_tiles": carried}
    torch.cuda.synchronize()
    ms = {f"{s} {c}": [] for s in MODES for c in CASES}
    for _ in range(ROUNDS):
        for c in CASES:
            for spec in MODES:
                st = stacks[spec]
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(BATCHES):
                    gpu._lib.tsdrgpu_stack_reset(st._h)
                    gpu._lib.tsdrgpu_stack_run(st._h, gpu.stream, data[c].data_ptr(), out.data_ptr(), w, h, 9, None)
                b.record()
                torch.cuda.synchronize()
                ms[f"{spec} {c}"].append(a.elapsed_time(b) / BATCHES)
    best = {k: min(v) for k, v in ms.items()}
    frame = {k: best[k] - best[f"{k.split()[0]} static"] + best[f"{k.split()[0]} static"] / 9 for k in ms}
    print(json.dumps({"hardware": {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max},
                      "width": w, "height": h, "tiles": ((w + 15) // 16) * ((h + 15) // 16), "ms_per_batch": ms,
                      "last_frame_ms": frame, "last_frame": last}))


if __name__ == "__main__":
    main()
