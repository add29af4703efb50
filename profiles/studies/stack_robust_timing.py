"""The glitch-tolerant stack ("robust:32") against "track:32" at 740 x 1125 (cfg2) and 1481 x 1125: what one frame costs when
no tile changed, when a band of lines is corrupted, and when the whole frame is noise (a glitch frame).

Each case is one 9-frame batch run after tsdrgpu_stack_reset: a restart frame, 7 frames of a static picture
(synth.video_like_frame, shifted by 1 px per frame, noise sigma 0.1) that settle every tile's level, and a last frame that is
  * "static": the same picture again (no tile changed);
  * "band": the picture with a third of its lines replaced by uniform noise (track restarts those tiles, robust holds them);
  * "noise": uniform noise (track restarts every tile after searching it; robust searches every tile and holds the frame).
CUDA events around BATCHES batches (reset + run), the cases and modes alternating, ROUNDS rounds -> ms per batch.  The cost of
the last frame over a static one is (case - static) + static / 9.  Prints one JSON line with the GPU's name and power limit,
read (read-only nvidia-smi queries) in the same call.
GPU only:  python profiles/studies/stack_robust_timing.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

ROUNDS = 5
BATCHES = 10
MODES = ("track:32", "robust:32")
CASES = ("static", "band", "noise")
SHAPES = ((740, 1125), (1481, 1125))


def smi(fields):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]


def frames_of(case, w, h):
    import numpy as np
    from tempestsdr_b200 import synth
    rng = np.random.default_rng(2)
    pic = synth.video_like_frame(w, h, seed=1, noise=0.0).reshape(h, w)
    seq = [np.roll(pic.reshape(-1), k) + rng.normal(0, 0.1, w * h) for k in range(9)]
    if case == "band":
        seq[8].reshape(h, w)[h // 3:2 * h // 3] = rng.uniform(0, 1, (2 * h // 3 - h // 3, w))
    elif case == "noise":
        seq[8] = rng.uniform(0, 1, w * h)
    return np.concatenate(seq).astype(np.float32)


def main():
    import numpy as np
    import torch
    from tempestsdr_b200 import api
    name, power, sm_max = smi("name,power.limit,clocks.max.sm")
    gpu = api.Context(0)
    result = {"hardware": {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max}, "shapes": {}}
    for w, h in SHAPES:
        data = {c: torch.from_numpy(frames_of(c, w, h)).cuda() for c in CASES}
        out = torch.empty_like(data["static"])
        stacks, last = {}, {}
        for spec in MODES:
            stacks[spec] = gpu.stack()
            stacks[spec].set(spec)
            for c in CASES:
                stacks[spec].reset()
                _, recs = stacks[spec].run(data[c], w, h, out=out)
                last[f"{spec} {c}"] = {"restarted_tiles": recs[-1].changed}
                if spec.startswith("robust"):
                    held, gated, hold = stacks[spec].robust_counts()
                    last[f"{spec} {c}"].update(held_tiles=held, gated_pixels=gated, glitch_frame=hold)
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
        result["shapes"][f"{w}x{h}"] = {"tiles": ((w + 15) // 16) * ((h + 15) // 16), "ms_per_batch": ms,
                                        "last_frame_ms": frame, "last_frame": last}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
