"""Richardson-Lucy deconvolution along the lines (deblur "rl:1" and "rl:4:64"): tsdrgpu_deblur on its own, beside the stack.

Prints one JSON line with
  * the GPU's name and power limit, read (read-only nvidia-smi queries) in the same call as the timings;
  * per shape (cfg2, cfg5, cfg1), the fs_deblur kernel over a 64-frame batch of that shape's frames (synth.video_like_frame with
    noise sigma 0.1), for sigma = 1 with I = 20 and sigma = 4 with I = 64: CUDA events around 5 batches after warm-up, three
    rounds -> ms per batch; beside it tsdrgpu_stack_run ("align:32") over the same batch;
  * the FP32 work each setting needs at least, counted from the definition: per pixel and iteration two correlations of 2R + 1
    multiplies and 2R adds, three more multiplies, one max and one division (counted as one operation here, though it costs
    several), and the bound that gives at the H100 SXM's data-sheet 67 TFLOP/s FP32.
GPU only:  python profiles/studies/deblur_timing.py
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

FRAMES = 64
ROUNDS = 3
BATCHES = 5
SETTINGS = {"rl:1": (100, 20), "rl:4:64": (400, 64)}
FP32_PER_S = 67e12


def smi(fields):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]


def shape_run():
    """One shape (BENCH_SHAPE), in a process of its own because bench.py fixes its shape at import."""
    import numpy as np
    import torch
    import bench
    from tempestsdr_b200 import api, synth
    gpu = api.Context(0)
    w = bench.geometry()
    n = w * bench.HEIGHT
    base = synth.video_like_frame(w, bench.HEIGHT, seed=1, noise=0.0)
    rng = np.random.default_rng(2)
    frames = torch.from_numpy(np.concatenate([np.roll(base, k) + rng.normal(0, 0.1, n).astype(np.float32)
                                              for k in range(FRAMES)]).astype(np.float32)).cuda()
    out = torch.empty_like(frames)

    def timed(launch):
        for _ in range(2):
            launch()
        torch.cuda.synchronize()
        ms = []
        for _ in range(ROUNDS):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(BATCHES):
                launch()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / BATCHES)
        return ms

    res = {"shape": bench.SHAPE, "width": w, "pixels_per_frame": n, "frames": FRAMES, "deblur": {}}
    for spec, (sc, it) in SETTINGS.items():
        # tsdrgpu_deblur synchronises its stream after the launch, so each call is one whole batch
        ms = timed(lambda: gpu.chk(gpu._lib.tsdrgpu_deblur(gpu._h, gpu.stream, frames.data_ptr(), out.data_ptr(), w, bench.HEIGHT,
                                                            FRAMES, sc, it)))
        r = (3 * sc + 99) // 100
        flops = FRAMES * n * it * (2 * (4 * r + 1) + 5)
        res["deblur"][spec] = {"ms": ms, "fp32_ops": flops, "fp32_bound_ms": flops / FP32_PER_S * 1e3,
                               "share_of_fp32_bound": flops / FP32_PER_S * 1e3 / min(ms)}
    st = gpu.stack()
    st.set("align:32")
    res["stack_align32_ms"] = timed(lambda: gpu._lib.tsdrgpu_stack_run(st._h, gpu.stream, frames.data_ptr(), out.data_ptr(), w,
                                                                         bench.HEIGHT, FRAMES, None))
    return res


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--shape":
        print(json.dumps(shape_run()))
        return
    name, power, sm_max = smi("name,power.limit,clocks.max.sm")
    result = {"hardware": {"gpu": name, "power_limit_w": power, "sm_clock_max_mhz": sm_max}, "shapes": {}}
    for shape in ("cfg2", "cfg5", "cfg1"):
        env = dict(os.environ, BENCH_SHAPE=shape)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--shape"], capture_output=True, text=True, env=env, cwd=ROOT)
        if r.returncode != 0:
            raise SystemExit(f"{shape} failed:\n{r.stderr[-3000:]}")
        result["shapes"][shape] = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps(result))


if __name__ == "__main__":
    main()
