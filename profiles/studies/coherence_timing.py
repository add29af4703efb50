"""The line-rate coherence's cost on the GPU, next to the Welch spectrum at the same N, and beside the whole device-resident step.

Prints one JSON line with
  * the GPU's name, power limit and SM clock (read-only nvidia-smi query), before and after;
  * per shape (cfg2, cfg5, cfg1, each in a process of its own because bench.py fixes its shape at import), at the shape's sample rate
    and line rate alpha = height x 60 Hz (N = 8192, 16384, 4096):
      - the coherence (line:1) and the Welch spectrum (welch:<N>:1) over the step's IQ (10 x FRAMES_PER_BATCH decimator blocks),
        one run per launch continuing the stream: CUDA events around at least 20 launches (at least 0.5 s) after warm-up, three
        rounds -> ms per batch, us per segment (segments = pairs / (N/2)) and ms per report (K segments at rate 1);
      - bench.DeviceStep's whole step with the coherence of the step's IQ on a low-priority stream of its own against the step
        alone, alternating, three rounds each (MS/s).
GPU only:  python profiles/studies/coherence_timing.py
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from profiles.studies.channel_filter_timing import ClockDuring, gpu_info  # noqa: E402

ROUNDS = 3
LAUNCHES = 20


def _time(run, x):
    import torch
    for _ in range(3):
        run(x)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); run(x); b.record()
    torch.cuda.synchronize()
    launches = max(LAUNCHES, int(500.0 / a.elapsed_time(b)))
    ms = []
    with ClockDuring() as clk:
        for _ in range(ROUNDS):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(launches):
                run(x)
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b) / launches)
    return ms, clk.mhz


def shape_run():
    import torch
    import bench
    from tempestsdr_b200 import api
    gpu = api.Context(0)
    w = bench.geometry()
    alpha = bench.HEIGHT * bench.FV
    n = api.Coherence.n_for(bench.FS, alpha)
    step_pairs = int(0.1 * bench.FS / bench.FV) * 10 * bench.FRAMES_PER_BATCH
    raw = torch.from_numpy(bench.make_iq(step_pairs, seed=1000)).cuda()
    co = gpu.coherence()
    co.set("line:1", bench.FS, alpha)
    sp = gpu.spectrum()
    sp.set(f"welch:{n}:1", bench.FS)
    segs = step_pairs / (n // 2)
    K = api.Spectrum.segments_per_report(f"welch:{n}:1", bench.FS)
    res = {"shape": bench.SHAPE, "fs": bench.FS, "alpha": alpha, "n": n, "K": K, "pairs_per_batch": step_pairs}
    for name, obj in (("coherence", co), ("welch", sp)):
        ms, mhz = _time(obj.run, raw)
        best = min(ms)
        res[name] = {"ms_per_batch": ms, "us_per_segment": round(1e3 * best / segs, 3), "ms_per_report": round(best * K / segs, 3),
                     "sm_mhz_during": mhz}
    side = torch.cuda.Stream()                      # torch's default priority is the lowest
    step_alone = bench.DeviceStep(gpu, raw, w)

    def step(k):
        if k == "on":
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                co.run(raw)
        step_alone()

    for k in ("off", "on"):
        for _ in range(2):
            step(k)
    torch.cuda.synchronize()
    res["step_msps"] = {"off": [], "on": []}
    n_steps = 8
    for _ in range(ROUNDS):
        for k in ("off", "on"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(n_steps):
                step(k)
            torch.cuda.synchronize()
            res["step_msps"][k].append(n_steps * step_pairs / (time.perf_counter() - t0) / 1e6)
    return res


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--shape":
        print(json.dumps(shape_run()))
        return
    result = {"hardware": gpu_info(), "shapes": {}}
    for shape in ("cfg2", "cfg5", "cfg1"):
        env = dict(os.environ, BENCH_SHAPE=shape)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--shape"], capture_output=True, text=True, env=env, cwd=ROOT)
        if r.returncode != 0:
            raise SystemExit(f"{shape} failed:\n{r.stderr[-3000:]}")
        result["shapes"][shape] = json.loads(r.stdout.strip().splitlines()[-1])
    result["hardware_after"] = gpu_info()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
