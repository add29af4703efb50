"""bench.py's DeviceStep against a stage-wise replay of the same IQ with the oracle (run by
tests/test_production_batches.py::test_bench_device_step_against_a_stagewise_replay, one process per BENCH_SHAPE).

Two steps, each over the same resident IQ (as the benchmark runs them): the oracle replays the stream fed twice -- am_demod,
the resampler block by block, the post-processor frame by frame (autoshift, low-pass before sync), the frame-rate detector over
every complete capture -- and every frame the steps handed over must be bit-exact, both plots within 1e-5 of their peak after
each step.  Prints "replay ok" and a summary on success.
"""
import numpy as np
import torch

import bench
from oracle import oracle as orc
from tempestsdr_b200 import api


def main():
    O = orc.best()
    gpu = api.Context(0)
    fs, h, fv = bench.FS, bench.HEIGHT, bench.FV
    w = bench.geometry()
    assert w == O.geometry(fs, h, fv)[0]
    n = w * h
    block = int(0.1 * fs / fv)
    pairs = block * 10 * bench.FRAMES_PER_BATCH
    iq = bench.make_iq(pairs, seed=1000)                    # rank 0's IQ in run_ours
    step = bench.DeviceStep(gpu, torch.from_numpy(iq).cuda(), w)
    handed, plots = [], []
    for _ in range(2):
        step()
        fo, done = step.last_frames
        handed.append((fo, done))
        step.frd.join()
        plots.append(step.frd.plots(fs))
    step.join()
    torch.cuda.synchronize()
    ncap = [pairs // step.cap, 2 * pairs // step.cap - pairs // step.cap]
    assert step.captures == sum(ncap) and min(ncap) >= 1

    # ---- the oracle, stage by stage, on the same stream fed twice
    mag = O.am_demod(iq)
    rs = O.resampler()
    pp = O.postprocessor(fs, h, fv, 1, 0)
    up = w * h * fv
    pix = np.zeros(0, np.float32)
    k = 0
    for s, (fo, done) in enumerate(handed):
        got_frames = fo[: done * n].view(done, n)
        b = 0
        f = 0
        while f < done:
            while pix.size < n:
                assert b < 10 * bench.FRAMES_PER_BATCH, f"step {s}: the replay ran out of blocks at frame {f} of {done}"
                pix = np.concatenate([pix, rs.run(mag[b * block:(b + 1) * block], up, float(fs))]); b += 1
            want, _ = pp.run(pix[:n], w, h, 0.0, 0.1, 1, 0)
            pix = pix[n:]
            got = got_frames[f].cpu().numpy()
            bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
            assert bad.size == 0, f"{bench.SHAPE} step {s} frame {f} (stream frame {k}): {bad.size} pixels differ, first at {bad[:5]}"
            f += 1; k += 1
        for bb in range(b, 10 * bench.FRAMES_PER_BATCH):      # the rest of the step's blocks: pixels carried to the next step
            pix = np.concatenate([pix, rs.run(mag[bb * block:(bb + 1) * block], up, float(fs))])
    det = O.framerate_detector()
    stream = np.concatenate([mag, mag])
    c = 0
    worst = 0.0
    for s in range(2):
        for _ in range(ncap[s]):
            (fo_, fp), (lo_, lp), calls = det.run(fs, stream[c * step.cap:(c + 1) * step.cap]); c += 1
        (gfo, gfp), (glo, glp) = plots[s]
        assert (gfo, glo) == (fo_, lo_) and calls == c
        for g, wv, what in ((gfp, fp, "frame"), (glp, lp, "line")):
            err = float(np.max(np.abs(g - wv))) / float(np.max(np.abs(wv)))
            worst = max(worst, err)
            assert err <= 1e-5, f"{bench.SHAPE} {what} plot after step {s}: max|err|/peak = {err:.3g}"     # 1e-5 of the plot peak
    print(f"replay ok: {bench.SHAPE} {w}x{h}, frames {[d for _, d in handed]}, captures {ncap}, worst plot error/peak {worst:.3g}")


if __name__ == "__main__":
    main()
