"""Frame quality of the coherent superbandwidth stitch, through the GPU pipeline (synthetic scene: no real capture).

Scene: a static raster of one-pixel detail (random levels in [0.35, 1], 4 % / 12 % blanking at 0.05) at 2 samples per pixel, AM on
a complex baseband at H fs = 4 MS/s, 100 lines at 60 Hz.  Four hops of 2^17 pairs at fs = 1 MS/s, 25 % overlap, are cut from it by
tests/superband_coherent_model.hops_from_truth: shift to c_i, a 1025-tap linear-phase FIR band limit, decimation, a fractional
delay of up to 3 samples, an LO phase and a gain of 0.5-2 per hop, noise 30 dB below each hop.  Each stream is decoded by a
normal-mode pipeline (autoshift off, box resampler) at its own rate, and frames 2-6 (as far as the stream reaches) are compared with
the frames the same pipeline decodes from the truth restricted to the stitched band, after a least-squares gain and offset per frame
(the auto-gain's state differs between streams), as PSNR with peak 1 over the pixels that are not sync markers:
  coherent             tsdrgpu_superb_stitch_coherent on the hops (the stage call; the pipeline's coherent mode hands exactly this
                       stream to its decimator)
  reference            tsdrgpu_superb_stitch on the same hops
  one hop at fs        a hop tuned to the centre, decoded at fs, its frames widened to the truth's width by linear interpolation
  coherent, roll-off   the coherent stitch of hops whose front-end filter cuts inside the overlap (0.25-0.5 fs): at 0.44 fs, where
                       the two hops still share the middle half of the overlap, and at 0.375 fs, where they share none of it
Run: python profiles/studies/superband_coherent_quality.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tempestsdr_b200 import api, pipeline  # noqa: E402
from tests import fft_model as fm  # noqa: E402
from tests import superband_coherent_model as sm  # noqa: E402

FS, H, O, FV, LINES = 1_000_000, 4, 25, 60.0, 100


def raster_truth(L, seed=3):
    """static raster at 2 samples per pixel, L pairs at H fs"""
    rng = np.random.default_rng(seed)
    spl = H * FS / (FV * LINES)                                 # samples per line
    tw = int(spl / 2)
    frame = np.full((LINES, tw), 0.05)
    aw, ah = int(tw * 0.88), int(LINES * 0.96)
    frame[:ah, :aw] = rng.uniform(0.35, 1.0, size=(ah, aw))
    flat = frame.reshape(-1)
    t = np.arange(L)
    return flat[np.floor(t * (flat.size * FV / (H * FS))).astype(np.int64) % flat.size] * np.exp(0.7j)


def frames_of(iq_complex, rate):
    out = []
    p = pipeline.Pipeline(samplerate=int(rate), height=LINES, refreshrate=FV, batch_frames=1, block_when_busy=True,
                          params={"autocorr_plots_off": 1}, on_frame=lambda f, w, h: out.append(f.reshape(h, w).copy()))
    x = np.ascontiguousarray(np.asarray(iq_complex, np.complex64)).view(np.float32)
    p.process(x, 0)
    p.flush(); p.close()
    return out


def widen(frames, w):
    res = []
    for f in frames:
        xs = (np.arange(w) + 0.5) * f.shape[1] / w - 0.5
        res.append(np.stack([np.interp(xs, np.arange(f.shape[1]), row) for row in f]))
    return res


def psnr(got, want):
    vals = []
    for k in range(2, min(7, len(got), len(want))):
        g, w = got[k].reshape(-1).astype(np.float64), want[k].reshape(-1).astype(np.float64)
        keep = (np.abs(g) <= 250) & (np.abs(w) <= 250)             # not the sync detector's marker pixels (autoshift off)
        g, w = g[keep], w[keep]
        A = np.stack([g, np.ones_like(g)], 1)
        fit = A @ np.linalg.lstsq(A, w, rcond=None)[0]
        vals.append(10 * np.log10(1.0 / np.mean((fit - w) ** 2)))
    return float(np.mean(vals)), float(np.min(vals))


def main():
    n = fm.getrealsize(10 * int(FS / FV))
    d = sm.spacing(n, O)
    L = H * n
    truth = raster_truth(L)
    rng = np.random.default_rng(5)
    delays, phases, gains = rng.uniform(-3, 3, H), rng.uniform(-np.pi, np.pi, H), rng.uniform(0.5, 2.0, H)
    r = (H - 1) // 2
    delays[r], phases[r], gains[r] = 0.0, 0.0, 1.0
    hops = sm.hops_from_truth(truth, H, n, d, delays, phases, gains, 30.0, 7)
    rolled = sm.hops_from_truth(truth, H, n, d, delays, phases, gains, 30.0, 7, cutoff=0.44)
    rolled_mid = sm.hops_from_truth(truth, H, n, d, delays, phases, gains, 30.0, 7, cutoff=0.375)
    centred = sm.hops_from_truth(truth, H, n, 0, [0.0] * H, [0.0] * H, [1.0] * H, 30.0, 9)[r]
    ctx = api.Context(0)

    def coherent(hs):
        y, est = ctx.superband_stitch_coherent([torch.from_numpy(h).cuda() for h in hs], d)
        rho = [round(e.rho, 3) for e in api.Context.superband_records(est)]
        return fm.as_complex(y.cpu().numpy()), rho
    yc, rho_c = coherent(hops)
    yr_, rho_r = coherent(rolled)
    ym_, rho_m = coherent(rolled_mid)
    yref, _ = ctx.superb_stitch([torch.from_numpy(h).cuda() for h in hops], int(FS / FV))
    yref = fm.as_complex(yref.cpu().numpy())
    want = frames_of(sm.truth_in_band(truth, H, n, d), H * FS)
    w = want[0].shape[1]
    rows = [("coherent", frames_of(yc, H * FS), f"rho {rho_c}"),
            ("reference stitch", frames_of(yref, H * FS), ""),
            ("one hop at fs", widen(frames_of(fm.as_complex(centred), FS), w), ""),
            ("coherent, roll-off 0.44 fs", frames_of(yr_, H * FS), f"rho {rho_r}"),
            ("coherent, roll-off 0.375 fs", frames_of(ym_, H * FS), f"rho {rho_m}")]
    print(f"card: {torch.cuda.get_device_name(0)}; H={H} o={O} N={n} D={d}; truth frames {len(want)} of {w}x{LINES}")
    for name, fr, note in rows:
        m, lo = psnr(fr, want)
        print(f"{name:28s}: PSNR {m:5.1f} dB mean, {lo:5.1f} dB worst over frames 2-{min(6, len(want) - 1)}  {note}")
    ctx.close()


if __name__ == "__main__":
    main()
