"""Seeded synthetic inputs shaped like the reference's workloads (SURVEY.md 8d).

Host-side numpy only: generates video-like IQ (a raster with horizontal/vertical blanking strips, repeated at the
refresh rate, AM-modulated onto a rotating carrier, plus noise) and plain noise / constant edge cases.  Used by the
tests, by bench.py and by __graft_entry__.smoke(); it is input generation, not part of the measured path.
"""
from __future__ import annotations

import numpy as np


def video_like_iq(n_pairs: int, samplerate: float, total_width: int, total_height: int, refreshrate: float,
                  seed: int = 0, snr_db: float = 30.0, blank_frac_x: float = 0.12, blank_frac_y: float = 0.04,
                  carrier_hz: float = 12345.0, fv_ppm: float = 0.0) -> np.ndarray:
    """Interleaved float32 I,Q of a raster video signal sampled at `samplerate`.

    The raster is total_width x total_height (blanking included, the GUI's convention: VideoMode.java), the
    active area holds a seeded blocky pattern, blanking sits at a distinct low level so the sync detector has a
    well separated optimum.
    """
    rng = np.random.default_rng(seed)
    act_w = int(total_width * (1.0 - blank_frac_x))
    act_h = int(total_height * (1.0 - blank_frac_y))
    frame = np.full((total_height, total_width), 0.05, dtype=np.float32)
    # blocky seeded picture: 16x16 tiles with levels in [0.35, 1.0]
    ty, tx = (act_h + 15) // 16, (act_w + 15) // 16
    tiles = rng.uniform(0.35, 1.0, size=(ty, tx)).astype(np.float32)
    pic = np.kron(tiles, np.ones((16, 16), dtype=np.float32))[:act_h, :act_w]
    frame[:act_h, :act_w] = pic
    flat = frame.reshape(-1)
    pixelrate = total_width * total_height * refreshrate * (1.0 + fv_ppm * 1e-6)
    t = np.arange(n_pairs, dtype=np.float64)
    idx = np.floor(t * (pixelrate / samplerate)).astype(np.int64) % flat.size
    amp = flat[idx].astype(np.float64)
    phase = 2.0 * np.pi * carrier_hz / samplerate * t + rng.uniform(0, 2 * np.pi)
    sigma = 10.0 ** (-snr_db / 20.0) * 0.5
    i = amp * np.cos(phase) + rng.normal(0.0, sigma, n_pairs)
    q = amp * np.sin(phase) + rng.normal(0.0, sigma, n_pairs)
    out = np.empty(2 * n_pairs, dtype=np.float32)
    out[0::2] = i
    out[1::2] = q
    return out


def noise_iq(n_pairs: int, seed: int = 0, scale: float = 1.0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(2 * n_pairs) * scale).astype(np.float32)


def video_like_frame(w: int, h: int, seed: int = 0, shift_x: int = 0, shift_y: int = 0, noise: float = 0.02,
                     blank_frac_x: float = 0.14, blank_frac_y: float = 0.05) -> np.ndarray:
    """A w x h float32 frame (already at pixel rate) with blanking strips, circularly shifted.  The blanking strips take
    blank_frac_x of the columns and blank_frac_y of the rows (1.0 - 0.14 == 0.86 exactly: the defaults give the frames
    the golden vectors were made from)."""
    rng = np.random.default_rng(seed)
    act_w, act_h = int(w * (1.0 - blank_frac_x)), int(h * (1.0 - blank_frac_y))
    f = np.full((h, w), 0.05, dtype=np.float32)
    ty, tx = (act_h + 7) // 8, (act_w + 7) // 8
    tiles = rng.uniform(0.35, 1.0, size=(ty, tx)).astype(np.float32)
    f[:act_h, :act_w] = np.kron(tiles, np.ones((8, 8), dtype=np.float32))[:act_h, :act_w]
    f += rng.normal(0, noise, size=f.shape).astype(np.float32)
    f = np.roll(np.roll(f, shift_y, axis=0), shift_x, axis=1)
    return np.ascontiguousarray(f.reshape(-1))
