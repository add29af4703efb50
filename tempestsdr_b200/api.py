"""Host-side mirror of the reference's stage interface, on top of the C-ABI (include/tsdrgpu.h).

Names and argument meaning follow the reference (TempestSDR/src): ``am_demod``, ``dsp_resample_process`` ->
:class:`Resampler`, ``dsp_post_process`` -> :class:`PostProcessor`, ``fft_perform`` / ``fft_autocorrelation`` /
``fft_crosscorrelation``, ``frameratedetector_runontodata`` -> :class:`FrameRateDetector`, ``superb_ondataready`` ->
:func:`superb_stitch`.  torch is used for device memory and streams only; every computation happens in the
hand-written sm_90a kernels of libtsdrgpu.so.  No CPU fallback exists: without the library or a GPU, calls raise.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native as N
from ._native import FrameResult, TsdrGpuError  # noqa: F401


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _f32(t: torch.Tensor) -> torch.Tensor:
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), "expected a contiguous float32 CUDA tensor"
    return t


class Context:
    """One tsdrgpu_ctx_t bound to one CUDA device (one per process/rank)."""

    def __init__(self, device: int | torch.device | None = None):
        if not torch.cuda.is_available():
            raise TsdrGpuError("no CUDA device: tempestsdr_b200 has no CPU fallback")
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device if isinstance(device, int) else device.index)
        self._lib = N.lib()
        h = C.c_void_p()
        N.check(self._lib.tsdrgpu_create(C.byref(h), self.device.index))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.tsdrgpu_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def chk(self, rc: int):
        N.check(rc, self._h)

    @property
    def stream(self) -> int:
        return _stream_ptr(self.device)

    @property
    def sm_count(self) -> int:
        return self._lib.tsdrgpu_sm_count(self._h)

    @property
    def launches(self) -> int:
        return self._lib.tsdrgpu_launch_count(self._h)

    # ------------------------------------------------------------------ a2
    def am_demod(self, iq: torch.Tensor) -> torch.Tensor:
        """TSDRLibrary.c:244-262 -- interleaved I,Q float32 -> magnitudes."""
        _f32(iq)
        out = torch.empty(iq.numel() // 2, dtype=torch.float32, device=iq.device)
        self.chk(self._lib.tsdrgpu_am_demod(self._h, self.stream, iq.data_ptr(), iq.numel() // 2, out.data_ptr()))
        return out

    def convert_samples(self, raw: torch.Tensor) -> torch.Tensor:
        """TSDRPlugin_RawFile.c:241-261 on the device: int8 / uint8 / int16 / uint16 (or float32) samples -> float32."""
        fmt = {torch.float32: 0, torch.int8: 1, torch.int16: 2, torch.uint8: 3, torch.uint16: 4}[raw.dtype]
        out = torch.empty(raw.numel(), dtype=torch.float32, device=raw.device)
        self.chk(self._lib.tsdrgpu_convert_samples(self._h, self.stream, raw.data_ptr(), fmt, raw.numel(), out.data_ptr()))
        return out

    # ------------------------------------------------------------------ a8-a10, a14 (stage level)
    def dsp_autogain_run(self, state: List[float], frame: torch.Tensor, norm: float, snr: bool = True) -> torch.Tensor:
        """dsp.c:41-94.  state = [lastmax, lastmin, snr] is updated in place."""
        _f32(frame)
        out = torch.empty_like(frame)
        a, b, c = C.c_float(state[0]), C.c_float(state[1]), C.c_float(state[2])
        self.chk(self._lib.tsdrgpu_autogain(self._h, self.stream, C.byref(a), C.byref(b), C.byref(c) if snr else None,
                                            frame.numel(), frame.data_ptr(), out.data_ptr(), norm))
        state[0], state[1], state[2] = a.value, b.value, c.value
        return out

    def dsp_timelowpass_run(self, coeff: float, frame: torch.Tensor, screen: torch.Tensor) -> None:
        """dsp.c:22-33, screen updated in place."""
        self.chk(self._lib.tsdrgpu_timelowpass(self._h, self.stream, coeff, frame.numel(), _f32(frame).data_ptr(), _f32(screen).data_ptr()))

    def dsp_average_v_h(self, frame: torch.Tensor, width: int, height: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """dsp.c:96-110 -> (widthcollapsebuffer, heightcollapsebuffer)."""
        wb = torch.empty(width, dtype=torch.float32, device=frame.device)
        hb = torch.empty(height, dtype=torch.float32, device=frame.device)
        self.chk(self._lib.tsdrgpu_average_v_h(self._h, self.stream, width, height, _f32(frame).data_ptr(), wb.data_ptr(), hb.data_ptr()))
        return wb, hb

    def gaussianblur(self, strip: torch.Tensor) -> torch.Tensor:
        """gaussian.c:18-79 (returns a blurred copy)."""
        s = _f32(strip).clone()
        self.chk(self._lib.tsdrgpu_gaussianblur(self._h, self.stream, s.data_ptr(), s.numel()))
        return s

    def pixels_argb(self, frame: torch.Tensor, inverted: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """JavaGUI/jni/TSDRLibraryNDK.c:222-283 float -> ARGB int32."""
        if out is None:
            out = torch.zeros(frame.numel(), dtype=torch.int32, device=frame.device)
        self.chk(self._lib.tsdrgpu_pixels_argb(self._h, self.stream, _f32(frame).data_ptr(), frame.numel(), int(inverted), out.data_ptr()))
        return out

    def frame_levels(self, frames: torch.Tensor, n: int, ppm: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Clip-mode auto-gain levels (tsdrgpu.h) of frames.numel() // n frames of n pixels: (lo, hi, n_valid) per frame."""
        nframes = _f32(frames).numel() // n
        lo, hi = np.empty(nframes, dtype=np.float32), np.empty(nframes, dtype=np.float32)
        nv = np.empty(nframes, dtype=np.uint64)
        self.chk(self._lib.tsdrgpu_frame_levels(self._h, self.stream, frames.data_ptr(), n, nframes, ppm, lo.ctypes.data_as(C.c_void_p),
                                                hi.ctypes.data_as(C.c_void_p), nv.ctypes.data_as(C.c_void_p)))
        return lo, hi, nv

    def clahe(self, frames: torch.Tensor, width: int, height: int, spec: str, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """CLAHE (tsdrgpu.h) of frames.numel() // (width * height) frames back to back, spec "clahe:<clip>[:<tx>x<ty>]";
        out may be frames itself."""
        mode, clip, tx, ty = N.contrast_mode(spec)
        if mode != N.CONTRAST_CLAHE:
            raise ValueError(f"Context.clahe needs a 'clahe:...' spec, not {spec!r}")
        frames = _f32(frames)
        out = torch.empty_like(frames) if out is None else out
        self.chk(self._lib.tsdrgpu_clahe(self._h, self.stream, frames.data_ptr(), out.data_ptr(), width, height,
                                         frames.numel() // (width * height), clip, tx, ty))
        return out

    def nlm(self, frames: torch.Tensor, width: int, height: int, spec: str, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Non-local means (tsdrgpu.h) of frames.numel() // (width * height) frames back to back, spec "nlm:<h>[:<R>:<P>]";
        out must not overlap frames."""
        mode, h_milli, r, p = N.denoise_mode(spec)
        if mode != N.DENOISE_NLM:
            raise ValueError(f"Context.nlm needs an 'nlm:...' spec, not {spec!r}")
        frames = _f32(frames)
        out = torch.empty_like(frames) if out is None else out
        self.chk(self._lib.tsdrgpu_nlm(self._h, self.stream, frames.data_ptr(), out.data_ptr(), width, height,
                                       frames.numel() // (width * height), h_milli, r, p))
        return out

    def deblur(self, frames: torch.Tensor, width: int, height: int, spec: str, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Richardson-Lucy deconvolution along the lines (tsdrgpu.h) of frames.numel() // (width * height) frames back to back,
        spec "rl:<sigma>[:<I>]"; out must not overlap frames."""
        mode, sigma_centi, iters = N.deblur_mode(spec)
        if mode != N.DEBLUR_RL:
            raise ValueError(f"Context.deblur needs an 'rl:...' spec, not {spec!r}")
        frames = _f32(frames)
        out = torch.empty_like(frames) if out is None else out
        self.chk(self._lib.tsdrgpu_deblur(self._h, self.stream, frames.data_ptr(), out.data_ptr(), width, height,
                                          frames.numel() // (width * height), sigma_centi, iters))
        return out

    # ------------------------------------------------------------------ a19, a20
    def fft_getrealsize(self, size: int) -> int:
        return self._lib.tsdrgpu_fft_getrealsize(size)

    def fft_perform(self, iq: torch.Tensor, size: int, inverse: bool) -> None:
        """fft.c:96-176, in place on the first 2^floor(log2 size) complex samples."""
        self.chk(self._lib.tsdrgpu_fft(self._h, self.stream, _f32(iq).data_ptr(), size, int(inverse)))

    def fft_autocorrelation(self, real: torch.Tensor) -> torch.Tensor:
        """fft.c:49-64 -> 2*size floats."""
        ans = torch.empty(2 * real.numel(), dtype=torch.float32, device=real.device)
        self.chk(self._lib.tsdrgpu_autocorrelation(self._h, self.stream, ans.data_ptr(), _f32(real).data_ptr(), real.numel()))
        return ans

    def fft_crosscorrelation(self, a: torch.Tensor, b: torch.Tensor, samples: int) -> None:
        """fft.c:69-93, result in `a`, `b` is clobbered."""
        self.chk(self._lib.tsdrgpu_crosscorrelation(self._h, self.stream, _f32(a).data_ptr(), _f32(b).data_ptr(), samples))

    def accummulate(self, out: torch.Tensor, calls: int, ac: torch.Tensor, startid: int, length: int) -> None:
        """frameratedetector.c:34-62 (the reference's spelling), out: float64 running means."""
        assert out.dtype == torch.float64 and out.is_cuda
        self.chk(self._lib.tsdrgpu_accumulate(self._h, self.stream, out.data_ptr(), calls, _f32(ac).data_ptr(), startid, length))

    # ------------------------------------------------------------------ a22
    def complex_to_abs_diff(self, iq: torch.Tensor) -> None:
        self.chk(self._lib.tsdrgpu_complex_to_abs_diff(self._h, self.stream, _f32(iq).data_ptr(), iq.numel()))

    def superb_bestfit(self, hop0: torch.Tensor, hopi: torch.Tensor, size_floats: int, samples_in_frame: int) -> int:
        r = C.c_int(0)
        self.chk(self._lib.tsdrgpu_superb_bestfit(self._h, self.stream, _f32(hop0).data_ptr(), _f32(hopi).data_ptr(), size_floats, samples_in_frame, C.byref(r)))
        return r.value

    def superb_stitch(self, hops: Sequence[torch.Tensor], samples_in_frame: int) -> Tuple[torch.Tensor, List[int]]:
        """superb_ondataready (superbandwidth.c:121-152) on one GPU."""
        pairs = hops[0].numel() // 2
        n = self.fft_getrealsize(pairs)
        out = torch.empty(len(hops) * n * 2, dtype=torch.float32, device=hops[0].device)
        ptrs = (C.c_void_p * len(hops))(*[_f32(h).data_ptr() for h in hops])
        offs = (C.c_int * len(hops))()
        total = C.c_int(0)
        self.chk(self._lib.tsdrgpu_superb_stitch(self._h, self.stream, ptrs, len(hops), pairs, samples_in_frame, out.data_ptr(), offs, C.byref(total)))
        return out[: 2 * total.value], list(offs)

    def superband_stitch_coherent(self, hops: Sequence[torch.Tensor], d: int,
                                  out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """The coherent superbandwidth stitch (tsdrgpu.h, tsdrgpu_superb_stitch_coherent) of H hops with spacing d bins,
        asynchronous: (H N interleaved pairs, the H - 1 join records as a uint8 tensor on the device, see superband_records)."""
        pairs = min(h.numel() for h in hops) // 2
        n = self.fft_getrealsize(pairs)
        if out is None:
            out = torch.empty(len(hops) * n * 2, dtype=torch.float32, device=hops[0].device)
        assert out.dtype == torch.float32 and out.is_cuda and out.is_contiguous() and out.numel() >= 2 * len(hops) * n, \
            "out must hold 2 H N contiguous float32 values on the device"
        for t in list(hops) + [out]:
            assert t.data_ptr() % 8 == 0, "hops and out must be 8-byte aligned (the kernels read and write them as float2)"
        est = torch.empty((len(hops) - 1) * C.sizeof(N.SuperbandEst), dtype=torch.uint8, device=hops[0].device)
        ptrs = (C.c_void_p * len(hops))(*[_f32(h).data_ptr() for h in hops])
        self.chk(self._lib.tsdrgpu_superb_stitch_coherent(self._h, self.stream, ptrs, len(hops), pairs, d, out.data_ptr(), est.data_ptr()))
        return out, est

    @staticmethod
    def superband_records(est: torch.Tensor) -> List["N.SuperbandEst"]:
        """The join records of superband_stitch_coherent's second result (copies them to the host: synchronises)."""
        raw = est.cpu().numpy().tobytes()
        k = C.sizeof(N.SuperbandEst)
        return [N.SuperbandEst.from_buffer_copy(raw[i * k:(i + 1) * k]) for i in range(len(raw) // k)]

    # ------------------------------------------------------------------ factories
    def resampler(self) -> "Resampler":
        return Resampler(self)

    def post_processor(self) -> "PostProcessor":
        return PostProcessor(self)

    def framerate_detector(self) -> "FrameRateDetector":
        return FrameRateDetector(self)

    def channel_filter(self) -> "ChannelFilter":
        return ChannelFilter(self)

    def spectrum(self) -> "Spectrum":
        return Spectrum(self)

    def coherence(self) -> "Coherence":
        return Coherence(self)

    def stack(self) -> "Stack":
        return Stack(self)


class Stack:
    """Drift-registered frame averaging (tsdrgpu.h): a running average that follows the picture from frame to frame, with its
    accumulator and offsets carried from run to run on the device."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(ctx._lib.tsdrgpu_stack_create(ctx._h, C.byref(h)))
        self._h = h
        self._rec = None                   # page-locked record array (torch), grown on demand

    def __del__(self):
        try:
            if self._h:
                self.ctx._lib.tsdrgpu_stack_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def set(self, spec: str) -> None:
        """"off", "align:<N>[:<rx>x<ry>]", "adapt:<N>[:<rx>x<ry>]" (restarting tile by tile where the picture changes) or
        "track:<N>[:<rx>x<ry>]" (carrying each tile's average with content that moves) or "robust:<N>[:<rx>x<ry>]" (track,
        ignoring disturbances that last one frame) from the next run on; new settings restart the average."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_stack_set(self._h, *N.stack_mode(spec)))

    def reset(self) -> None:
        """Restart the average at the next frame."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_stack_reset(self._h))

    def run(self, frames: torch.Tensor, width: int, height: int, out: Optional[torch.Tensor] = None):
        """frames: nframes * width * height float32 on the device, frames back to back -> (out, [StackRecord]).  Synchronises
        the context's stream to read the records."""
        frames = _f32(frames)
        nframes = frames.numel() // (width * height)
        out = torch.empty_like(frames) if out is None else _f32(out)
        nbytes = C.sizeof(N.StackRecord) * max(nframes, 1)
        if self._rec is None or self._rec.numel() < nbytes:
            self._rec = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        self.ctx.chk(self.ctx._lib.tsdrgpu_stack_run(self._h, self.ctx.stream, frames.data_ptr(), out.data_ptr(), width, height,
                                                     nframes, self._rec.data_ptr()))
        self.ctx.chk(self.ctx._lib.tsdrgpu_stream_sync(self.ctx._h, self.ctx.stream))
        recs = (N.StackRecord * nframes).from_address(self._rec.data_ptr())
        return out, [N.StackRecord.from_buffer_copy(r) for r in recs]

    def vectors(self, width: int, height: int) -> np.ndarray:
        """Track and robust modes: where each 16 x 16 tile of the last frame moved -> (tiles down, tiles across, 2) int32 of (vx, vy), (0, 0)
        for tiles that did not move or restarted.  Synchronises the device."""
        ty, tx = (height + 15) // 16, (width + 15) // 16
        v = np.zeros((ty, tx, 2), np.int32)
        self.ctx.chk(self.ctx._lib.tsdrgpu_stack_vectors(self._h, v.ctypes.data, ty * tx))
        return v

    def robust_counts(self) -> tuple:
        """Robust mode: the last frame's (held tiles, gated pixels, glitch frame as a bool).  Synchronises the device."""
        held, gated, hold = C.c_int32(), C.c_uint64(), C.c_int32()
        self.ctx.chk(self.ctx._lib.tsdrgpu_stack_robust_counts(self._h, C.byref(held), C.byref(gated), C.byref(hold)))
        return held.value, gated.value, bool(hold.value)


class _SegmentReports:
    """What Spectrum and Coherence share: the object tsdrgpu_<_kind>_* of tsdrgpu.h, its reset and its runs."""
    _kind = ""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(self._fn("create")(ctx._h, C.byref(h)))
        self._h = h
        self.n = 0

    def _fn(self, name: str):
        return getattr(self.ctx._lib, f"tsdrgpu_{self._kind}_{name}")

    def __del__(self):
        try:
            if self._h:
                self._fn("destroy")(self._h)
                self._h = None
        except Exception:
            pass

    def reset(self) -> None:
        """Discard the open segment and the report in progress."""
        self.ctx.chk(self._fn("reset")(self._h))

    def run(self, iq: torch.Tensor, discontinuity: bool = False) -> torch.Tensor:
        """Interleaved float32 I,Q on the device (8-byte aligned) -> the reports this run completes, (R, N) float64 on the device in
        fftshift order (asynchronous on the current stream).  discontinuity: these pairs do not follow the last run's."""
        _f32(iq)
        pairs = iq.numel() // 2
        n = C.c_uint32(0)
        self.ctx.chk(self._fn("plan")(self._h, pairs, int(discontinuity), C.byref(n)))
        out = torch.empty((n.value, self.n), dtype=torch.float64, device=iq.device)
        got = C.c_uint32(0)
        self.ctx.chk(self._fn("run")(self._h, self.ctx.stream, iq.data_ptr(), pairs, int(discontinuity),
                                     out.data_ptr() if n.value else None, n.value, C.byref(got)))
        assert got.value == n.value
        return out


class Spectrum(_SegmentReports):
    """The Welch power spectrum of tsdrgpu.h: windowed, 50 % overlapping segments of the IQ stream, K of them averaged per report,
    with the open segment carried from run to run."""
    _kind = "spectrum"

    def set(self, spec: str, samplerate: int) -> None:
        """"welch:<N>[:<rate>]" at `samplerate` from the next run on; a new spec or rate starts a new report."""
        s = N.spectrum_spec(spec)
        if s.n == 0:
            raise ValueError("Spectrum.set needs a 'welch:...' spec")
        self.ctx.chk(self.ctx._lib.tsdrgpu_spectrum_set(self._h, C.byref(s), samplerate))
        self.n = s.n

    @staticmethod
    def window(n: int) -> np.ndarray:
        """The window of N points in double, before its rounding to float32."""
        w = np.empty(n, dtype=np.float64)
        N.check(N.lib().tsdrgpu_spectrum_window(n, w.ctypes.data_as(C.c_void_p)))
        return w

    @staticmethod
    def segments_per_report(spec: str, samplerate: int) -> int:
        """K of `spec` at `samplerate` (0 for "off" or samplerate 0)."""
        return N.lib().tsdrgpu_spectrum_k(C.byref(N.spectrum_spec(spec)), samplerate)


class Coherence(_SegmentReports):
    """The spectral coherence at the line rate of tsdrgpu.h: each segment of the Welch spectrum's segmentation transformed with the
    complex windows w+ and w-, |sum U+ conj(U-) e^{-2 pi i alpha s/fs}| / sqrt(sum |U+|^2 sum |U-|^2) per report."""
    _kind = "coherence"

    def set(self, spec: str, samplerate: int, alpha: float) -> None:
        """"line[:<rate>]" at `samplerate` and line rate `alpha` (Hz) from the next run on; alpha alone takes effect at the next
        report, a new rate, samplerate or N starts a new report."""
        s = N.coherence_spec(spec)
        if s.rate == 0:
            raise ValueError("Coherence.set needs a 'line...' spec")
        self.ctx.chk(self.ctx._lib.tsdrgpu_coherence_set(self._h, C.byref(s), samplerate, float(alpha)))
        self.n = Coherence.n_for(samplerate, alpha)

    @staticmethod
    def n_for(samplerate: int, alpha: float) -> int:
        """N at `samplerate` and line rate `alpha`; 0 when unresolvable."""
        return N.lib().tsdrgpu_coherence_n(samplerate, float(alpha))

    @staticmethod
    def window(n: int, alpha: float, samplerate: int) -> np.ndarray:
        """w+ of N points in double, before its rounding to float32, as complex128."""
        w = np.empty(2 * n, dtype=np.float64)
        N.check(N.lib().tsdrgpu_coherence_window(n, float(alpha), samplerate, w.ctypes.data_as(C.c_void_p)))
        return w[0::2] + 1j * w[1::2]


class ChannelFilter:
    """The channel filter of tsdrgpu.h: one complex FIR (a pass band minus up to four stop bands) on interleaved IQ, with the
    last T-1 input pairs carried from run to run."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(ctx._lib.tsdrgpu_chanfilt_create(ctx._h, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.ctx._lib.tsdrgpu_chanfilt_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def set(self, spec: str, samplerate: int) -> None:
        """"pass:<lo>:<hi>[,stop:<a>:<b>]...[,taps:<T>]" (Hz) at `samplerate` from the next run on; new taps zero the history."""
        s = N.channel_spec(spec)
        if s.taps == 0:
            raise ValueError("ChannelFilter.set needs a 'pass:...' spec")
        self.ctx.chk(self.ctx._lib.tsdrgpu_chanfilt_set(self._h, C.byref(s), samplerate))

    def reset(self) -> None:
        """Zero the history."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_chanfilt_reset(self._h, self.ctx.stream))

    def run(self, iq: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Interleaved float32 I,Q on the device -> the filtered pairs (asynchronous on the current stream)."""
        _f32(iq)
        out = torch.empty_like(iq) if out is None else _f32(out)
        self.ctx.chk(self.ctx._lib.tsdrgpu_chanfilt_run(self._h, self.ctx.stream, iq.data_ptr(), iq.numel() // 2, out.data_ptr()))
        return out

    @staticmethod
    def taps(spec: str, samplerate: int) -> np.ndarray:
        """The float32 taps of `spec` at `samplerate` as complex64, h[0] first."""
        s = N.channel_spec(spec)
        T = C.c_int(0)
        N.check(N.lib().tsdrgpu_channel_taps(C.byref(s), samplerate, None, C.byref(T)))
        h = np.empty(2 * T.value, dtype=np.float32)
        N.check(N.lib().tsdrgpu_channel_taps(C.byref(s), samplerate, h.ctypes.data_as(C.c_void_p), C.byref(T)))
        return h.view(np.complex64)


class Resampler:
    """dsp_resample_t + dsp_resample_process (dsp.c:250-307), optionally fused with am_demod."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(ctx._lib.tsdrgpu_resampler_create(ctx._h, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.ctx._lib.tsdrgpu_resampler_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def reset(self):
        self.ctx.chk(self.ctx._lib.tsdrgpu_resampler_reset(self._h, self.ctx.stream))

    def set_kernel(self, kernel: str) -> None:
        """"box" (the reference's area integrator, the default) or "sinc" (the windowed-sinc interpolator of tsdrgpu.h) for the
        following runs; ``nearest=True`` on a run still takes precedence."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_resampler_set_kernel(self._h, N.RESAMPLER_KERNELS[kernel]))

    @staticmethod
    def sinc_taps(r: float) -> np.ndarray:
        """The sinc mode's tap table for ratio r = upsample_by/downsample_by, shape (phases, taps), float32."""
        T, L = C.c_int(0), C.c_int(0)
        N.lib().tsdrgpu_sinc_taps(r, None, C.byref(T), C.byref(L))
        taps = np.empty((L.value, T.value), dtype=np.float32)
        N.check(N.lib().tsdrgpu_sinc_taps(r, taps.ctypes.data_as(C.c_void_p), C.byref(T), C.byref(L)))
        return taps

    @property
    def state(self) -> Tuple[float, float]:
        c, o = C.c_double(0), C.c_double(0)
        self.ctx.chk(self.ctx._lib.tsdrgpu_resampler_get_state(self._h, self.ctx.stream, C.byref(c), C.byref(o)))
        return c.value, o.value

    @state.setter
    def state(self, co):
        self.ctx.chk(self.ctx._lib.tsdrgpu_resampler_set_state(self._h, self.ctx.stream, co[0], co[1]))

    @staticmethod
    def _blocks(block_sizes):
        if isinstance(block_sizes, tuple):           # (uniform_block, nblocks)
            return None, int(block_sizes[0]), int(block_sizes[1]), None
        arr = np.ascontiguousarray(block_sizes, dtype=np.uint32)
        return arr.ctypes.data_as(C.c_void_p), 0, int(arr.size), arr

    def plan(self, block_sizes, upsample_by: float, downsample_by: float) -> int:
        p, u, n, keep = self._blocks(block_sizes)
        return self.ctx._lib.tsdrgpu_resampler_plan(self._h, p, u, n, upsample_by, downsample_by)

    def process(self, x: torch.Tensor, block_sizes, upsample_by: float, downsample_by: float, nearest: bool = False,
                in_is_iq: bool = False, out: Optional[torch.Tensor] = None, mag_out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Run consecutive decimator blocks.  block_sizes: sequence of sizes, or (uniform_block, nblocks).
        mag_out (IQ input only): also receives |x| of every input sample (am_demod's output for the frame-rate detector)."""
        p, u, n, keep = self._blocks(block_sizes)
        if mag_out is not None:
            self.ctx.chk(self.ctx._lib.tsdrgpu_resampler_set_mag_out(self._h, _f32(mag_out).data_ptr()))
        need = self.ctx._lib.tsdrgpu_resampler_plan(self._h, p, u, n, upsample_by, downsample_by)
        if out is None:
            out = torch.empty(max(int(need), 1), dtype=torch.float32, device=x.device)
        n_out = C.c_uint64(0)
        rc = self.ctx._lib.tsdrgpu_resampler_run(self._h, self.ctx.stream, _f32(x).data_ptr(), int(in_is_iq), p, u, n,
                                                 upsample_by, downsample_by, int(nearest), out.data_ptr(), out.numel(), C.byref(n_out))
        if rc != N.OK and mag_out is not None:       # a refused run leaves mag_out armed: disarm it, it belongs to this call only
            self.ctx._lib.tsdrgpu_resampler_set_mag_out(self._h, None)
        self.ctx.chk(rc)
        return out[: n_out.value]


@dataclass
class PostProcessFlags:
    autoshift: bool = True            # PARAM_INT_AUTOSHIFT
    lowpass_before_sync: bool = True  # PARAM_LOW_PASS_BEFORE_SYNC
    autogain_after_proc: bool = False # PARAM_AUTOGAIN_AFTER_PROCESSING
    superresolution: bool = False     # PARAM_AUTOCORR_SUPERRESOLUTION
    compute_snr: bool = False

    def bits(self) -> int:
        return (N.FS_AUTOSHIFT * self.autoshift | N.FS_LOWPASS_BEFORE_SYNC * self.lowpass_before_sync |
                N.FS_AUTOGAIN_AFTER_PROC * self.autogain_after_proc | N.FS_SUPERRESOLUTION * self.superresolution |
                N.FS_COMPUTE_SNR * self.compute_snr)


class PostProcessor:
    """dsp_postprocess_t + dsp_post_process (dsp.c:112-239) for batches of frames."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(ctx._lib.tsdrgpu_framestage_create(ctx._h, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.ctx._lib.tsdrgpu_framestage_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def reset(self):
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_reset(self._h, self.ctx.stream))

    def set_overlap(self, on: bool):
        """Run the sync search + re-centring of batch k on a side stream under batch k+1 (see tsdrgpu.h); outputs are
        valid after :meth:`join`."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_overlap(self._h, int(on)))

    def join(self):
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_join(self._h, self.ctx.stream))

    def set_autogain(self, spec: str) -> None:
        """"minmax" (the reference's levels, the default) or "clip:<percent>" (the levels <percent> % of the valid pixels inside
        each end, tsdrgpu.h) for the following runs; lastmin / lastmax carry on across a switch."""
        mode, ppm = N.autogain_mode(spec)
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_autogain(self._h, mode, ppm))

    def set_contrast(self, spec: str) -> None:
        """"off" (the default) or "clahe:<clip>[:<tx>x<ty>]" (contrast-limited adaptive histogram equalisation of the delivered
        frames, tsdrgpu.h) for the following runs; kept across reset."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_contrast(self._h, *N.contrast_mode(spec)))

    def set_denoise(self, spec: str) -> None:
        """"off" (the default) or "nlm:<h>[:<R>:<P>]" (non-local means of the delivered frames, ahead of CLAHE, tsdrgpu.h) for
        the following runs; kept across reset."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_denoise(self._h, *N.denoise_mode(spec)))

    def set_deblur(self, spec: str) -> None:
        """"off" (the default) or "rl:<sigma>[:<I>]" (Richardson-Lucy deconvolution along the lines of the delivered frames,
        after the stack and ahead of NLM and CLAHE, tsdrgpu.h) for the following runs; kept across reset."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_deblur(self._h, *N.deblur_mode(spec)))

    def set_stack(self, spec: str) -> None:
        """"off" (the default), "align:<N>[:<rx>x<ry>]" (drift-registered averaging of the delivered frames, ahead of NLM and
        CLAHE, tsdrgpu.h), "adapt:<N>[:<rx>x<ry>]" (the same, restarting tile by tile where the picture changes) or
        "track:<N>[:<rx>x<ry>]" (the same, carrying each tile's average with content that scrolls or moves) or
        "robust:<N>[:<rx>x<ry>]" (track, ignoring disturbances that last one frame) for the following runs; the mode is kept
        across reset, the average restarts there."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_set_stack(self._h, *N.stack_mode(spec)))

    def stack_records(self, nframes: int):
        """The stack records of the last run with the stack on (first nframes of them); synchronises the device."""
        recs = (N.StackRecord * nframes)()
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_stack_records(self._h, recs, nframes))
        return list(recs)

    def process(self, frames: torch.Tensor, width: int, height: int, motionblur: float = 0.0, lowpasscoeff: float = 0.1,
                flags: PostProcessFlags = PostProcessFlags(), out: Optional[torch.Tensor] = None, want_results: bool = True):
        """frames: nframes*width*height float32, frames back to back.  Returns (frames_out, [FrameResult])."""
        nframes = frames.numel() // (width * height)
        assert nframes * width * height == frames.numel()
        if out is None:
            out = torch.empty_like(frames)
        res = (FrameResult * nframes)() if want_results else None
        self.ctx.chk(self.ctx._lib.tsdrgpu_framestage_run(self._h, self.ctx.stream, _f32(frames).data_ptr(), nframes, width, height,
                                                          motionblur, lowpasscoeff, flags.bits(), out.data_ptr(), res))
        return out, (list(res) if want_results else None)


class FrameRateDetector:
    """frameratedetector_runontodata + the two running-mean plots (frameratedetector.c:87-126)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        h = C.c_void_p()
        ctx.chk(ctx._lib.tsdrgpu_frd_create(ctx._h, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                self.ctx._lib.tsdrgpu_frd_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def reset(self):
        self.ctx._lib.tsdrgpu_frd_reset(self._h)

    def set_overlap(self, on: bool) -> None:
        """Runs go to the detector's own stream and work buffers (tsdrgpu_frd_set_overlap); see :meth:`join`."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_set_overlap(self._h, 1 if on else 0))

    def join(self) -> None:
        """The context's stream waits (on the device) for the last overlapped run: call before the capture memory is reused."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_join(self._h, self.ctx.stream))

    @staticmethod
    def capture_size(samplerate: int) -> int:
        return N.lib().tsdrgpu_frd_capture_size(samplerate)

    @staticmethod
    def windows(samplerate: int) -> Tuple[int, int, int, int]:
        v = [C.c_int(0) for _ in range(4)]
        N.lib().tsdrgpu_frd_windows(samplerate, *[C.byref(x) for x in v])
        return tuple(x.value for x in v)

    def run_batch(self, samplerate: int, captures: torch.Tensor, size: int, batch: int, stride: Optional[int] = None) -> int:
        """`batch` consecutive captures of `size` samples (capture b at captures[b*stride:]) accumulated in order;
        asynchronous, the plots stay on the device (see :meth:`plots`)."""
        calls = C.c_uint64(0)
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_run_batch(self._h, self.ctx.stream, samplerate, _f32(captures).data_ptr(), size, batch,
                                                         stride if stride is not None else size, C.byref(calls)))
        return calls.value

    def dump_csv(self, samplerate: int, capture: torch.Tensor, path: str) -> None:
        """dump_autocorrect (frameratedetector.c:64-85) of one capture."""
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_dump_csv(self._h, self.ctx.stream, samplerate, _f32(capture).data_ptr(), capture.numel(), path.encode()))

    def plots(self, samplerate: int):
        fmin, fmax, lmin, lmax = self.windows(samplerate)
        fp, lp = np.zeros(fmax - fmin), np.zeros(lmax - lmin)
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_get_plots(self._h, self.ctx.stream, samplerate, fp.ctypes.data_as(C.c_void_p), fp.size,
                                                         lp.ctypes.data_as(C.c_void_p), lp.size))
        return (fmin, fp), (lmin, lp)

    def run(self, samplerate: int, capture: torch.Tensor, copy_out: bool = True):
        fmin, fmax, lmin, lmax = self.windows(samplerate)
        fp = np.zeros(fmax - fmin) if copy_out else None
        lp = np.zeros(lmax - lmin) if copy_out else None
        calls = C.c_uint64(0)
        self.ctx.chk(self.ctx._lib.tsdrgpu_frd_run(self._h, self.ctx.stream, samplerate, _f32(capture).data_ptr(), capture.numel(),
                                                   fp.ctypes.data_as(C.c_void_p) if copy_out else None, fmax - fmin,
                                                   lp.ctypes.data_as(C.c_void_p) if copy_out else None, lmax - lmin, C.byref(calls)))
        return (fmin, fp), (lmin, lp), calls.value
