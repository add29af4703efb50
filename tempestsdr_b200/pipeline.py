"""Python face of the streaming pipeline (tsdrgpu_pipeline_*): host IQ blocks in, host frames / plots out.

Mirrors what a host of the reference sees: ``process(buf, samples_dropped)`` is the plugin callback
(TSDRPlugin.h:49), ``on_frame`` is tsdr_readasync_function, ``on_value`` / ``on_plot`` are the two tsdr_init
callbacks (TSDRLibrary.h:57-59).  Callbacks run on the library's delivery thread.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Optional

import numpy as np

from . import _native as N

RAW_FORMATS = {"float32": 0, "int8": 1, "int16": 2, "uint8": 3, "uint16": 4}     # TSDRPlugin_RawFile.c:29-33
PARAM_IDS = {"autoshift": 0, "framerate_pll": 1, "autocorr_plots_reset": 2, "autocorr_plots_off": 3,
             "superresolution": 4, "nearest_neighbour_resampling": 5, "lowpass_before_sync": 6,
             "autogain_after_processing": 7, "autocorr_dump": 8}


class Pipeline:
    def __init__(self, samplerate: int, height: int, refreshrate: float, motionblur: float = 0.0,
                 params: Optional[Dict[str, int]] = None, batch_frames: int = 1, batch_blocks: int = 10,
                 block_when_busy: bool = False, device: int = 0,
                 on_frame: Optional[Callable] = None, on_value: Optional[Callable] = None, on_plot: Optional[Callable] = None,
                 on_retune: Optional[Callable] = None, resampler: str = "box", autogain: str = "minmax",
                 contrast: str = "off", channel: str = "off", denoise: str = "off", spectrum: str = "off",
                 stack: str = "off", deblur: str = "off", coherence: str = "off", superband: str = "reference"):
        self._lib = N.lib()
        ctx = C.c_void_p()
        N.check(self._lib.tsdrgpu_create(C.byref(ctx), device))
        self._ctx = ctx
        cfg = N.PipelineConfig()
        cfg.samplerate, cfg.height, cfg.refreshrate, cfg.motionblur = samplerate, height, refreshrate, motionblur
        for k, v in (params or {}).items():
            cfg.params_int[PARAM_IDS[k]] = int(v)
        cfg.batch_frames, cfg.batch_blocks, cfg.block_when_busy = batch_frames, batch_blocks, int(block_when_busy)
        self.errors = []

        def _frame(buf, w, h, _):
            try:
                if on_frame:
                    on_frame(np.ctypeslib.as_array(buf, shape=(w * h,)), w, h)
            except Exception as e:      # never let an exception cross the C boundary
                self.errors.append(e)

        def _value(vid, a, b, _):
            try:
                if on_value:
                    on_value(vid, a, b)
            except Exception as e:
                self.errors.append(e)

        def _plot(pid, off, vals, size, sr, _):
            try:
                if on_plot:
                    on_plot(pid, off, np.ctypeslib.as_array(vals, shape=(size,)), sr)
            except Exception as e:
                self.errors.append(e)

        self._cbs = (N.FRAME_CB(_frame), N.VALUE_CB(_value), N.PLOT_CB(_plot))    # keep alive
        h = C.c_void_p()
        N.check(self._lib.tsdrgpu_pipeline_create(ctx, C.byref(cfg), *self._cbs, None, C.byref(h)), ctx)
        self._h = h
        if resampler != "box":
            self.set_resampler(resampler)
        if autogain != "minmax":
            self.set_autogain(autogain)
        if contrast != "off":
            self.set_contrast(contrast)
        if channel != "off":
            self.set_channel(channel)
        if denoise != "off":
            self.set_denoise(denoise)
        if spectrum != "off":
            self.set_spectrum(spectrum)
        if coherence != "off":
            self.set_coherence(coherence)
        if stack != "off":
            self.set_stack(stack)
        if deblur != "off":
            self.set_deblur(deblur)
        if superband != "reference":
            self.set_superband(superband)
        if on_retune:
            def _retune(off, _):
                try:
                    on_retune(off)
                except Exception as e:
                    self.errors.append(e)
            self._retune_cb = N.RETUNE_CB(_retune)
            N.check(self._lib.tsdrgpu_pipeline_set_retune(h, self._retune_cb), ctx)

    def process(self, iq: np.ndarray, samples_dropped: int = 0) -> None:
        """iq: interleaved float32 I,Q on the HOST (numpy, or a pinned torch tensor's .numpy())."""
        assert iq.dtype == np.float32 and iq.flags.c_contiguous
        N.check(self._lib.tsdrgpu_pipeline_process(self._h, iq.ctypes.data_as(C.c_void_p), iq.size, samples_dropped), self._ctx)

    def process_ptr(self, ptr: int, items: int, samples_dropped: int = 0) -> None:
        N.check(self._lib.tsdrgpu_pipeline_process(self._h, C.c_void_p(ptr), items, samples_dropped), self._ctx)

    def process_raw(self, samples: np.ndarray, samples_dropped: int = 0) -> None:
        """samples: interleaved I,Q on the HOST still in the front end's wire format (int8 / uint8 / int16 / uint16 /
        float32); converted on the device to the floats TSDRPlugin_RawFile.c:241-261 produces on the host."""
        fmt = RAW_FORMATS[samples.dtype.name]
        assert samples.flags.c_contiguous
        N.check(self._lib.tsdrgpu_pipeline_process_raw(self._h, samples.ctypes.data_as(C.c_void_p), fmt, samples.size, samples_dropped), self._ctx)

    def process_raw_ptr(self, ptr: int, fmt: int, items: int, samples_dropped: int = 0) -> None:
        N.check(self._lib.tsdrgpu_pipeline_process_raw(self._h, C.c_void_p(ptr), fmt, items, samples_dropped), self._ctx)

    def process_raw_ptr_async(self, ptr: int, fmt: int, items: int, samples_dropped: int = 0) -> None:
        """Page-locked buffers only: returns once enqueued; the buffer must stay untouched until sync_input()."""
        N.check(self._lib.tsdrgpu_pipeline_process_raw_async(self._h, C.c_void_p(ptr), fmt, items, samples_dropped), self._ctx)

    def sync_input(self) -> None:
        N.check(self._lib.tsdrgpu_pipeline_sync_input(self._h), self._ctx)

    def flush(self) -> None:
        N.check(self._lib.tsdrgpu_pipeline_flush(self._h), self._ctx)
        if self.errors:
            raise self.errors[0]

    def set_output_argb(self, on: bool, inverted: bool = False) -> None:
        """Deliver the JNI glue's int32 pixels (TSDRLibraryNDK.c:222-283) instead of floats; on_frame then receives the
        same float32 array object whose bytes are int32 pixels: use frame.view(np.int32)."""
        N.check(self._lib.tsdrgpu_pipeline_set_output_argb(self._h, int(on), int(inverted)), self._ctx)

    def set_reports(self, snr: bool = False, detect_mode: bool = False) -> None:
        """on_value then also receives (4, snr, 0) beside every auto-gain report and (100, fps, height) after every pair of plots."""
        N.check(self._lib.tsdrgpu_pipeline_set_reports(self._h, int(snr), int(detect_mode)), self._ctx)

    def set_resampler(self, kernel: str) -> None:
        """"box" (the reference's, the default) or "sinc" (windowed-sinc interpolation, tsdrgpu.h) from the next group of
        decimator blocks on; the nearest_neighbour_resampling parameter still wins."""
        N.check(self._lib.tsdrgpu_pipeline_set_resampler(self._h, N.RESAMPLER_KERNELS[kernel]), self._ctx)

    def set_autogain(self, spec: str) -> None:
        """"minmax" (the reference's, the default) or "clip:<percent>" (percentile levels, tsdrgpu.h) from the next frame-stage
        batch on."""
        mode, ppm = N.autogain_mode(spec)
        N.check(self._lib.tsdrgpu_pipeline_set_autogain(self._h, mode, ppm), self._ctx)

    def set_contrast(self, spec: str) -> None:
        """"off" (the default) or "clahe:<clip>[:<tx>x<ty>]" (CLAHE of the delivered frames, tsdrgpu.h) from the next frame-stage
        batch on."""
        N.check(self._lib.tsdrgpu_pipeline_set_contrast(self._h, *N.contrast_mode(spec)), self._ctx)

    def set_denoise(self, spec: str) -> None:
        """"off" (the default) or "nlm:<h>[:<R>:<P>]" (non-local means of the delivered frames, ahead of CLAHE, tsdrgpu.h) from
        the next frame-stage batch on."""
        N.check(self._lib.tsdrgpu_pipeline_set_denoise(self._h, *N.denoise_mode(spec)), self._ctx)

    def set_stack(self, spec: str) -> None:
        """"off" (the default), "align:<N>[:<rx>x<ry>]" (drift-registered averaging of the delivered frames, ahead of NLM and
        CLAHE, tsdrgpu.h), "adapt:<N>[:<rx>x<ry>]" (the same, restarting tile by tile where the picture changes) or
        "track:<N>[:<rx>x<ry>]" (the same, carrying each tile's average with content that scrolls or moves) or
        "robust:<N>[:<rx>x<ry>]" (track, ignoring disturbances that last one frame) from the next frame-stage batch on.  While it is on, on_value also receives (101, drift in px/frame,
        offset mod W H) beside every auto-gain report; sync() restarts the average."""
        N.check(self._lib.tsdrgpu_pipeline_set_stack(self._h, *N.stack_mode(spec)), self._ctx)

    def set_deblur(self, spec: str) -> None:
        """"off" (the default) or "rl:<sigma>[:<I>]" (Richardson-Lucy deconvolution along the lines of the delivered frames,
        after the stack and ahead of NLM and CLAHE, tsdrgpu.h) from the next frame-stage batch on."""
        N.check(self._lib.tsdrgpu_pipeline_set_deblur(self._h, *N.deblur_mode(spec)), self._ctx)

    def set_channel(self, spec: str) -> None:
        """"off" (the default) or "pass:<lo>:<hi>[,stop:<a>:<b>]...[,taps:<T>]" (the channel filter on the IQ stream before
        demodulation, Hz relative to the tuned centre, tsdrgpu.h) from the next process() on."""
        N.check(self._lib.tsdrgpu_pipeline_set_channel(self._h, C.byref(N.channel_spec(spec))), self._ctx)

    def set_spectrum(self, spec: str) -> None:
        """"off" (the default) or "welch:<N>[:<rate>]" (a Welch power spectrum of the IQ stream before the channel filter, tsdrgpu.h)
        from the next process() on.  Reports reach on_plot as (100, -N/2, N values in fftshift order, samplerate)."""
        N.check(self._lib.tsdrgpu_pipeline_set_spectrum(self._h, C.byref(N.spectrum_spec(spec))), self._ctx)

    def set_coherence(self, spec: str) -> None:
        """"off" (the default) or "line[:<rate>]" (the spectral coherence of the IQ stream at the line rate, before the channel
        filter, tsdrgpu.h) from the next process() on.  Reports reach on_plot as (101, -N/2, N values of gamma in fftshift order,
        samplerate), on the axis of the spectrum's plot 100."""
        N.check(self._lib.tsdrgpu_pipeline_set_coherence(self._h, C.byref(N.coherence_spec(spec))), self._ctx)

    def set_param(self, name: str, value: int) -> None:
        N.check(self._lib.tsdrgpu_pipeline_set_param_int(self._h, PARAM_IDS[name], value), self._ctx)

    def set_resolution(self, height: int, refreshrate: float) -> None:
        N.check(self._lib.tsdrgpu_pipeline_set_resolution(self._h, height, refreshrate), self._ctx)

    def set_superb_devices(self, devices) -> None:
        """Superbandwidth mode with one hop per GPU: devices[0] is this pipeline's device, len(devices) in {2, 4, 8} = hops."""
        arr = (C.c_int * len(devices))(*devices)
        N.check(self._lib.tsdrgpu_pipeline_set_superb_devices(self._h, arr, len(devices)), self._ctx)

    def set_superband(self, spec: str) -> None:
        """"reference" (the reference's stitch, the default) or "coherent[:<H>[:<o>]]" (H overlapping hops at their true
        frequencies, matched in delay, phase and gain, tsdrgpu.h) from the next superbandwidth round on.  One GPU only."""
        N.check(self._lib.tsdrgpu_pipeline_set_superband(self._h, C.byref(N.superband_spec(spec))), self._ctx)

    def superband_estimates(self):
        """The last coherent round's joins (tsdrgpu_superband_est_t records, one per hop but the reference hop); synchronises."""
        recs = (N.SuperbandEst * 8)()
        n = C.c_int(0)
        N.check(self._lib.tsdrgpu_pipeline_superband_estimates(self._h, recs, 8, C.byref(n)), self._ctx)
        return list(recs[: n.value])

    def set_motionblur(self, coeff: float) -> None:
        N.check(self._lib.tsdrgpu_pipeline_set_motionblur(self._h, coeff), self._ctx)

    def sync(self, pixels: int) -> None:
        N.check(self._lib.tsdrgpu_pipeline_sync(self._h, pixels), self._ctx)

    def geometry(self):
        w, h, fv = C.c_int(0), C.c_int(0), C.c_double(0)
        N.check(self._lib.tsdrgpu_pipeline_get_geometry(self._h, C.byref(w), C.byref(h), C.byref(fv)), self._ctx)
        return w.value, h.value, fv.value

    def stats(self) -> N.PipelineStats:
        s = N.PipelineStats()
        N.check(self._lib.tsdrgpu_pipeline_stats(self._h, C.byref(s)), self._ctx)
        return s

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.tsdrgpu_pipeline_destroy(self._h)
            self._h = None
            self._lib.tsdrgpu_destroy(self._ctx)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
