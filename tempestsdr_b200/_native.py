"""ctypes loader of tempestsdr_b200/lib/libtsdrgpu.so (the C-ABI of include/tsdrgpu.h).

There is no fallback of any kind: a missing library or a missing CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtsdrgpu.so")

OK = 0


class FrameResult(C.Structure):
    """tsdrgpu_frame_result_t"""
    _fields_ = [("x_dx", C.c_int32), ("x_vx", C.c_int32), ("x_absvx", C.c_int32), ("x_stripsize", C.c_int32),
                ("y_dx", C.c_int32), ("y_vx", C.c_int32), ("y_absvx", C.c_int32), ("y_stripsize", C.c_int32),
                ("avg_speed", C.c_double), ("pll_state", C.c_int32),
                ("lastmax", C.c_float), ("lastmin", C.c_float), ("snr", C.c_float),
                ("autogain_report", C.c_int32), ("reserved", C.c_int32)]


class PipelineConfig(C.Structure):
    """tsdrgpu_pipeline_config_t"""
    _fields_ = [("samplerate", C.c_uint32), ("height", C.c_int), ("refreshrate", C.c_double), ("motionblur", C.c_float),
                ("params_int", C.c_uint32 * 9), ("batch_frames", C.c_int), ("batch_blocks", C.c_int), ("block_when_busy", C.c_int)]


class PipelineStats(C.Structure):
    """tsdrgpu_pipeline_stats_t"""
    _fields_ = [(n, C.c_uint64) for n in ("samples_in", "samples_dropped_upstream", "samples_resampled", "frames_processed",
                                          "frames_delivered", "frames_dropped", "captures", "plots_delivered",
                                          "h2d_bytes", "d2h_bytes", "gpu_launches", "stitches", "host_buffers_registered",
                                          "spectra_delivered", "spectra_skipped", "coherence_delivered", "coherence_skipped")]


FRAME_CB = C.CFUNCTYPE(None, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_void_p)
VALUE_CB = C.CFUNCTYPE(None, C.c_int, C.c_double, C.c_double, C.c_void_p)
PLOT_CB = C.CFUNCTYPE(None, C.c_int, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_uint32, C.c_void_p)
RETUNE_CB = C.CFUNCTYPE(None, C.c_int32, C.c_void_p)

FS_AUTOSHIFT, FS_LOWPASS_BEFORE_SYNC, FS_AUTOGAIN_AFTER_PROC, FS_SUPERRESOLUTION, FS_COMPUTE_SNR = 1, 2, 4, 8, 16

RESAMPLER_KERNELS = {"box": 0, "sinc": 1}          # TSDRGPU_RS_BOX / TSDRGPU_RS_SINC
AG_MINMAX, AG_CLIP, AG_MAX_PPM = 0, 1, 250000      # TSDRGPU_AG_MINMAX / TSDRGPU_AG_CLIP / TSDRGPU_AG_MAX_PPM


def autogain_mode(spec: str):
    """"minmax" or "clip:<percent>" (the host library's TSDR_AUTOGAIN spelling) -> (mode, ppm), read by tsdrgpu_autogain_ppm."""
    if spec == "minmax":
        return AG_MINMAX, 0
    ppm = lib().tsdrgpu_autogain_ppm(spec[5:].encode()) if spec.startswith("clip:") else -1
    if ppm < 0:
        raise ValueError(f"auto-gain must be 'minmax' or 'clip:<percent>' with percent in [0, 25], not {spec!r}")
    return AG_CLIP, ppm


CONTRAST_OFF, CONTRAST_CLAHE = 0, 1                 # TSDRGPU_CONTRAST_OFF / TSDRGPU_CONTRAST_CLAHE


def contrast_mode(spec: str):
    """"off", "clahe:<clip>" or "clahe:<clip>:<tx>x<ty>" (the host library's TSDR_CONTRAST spelling) -> (mode, clip_centi, tx, ty),
    read by tsdrgpu_contrast_parse."""
    out = [C.c_int() for _ in range(4)]
    if lib().tsdrgpu_contrast_parse(spec.encode(), *[C.byref(o) for o in out]) != 0:
        raise ValueError(f"contrast must be 'off' or 'clahe:<clip>[:<tx>x<ty>]' with clip in [1, 256] and tiles in [1, 64], not {spec!r}")
    return tuple(o.value for o in out)


class ChannelSpec(C.Structure):
    """tsdrgpu_channel_t"""
    _fields_ = [("taps", C.c_int32), ("nstop", C.c_int32), ("pass_lo_hz", C.c_int64), ("pass_hi_hz", C.c_int64),
                ("stop_lo_hz", C.c_int64 * 4), ("stop_hi_hz", C.c_int64 * 4)]


def channel_spec(spec: str) -> ChannelSpec:
    """"off" or "pass:<lo>:<hi>[,stop:<a>:<b>]...[,taps:<T>]" (the host library's TSDR_CHANNEL spelling), read by
    tsdrgpu_channel_parse.  "off" gives taps == 0."""
    out = ChannelSpec()
    if lib().tsdrgpu_channel_parse(spec.encode(), C.byref(out)) != 0:
        raise ValueError(f"channel must be 'off' or 'pass:<lo>:<hi>' with up to four ',stop:<a>:<b>' and an optional ',taps:<T>' "
                         f"(integer Hz, odd T in [9, 257]), not {spec!r}")
    return out


class WelchSpec(C.Structure):
    """tsdrgpu_welch_t"""
    _fields_ = [("n", C.c_int32), ("rate", C.c_int32)]


PLOT_ID_SPECTRUM = 100                              # TSDRGPU_PLOT_ID_SPECTRUM


def spectrum_spec(spec: str) -> WelchSpec:
    """"off" or "welch:<N>[:<rate>]" (the host library's TSDR_SPECTRUM spelling), read by tsdrgpu_spectrum_parse.  "off" gives
    n == 0."""
    out = WelchSpec()
    if lib().tsdrgpu_spectrum_parse(spec.encode(), C.byref(out)) != 0:
        raise ValueError(f"spectrum must be 'off' or 'welch:<N>[:<rate>]' with N a power of two in [256, 65536] and rate in "
                         f"[1, 100], not {spec!r}")
    return out


class CoherenceSpec(C.Structure):
    """tsdrgpu_coherence_t"""
    _fields_ = [("rate", C.c_int32)]


PLOT_ID_COHERENCE = 101                             # TSDRGPU_PLOT_ID_COHERENCE


def coherence_spec(spec: str) -> CoherenceSpec:
    """"off" or "line[:<rate>]" (the host library's TSDR_COHERENCE spelling), read by tsdrgpu_coherence_parse.  "off" gives
    rate == 0."""
    out = CoherenceSpec()
    if lib().tsdrgpu_coherence_parse(spec.encode(), C.byref(out)) != 0:
        raise ValueError(f"coherence must be 'off' or 'line[:<rate>]' with rate in [1, 100], not {spec!r}")
    return out


DENOISE_OFF, DENOISE_NLM = 0, 1                     # TSDRGPU_DENOISE_OFF / TSDRGPU_DENOISE_NLM


def denoise_mode(spec: str):
    """"off", "nlm:<h>" or "nlm:<h>:<R>:<P>" (the host library's TSDR_DENOISE spelling) -> (mode, h_milli, R, P), read by
    tsdrgpu_denoise_parse."""
    out = [C.c_int() for _ in range(4)]
    if lib().tsdrgpu_denoise_parse(spec.encode(), *[C.byref(o) for o in out]) != 0:
        raise ValueError(f"denoise must be 'off' or 'nlm:<h>[:<R>:<P>]' with h in [0.001, 1], R in [1, 10] and P in [1, 3], not {spec!r}")
    return tuple(o.value for o in out)


DEBLUR_OFF, DEBLUR_RL = 0, 1                       # TSDRGPU_DEBLUR_OFF / TSDRGPU_DEBLUR_RL


def deblur_mode(spec: str):
    """"off", "rl:<sigma>" or "rl:<sigma>:<I>" (the host library's TSDR_DEBLUR spelling) -> (mode, sigma_centi, I), read by
    tsdrgpu_deblur_parse."""
    out = [C.c_int() for _ in range(3)]
    if lib().tsdrgpu_deblur_parse(spec.encode(), *[C.byref(o) for o in out]) != 0:
        raise ValueError(f"deblur must be 'off' or 'rl:<sigma>[:<I>]' with sigma in [0.25, 4] and I in [1, 64], not {spec!r}")
    return tuple(o.value for o in out)


STACK_OFF, STACK_ALIGN, STACK_ADAPT, STACK_TRACK, STACK_ROBUST = 0, 1, 4, 8, 16   # TSDRGPU_STACK_OFF / _ALIGN / _ADAPT / _TRACK / _ROBUST
VALUE_ID_STACK_DRIFT = 101                          # TSDRGPU_VALUE_ID_STACK_DRIFT


class StackRecord(C.Structure):
    """tsdrgpu_stack_record_t"""
    _fields_ = [("offset", C.c_double), ("score", C.c_int64), ("dx", C.c_int32), ("dy", C.c_int32),
                ("restarted", C.c_int32), ("changed", C.c_int32)]


def stack_mode(spec: str):
    """"off", "align:<N>[:<rx>x<ry>]", "adapt:<N>[:<rx>x<ry>]", "track:<N>[:<rx>x<ry>]" or "robust:<N>[:<rx>x<ry>]" (the host
    library's TSDR_STACK spelling) -> (mode, N, rx, ry), read by tsdrgpu_stack_parse."""
    out = [C.c_int() for _ in range(4)]
    if lib().tsdrgpu_stack_parse(spec.encode(), *[C.byref(o) for o in out]) != 0:
        raise ValueError(f"stack must be 'off', 'align:<N>[:<rx>x<ry>]', 'adapt:<N>[:<rx>x<ry>]', 'track:<N>[:<rx>x<ry>]' or 'robust:<N>[:<rx>x<ry>]' with N in [2, 1024], rx in [1, 32] and ry in [0, 8], not {spec!r}")
    return tuple(o.value for o in out)


SUPERBAND_REFERENCE, SUPERBAND_COHERENT = 0, 1          # TSDRGPU_SUPERBAND_REFERENCE / _COHERENT


class SuperbandSpec(C.Structure):
    """tsdrgpu_superband_t"""
    _fields_ = [("mode", C.c_int32), ("hops", C.c_int32), ("overlap_pct", C.c_int32)]


class SuperbandEst(C.Structure):
    """tsdrgpu_superband_est_t: one join of a coherent stitch"""
    _fields_ = [("hop", C.c_int32), ("neighbour", C.c_int32), ("tau0", C.c_int32), ("kappa0", C.c_int32), ("tau_1024", C.c_int64),
                ("tau", C.c_double), ("g_re", C.c_double), ("g_im", C.c_double), ("rho", C.c_double)]


def superband_spec(spec: str) -> SuperbandSpec:
    """"reference" or "coherent[:<H>[:<o>]]" (the host library's TSDR_SUPERBAND spelling), read by tsdrgpu_superband_parse."""
    out = SuperbandSpec()
    if lib().tsdrgpu_superband_parse(spec.encode(), C.byref(out)) != 0:
        raise ValueError(f"superband must be 'reference' or 'coherent[:<H>[:<o>]]' with H in {{2, 4, 8}} and o in [10, 50], not {spec!r}")
    return out


def superband_schedule(spec: str, samplerate: int, refreshrate: float):
    """(N, D, retune offsets in Hz) of a coherent spec, from tsdrgpu_superband_schedule."""
    s = superband_spec(spec)
    n, d = C.c_uint32(0), C.c_uint32(0)
    offs = (C.c_int32 * max(s.hops, 1))()
    if lib().tsdrgpu_superband_schedule(C.byref(s), samplerate, refreshrate, C.byref(n), C.byref(d), offs) != 0:
        raise ValueError(f"no coherent superbandwidth schedule for {spec!r} at {samplerate} S/s and {refreshrate} Hz")
    return n.value, d.value, list(offs)


_SIGS = {
    "tsdrgpu_device_count": (C.c_int, []),
    "tsdrgpu_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "tsdrgpu_destroy": (None, [C.c_void_p]),
    "tsdrgpu_last_error": (C.c_char_p, [C.c_void_p]),
    "tsdrgpu_sm_count": (C.c_int, [C.c_void_p]),
    "tsdrgpu_launch_count": (C.c_uint64, [C.c_void_p]),
    "tsdrgpu_profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_profile_collect": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_int, C.POINTER(C.c_int)]),
    "tsdrgpu_malloc": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    "tsdrgpu_free": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_malloc_host": (C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    "tsdrgpu_free_host": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_memcpy_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "tsdrgpu_memcpy_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "tsdrgpu_memcpy_d2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]),
    "tsdrgpu_device_numa_node": (C.c_int, [C.c_void_p]),
    "tsdrgpu_bind_thread_near_device": (C.c_int, [C.c_void_p]),
    "tsdrgpu_memset": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_size_t]),
    "tsdrgpu_stream_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_stream_destroy": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_stream_sync": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_geometry": (None, [C.c_uint32, C.c_int, C.c_double, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "tsdrgpu_plan_resample": (C.c_uint64, [C.POINTER(C.c_double), C.c_void_p, C.c_uint32, C.c_uint32, C.c_double, C.c_double, C.c_void_p]),
    "tsdrgpu_fft_reference_eps": (None, [C.c_int, C.c_int, C.POINTER(C.c_double)]),
    "tsdrgpu_gauss_taps": (None, [C.POINTER(C.c_float * 5)]),
    "tsdrgpu_pll_step": (C.c_int, [C.POINTER(C.c_double), C.c_int32, C.c_int32, C.c_double]),
    "tsdrgpu_am_demod": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "tsdrgpu_resampler_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_resampler_destroy": (None, [C.c_void_p]),
    "tsdrgpu_resampler_reset": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_resampler_get_state": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "tsdrgpu_resampler_set_state": (C.c_int, [C.c_void_p, C.c_void_p, C.c_double, C.c_double]),
    "tsdrgpu_resampler_plan": (C.c_uint64, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_double, C.c_double]),
    "tsdrgpu_resampler_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_uint32,
                                        C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "tsdrgpu_resampler_set_mag_out": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_resampler_set_kernel": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_sinc_taps": (C.c_int, [C.c_double, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_sinc_tile_pixels": (C.c_uint32, [C.c_double]),
    "tsdrgpu_channel_parse": (C.c_int, [C.c_char_p, C.POINTER(ChannelSpec)]),
    "tsdrgpu_channel_taps": (C.c_int, [C.POINTER(ChannelSpec), C.c_uint32, C.c_void_p, C.POINTER(C.c_int)]),
    "tsdrgpu_chanfilt_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_chanfilt_destroy": (None, [C.c_void_p]),
    "tsdrgpu_chanfilt_reset": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_chanfilt_set": (C.c_int, [C.c_void_p, C.POINTER(ChannelSpec), C.c_uint32]),
    "tsdrgpu_chanfilt_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]),
    "tsdrgpu_spectrum_parse": (C.c_int, [C.c_char_p, C.POINTER(WelchSpec)]),
    "tsdrgpu_spectrum_window": (C.c_int, [C.c_int, C.c_void_p]),
    "tsdrgpu_spectrum_k": (C.c_uint32, [C.POINTER(WelchSpec), C.c_uint32]),
    "tsdrgpu_spectrum_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_spectrum_destroy": (None, [C.c_void_p]),
    "tsdrgpu_spectrum_set": (C.c_int, [C.c_void_p, C.POINTER(WelchSpec), C.c_uint32]),
    "tsdrgpu_spectrum_reset": (C.c_int, [C.c_void_p]),
    "tsdrgpu_spectrum_plan": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint32)]),
    "tsdrgpu_spectrum_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32,
                                       C.POINTER(C.c_uint32)]),
    "tsdrgpu_coherence_parse": (C.c_int, [C.c_char_p, C.POINTER(CoherenceSpec)]),
    "tsdrgpu_coherence_n": (C.c_uint32, [C.c_uint32, C.c_double]),
    "tsdrgpu_coherence_window": (C.c_int, [C.c_int, C.c_double, C.c_uint32, C.c_void_p]),
    "tsdrgpu_coherence_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_coherence_destroy": (None, [C.c_void_p]),
    "tsdrgpu_coherence_set": (C.c_int, [C.c_void_p, C.POINTER(CoherenceSpec), C.c_uint32, C.c_double]),
    "tsdrgpu_coherence_reset": (C.c_int, [C.c_void_p]),
    "tsdrgpu_coherence_plan": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint32)]),
    "tsdrgpu_coherence_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint32,
                                        C.POINTER(C.c_uint32)]),
    "tsdrgpu_framestage_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_framestage_destroy": (None, [C.c_void_p]),
    "tsdrgpu_framestage_reset": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_framestage_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                         C.c_uint, C.c_void_p, C.POINTER(FrameResult)]),
    "tsdrgpu_framestage_run_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                               C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tsdrgpu_framestage_set_overlap": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_framestage_set_autogain": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "tsdrgpu_autogain_ppm": (C.c_int, [C.c_char_p]),
    "tsdrgpu_frame_levels": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tsdrgpu_framestage_set_contrast": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_contrast_parse": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_clahe": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_framestage_set_denoise": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_denoise_parse": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_nlm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_deblur_parse": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_deblur_taps": (C.c_int, [C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "tsdrgpu_deblur": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_framestage_set_deblur": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_stack_parse": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_stack_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_stack_destroy": (None, [C.c_void_p]),
    "tsdrgpu_stack_reset": (C.c_int, [C.c_void_p]),
    "tsdrgpu_stack_set": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_stack_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "tsdrgpu_stack_vectors": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "tsdrgpu_stack_robust_counts": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tsdrgpu_framestage_set_stack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_framestage_stack_records": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "tsdrgpu_framestage_join": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_autogain": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                   C.c_int, C.c_void_p, C.c_void_p, C.c_float]),
    "tsdrgpu_timelowpass": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_void_p, C.c_void_p]),
    "tsdrgpu_average_v_h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "tsdrgpu_gaussianblur": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "tsdrgpu_pixels_argb": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "tsdrgpu_fft_getrealsize": (C.c_uint32, [C.c_uint32]),
    "tsdrgpu_fft": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int]),
    "tsdrgpu_autocorrelation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    "tsdrgpu_autocorrelation_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64]),
    "tsdrgpu_crosscorrelation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]),
    "tsdrgpu_frd_create": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_frd_destroy": (None, [C.c_void_p]),
    "tsdrgpu_frd_reset": (C.c_int, [C.c_void_p]),
    "tsdrgpu_frd_set_overlap": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_frd_join": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_frd_capture_size": (C.c_uint32, [C.c_uint32]),
    "tsdrgpu_frd_windows": (None, [C.c_uint32] + [C.POINTER(C.c_int)] * 4),
    "tsdrgpu_frd_run": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]),
    "tsdrgpu_frd_run_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_int, C.POINTER(C.c_uint64)]),
    "tsdrgpu_frd_run_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64)]),
    "tsdrgpu_frd_dump_csv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_char_p]),
    "tsdrgpu_frd_get_plots": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_int]),
    "tsdrgpu_frd_peaks": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "tsdrgpu_plot_peaks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int32)]),
    "tsdrgpu_frd_peaks_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "tsdrgpu_videomode_from_peaks": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "tsdrgpu_accumulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int]),
    "tsdrgpu_complex_to_abs_diff": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
    "tsdrgpu_superb_bestfit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "tsdrgpu_superb_stitch": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_void_p,
                                        C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_superb_local_spectra": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "tsdrgpu_superb_lags": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(C.c_int)]),
    "tsdrgpu_superb_residue_ifft_lag": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.c_int, C.POINTER(C.c_int), C.c_void_p]),
    "tsdrgpu_superb_mgpu_create": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.POINTER(C.c_void_p)]),
    "tsdrgpu_superb_mgpu_destroy": (None, [C.c_void_p]),
    "tsdrgpu_superb_mgpu_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_superb_mgpu_connect_ipc": (C.c_int, [C.c_void_p, C.c_void_p]),
    "tsdrgpu_superb_mgpu_connect_local": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "tsdrgpu_superb_mgpu_disconnect": (C.c_int, [C.c_void_p]),
    "tsdrgpu_superb_mgpu_stitch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_uint32)]),
    "tsdrgpu_superb_mgpu_stream_window": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_superb_mgpu_lags": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32)]),
    "tsdrgpu_superband_parse": (C.c_int, [C.c_char_p, C.POINTER(SuperbandSpec)]),
    "tsdrgpu_superband_schedule": (C.c_int, [C.POINTER(SuperbandSpec), C.c_uint32, C.c_double, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                             C.POINTER(C.c_int32)]),
    "tsdrgpu_superb_stitch_coherent": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "tsdrgpu_pipeline_create": (C.c_int, [C.c_void_p, C.POINTER(PipelineConfig), FRAME_CB, VALUE_CB, PLOT_CB, C.c_void_p, C.POINTER(C.c_void_p)]),
    "tsdrgpu_pipeline_destroy": (None, [C.c_void_p]),
    "tsdrgpu_pipeline_process": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int64]),
    "tsdrgpu_convert_samples": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_void_p]),
    "tsdrgpu_pipeline_process_raw": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_int64]),
    "tsdrgpu_pipeline_process_raw_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_uint64, C.c_int64]),
    "tsdrgpu_pipeline_sync_input": (C.c_int, [C.c_void_p]),
    "tsdrgpu_pipeline_flush": (C.c_int, [C.c_void_p]),
    "tsdrgpu_pipeline_set_param_int": (C.c_int, [C.c_void_p, C.c_int, C.c_uint32]),
    "tsdrgpu_pipeline_set_resolution": (C.c_int, [C.c_void_p, C.c_int, C.c_double]),
    "tsdrgpu_pipeline_set_samplerate": (C.c_int, [C.c_void_p, C.c_uint32]),
    "tsdrgpu_pipeline_set_retune": (C.c_int, [C.c_void_p, RETUNE_CB]),
    "tsdrgpu_pipeline_set_motionblur": (C.c_int, [C.c_void_p, C.c_float]),
    "tsdrgpu_pipeline_set_host_registration": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_pipeline_set_superb_devices": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int]),
    "tsdrgpu_pipeline_set_superband": (C.c_int, [C.c_void_p, C.POINTER(SuperbandSpec)]),
    "tsdrgpu_pipeline_superband_estimates": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
    "tsdrgpu_pipeline_set_reports": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_resampler": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_pipeline_set_autogain": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_contrast": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_denoise": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_deblur": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_stack": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "tsdrgpu_pipeline_set_channel": (C.c_int, [C.c_void_p, C.POINTER(ChannelSpec)]),
    "tsdrgpu_pipeline_set_spectrum": (C.c_int, [C.c_void_p, C.POINTER(WelchSpec)]),
    "tsdrgpu_pipeline_set_coherence": (C.c_int, [C.c_void_p, C.POINTER(CoherenceSpec)]),
    "tsdrgpu_detect_videomode": (C.c_int, [C.POINTER(C.c_double), C.c_int, C.c_int, C.POINTER(C.c_double), C.c_int, C.c_int, C.c_uint32,
                                           C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "tsdrgpu_pipeline_set_output_argb": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "tsdrgpu_pixels_argb_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p]),
    "tsdrgpu_pipeline_sync": (C.c_int, [C.c_void_p, C.c_int]),
    "tsdrgpu_pipeline_get_geometry": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double)]),
    "tsdrgpu_pipeline_stats": (C.c_int, [C.c_void_p, C.POINTER(PipelineStats)]),
}

#: every symbol include/tsdrgpu.h declares (tests check the built library exports all of them)
DECLARED_SYMBOLS = tuple(_SIGS)

_lib = None


def lib() -> C.CDLL:
    """The loaded libtsdrgpu.so.  Raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make -C tempestsdr_b200/csrc` "
                               "(or __graft_entry__.build()).  There is no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class TsdrGpuError(RuntimeError):
    pass


def check(rc: int, ctx=None) -> None:
    if rc != OK:
        msg = lib().tsdrgpu_last_error(ctx)
        raise TsdrGpuError(f"libtsdrgpu error {rc}: {msg.decode() if msg else '?'}")
