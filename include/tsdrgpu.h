/*
 * tsdrgpu.h -- C-ABI of the H100 (sm_90a) implementation of TempestSDR's IQ->raster DSP path.
 *
 * This is the drop-in boundary below the reference's own C host code: plain C, plain pointers and sizes, no
 * C++ or torch types.  Every entry point names the reference function(s) it replaces
 * (paths relative to /root/reference/TempestSDR/src).  The tsdr_* / tsdrplugin_* ABI above it is declared
 * unchanged in TSDRLibrary.h / TSDRPlugin.h / TSDRCodes.h beside this file.
 *
 * Conventions
 *   - every function returns TSDRGPU_OK (0) or a negative TSDRGPU_E* code; tsdrgpu_last_error() gives text;
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream); calls are asynchronous on
 *     that stream unless the comment says "synchronises";
 *   - pointers named d_* are device pointers on the context's device, h_* are host pointers;
 *   - there is NO CPU fallback: without a CUDA device every call fails with TSDRGPU_ENODEVICE.
 */
#ifndef TSDRGPU_H_
#define TSDRGPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TSDRGPU_API __attribute__((visibility("default")))
#else
#define TSDRGPU_API
#endif

enum {
	TSDRGPU_OK        = 0,
	TSDRGPU_ENODEVICE = -1,   /* no usable CUDA device / wrong architecture */
	TSDRGPU_ECUDA     = -2,   /* a CUDA runtime call failed (text in tsdrgpu_last_error) */
	TSDRGPU_EINVAL    = -3,   /* bad argument */
	TSDRGPU_ENOMEM    = -4,
	TSDRGPU_ECAPACITY = -5    /* caller's output buffer too small */
};

typedef struct tsdrgpu_ctx tsdrgpu_ctx_t;

/* ------------------------------------------------------------------------------------------------ context */
TSDRGPU_API int         tsdrgpu_device_count(void);
TSDRGPU_API int         tsdrgpu_create(tsdrgpu_ctx_t **ctx, int device);
TSDRGPU_API void        tsdrgpu_destroy(tsdrgpu_ctx_t *ctx);
TSDRGPU_API const char *tsdrgpu_last_error(tsdrgpu_ctx_t *ctx);      /* ctx may be NULL (creation errors) */
TSDRGPU_API int         tsdrgpu_sm_count(tsdrgpu_ctx_t *ctx);
/* number of kernels this library has launched through ctx since creation (bench.py's gpu_launches) */
TSDRGPU_API uint64_t    tsdrgpu_launch_count(tsdrgpu_ctx_t *ctx);

/* per-kernel timing for roofline reporting: when enabled, the library brackets its main kernel launches with CUDA
 * events on the launching stream.  collect() synchronises the device, returns per-name totals (names: cap x 48
 * chars) and resets.  Not for production paths (adds two event records per launch). */
TSDRGPU_API int tsdrgpu_profile_enable(tsdrgpu_ctx_t *ctx, int on);
TSDRGPU_API int tsdrgpu_profile_collect(tsdrgpu_ctx_t *ctx, char *names, double *total_ms, uint64_t *counts, int cap, int *n);

/* plumbing for C hosts that do not bring their own allocator (Python callers use torch tensors instead) */
TSDRGPU_API int tsdrgpu_malloc(tsdrgpu_ctx_t *ctx, size_t bytes, void **d_ptr);
TSDRGPU_API int tsdrgpu_free(tsdrgpu_ctx_t *ctx, void *d_ptr);
TSDRGPU_API int tsdrgpu_malloc_host(tsdrgpu_ctx_t *ctx, size_t bytes, void **h_ptr);   /* pinned, on the device's NUMA node when known */
/* NUMA node the device hangs off (sysfs), -1 when unknown; pin the calling thread to that node's cores (0 = done).
 * TSDRGPU_NO_NUMA=1 switches both off. */
TSDRGPU_API int tsdrgpu_device_numa_node(tsdrgpu_ctx_t *ctx);
TSDRGPU_API int tsdrgpu_bind_thread_near_device(tsdrgpu_ctx_t *ctx);
TSDRGPU_API int tsdrgpu_free_host(tsdrgpu_ctx_t *ctx, void *h_ptr);
TSDRGPU_API int tsdrgpu_memcpy_h2d(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, const void *h_src, size_t bytes);
TSDRGPU_API int tsdrgpu_memcpy_d2h(tsdrgpu_ctx_t *ctx, void *stream, void *h_dst, const void *d_src, size_t bytes);
TSDRGPU_API int tsdrgpu_memcpy_d2d(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, const void *d_src, size_t bytes);
TSDRGPU_API int tsdrgpu_memset(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, int value, size_t bytes);
TSDRGPU_API int tsdrgpu_stream_create(tsdrgpu_ctx_t *ctx, void **stream);
TSDRGPU_API int tsdrgpu_stream_destroy(tsdrgpu_ctx_t *ctx, void *stream);
TSDRGPU_API int tsdrgpu_stream_sync(tsdrgpu_ctx_t *ctx, void *stream);                 /* synchronises */

/* ---------------------------------------------------------------------------- host-only scalar helpers (no GPU needed)
 * a4: set_internal_samplerate's geometry (TSDRLibrary.c:540-550). */
TSDRGPU_API void tsdrgpu_geometry(uint32_t samplerate, int height, double refreshrate, int *width, double *pixelrate,
                                  double *pixeltimeoversampletime);
/* one decimator block as the device sees it (40 bytes, no padding) */
typedef struct {
	uint64_t in_start;    /* first sample of the block in the input stream (sample index, not float index) */
	uint64_t out_start;   /* first pixel of the block in the output stream */
	uint32_t size;        /* samples in the block                            (dsp.c:261) */
	uint32_t n_out;       /* output_samples                                  (dsp.c:262) */
	double   r;           /* sampletimeoverpixel = upsample_by/downsample_by (dsp.c:258) */
	double   phase;       /* offset_sample = -offset * r                     (dsp.c:272) */
} tsdrgpu_rs_block_t;
/* the per-call phase recurrence of dsp_resample_process (dsp.c:258-262,272,306) for nblocks consecutive calls:
 * advances *offset, returns the total of the reference's output_samples (UINT64_MAX if a block yields none:
 * the reference asserts there, extbuffer.c:48).  `blocks` may be NULL (count only). */
TSDRGPU_API uint64_t tsdrgpu_plan_resample(double *offset, const uint32_t *sizes, uint32_t uniform, uint32_t nblocks,
                                           double upsample_by, double downsample_by, tsdrgpu_rs_block_t *blocks);
/* relative angle errors eps[l] of the reference FFT's stage twiddles (half-angle recurrence, fft.c:132-165): stage l
 * rotates by (pi/2^l)(1+eps[l]) instead of pi/2^l.  Used by tsdrgpu_fft to track the reference at large N. */
TSDRGPU_API void tsdrgpu_fft_reference_eps(int stages, int inverse, double *eps);
/* host-only: the GUI's auto-resolution arithmetic on the two autocorrelation plots (JavaGUI .../PlotVisualizer.java:203-236,
 * Main.java:1233-1253,1301-1303,1346-1350): first strict maximum of each plot -> fps, height.  Optional outputs may be NULL. */
TSDRGPU_API int tsdrgpu_detect_videomode(const double *frame_plot, int frame_offset, int frame_len, const double *line_plot, int line_offset,
                                         int line_len, uint32_t samplerate, double *fps, int *height, int *frame_index, int *line_index);
/* frameratepll's write-back (syncdetector.c:141-152) for one frame, from the frame stage's per-frame result: returns 1 and
 * moves *refreshrate when the reference would (PLL on is the caller's condition; x_vx != 0 is checked here), else 0. */
TSDRGPU_API int tsdrgpu_pll_step(double *refreshrate, int32_t x_vx, int32_t pll_state, double avg_speed);
/* the same arithmetic from peak indices picked elsewhere (tsdrgpu_frd_peaks: on the device) */
TSDRGPU_API int tsdrgpu_videomode_from_peaks(int frame_offset, int frame_index, int line_offset, int line_index, uint32_t samplerate, double *fps, int *height);
/* the normalised 5-tap Gaussian of gaussian.c:16-30 */
TSDRGPU_API void tsdrgpu_gauss_taps(float taps[5]);

/* ---------------------------------------------------------------------------- a2  AM demodulation
 * replaces am_demod (TSDRLibrary.c:244-262): out[k] = sqrtf(I*I + Q*Q), bit-exact (no FMA, IEEE sqrt). */
TSDRGPU_API int tsdrgpu_am_demod(tsdrgpu_ctx_t *ctx, void *stream, const float *d_iq, uint64_t pairs, float *d_out);

/* ---------------------------------------------------------------------------- a6  resampler (+ fused a2)
 * replaces dsp_resample_init / dsp_resample_process / dsp_resample_t (dsp.c:250-307, dsp.h:79-82), optionally
 * fused with am_demod.  The object carries the reference's {contrib, offset} across calls; `offset` lives on
 * the host (it depends only on sizes and rates), `contrib` on the device (it depends on the data).
 *
 * One run processes `nblocks` CONSECUTIVE decimator blocks (the reference's decimatingthread calls
 * dsp_resample_process once per 0.1 frame, TSDRLibrary.c:335-340); the per-block phase recurrence
 * (dsp.c:262,272,306) is replayed on the host in C, the pixels are computed on the GPU, bit-exact.
 * Deviation: a slot the reference leaves stale because its loop writes one pixel fewer than output_samples
 * (exact-integer landings, e.g. r == 2.0) is written as 0.0f.
 */
typedef struct tsdrgpu_resampler tsdrgpu_resampler_t;
TSDRGPU_API int  tsdrgpu_resampler_create(tsdrgpu_ctx_t *ctx, tsdrgpu_resampler_t **r);
TSDRGPU_API void tsdrgpu_resampler_destroy(tsdrgpu_resampler_t *r);
TSDRGPU_API int  tsdrgpu_resampler_reset(tsdrgpu_resampler_t *r, void *stream);                 /* dsp_resample_init */
TSDRGPU_API int  tsdrgpu_resampler_get_state(tsdrgpu_resampler_t *r, void *stream, double *contrib, double *offset); /* synchronises */
TSDRGPU_API int  tsdrgpu_resampler_set_state(tsdrgpu_resampler_t *r, void *stream, double contrib, double offset);
/* host-only: pixels the next run would produce (sum of the reference's output_samples), state untouched.
 * block_sizes may be NULL: then every block has `uniform_block` samples. */
TSDRGPU_API uint64_t tsdrgpu_resampler_plan(tsdrgpu_resampler_t *r, const uint32_t *block_sizes, uint32_t uniform_block,
                                            uint32_t nblocks, double upsample_by, double downsample_by);
/* d_in: IQ pairs (in_is_iq != 0, 2 floats per sample) or magnitudes (1 float per sample), blocks back to back.
 * Writes *h_n_out pixels to d_out (blocks back to back) and advances the state. */
TSDRGPU_API int  tsdrgpu_resampler_run(tsdrgpu_resampler_t *r, void *stream, const float *d_in, int in_is_iq,
                                       const uint32_t *block_sizes, uint32_t uniform_block, uint32_t nblocks,
                                       double upsample_by, double downsample_by, int nearest_neighbour,
                                       float *d_out, uint64_t out_capacity, uint64_t *h_n_out);

/* One-shot: the NEXT tsdrgpu_resampler_run with IQ input also writes |x| of every input sample to d_mag (one float per
 * sample, blocks back to back like d_in) -- am_demod's output for the frame-rate detector (TSDRLibrary.c:286-292 feeds both
 * consumers from one demodulated buffer) without a second pass over the IQ.  A refused run leaves it armed, as it leaves
 * the state: a run refused for asking magnitudes of magnitude input or of the nearest-neighbour mode is refused again
 * until the caller disarms it (d_mag = NULL). */
TSDRGPU_API int  tsdrgpu_resampler_set_mag_out(tsdrgpu_resampler_t *r, float *d_mag);

/* ---------------------------------------------------------------------------- a2-  channel filter (beyond the reference)
 * An opt-in complex FIR on the interleaved float32 IQ stream, before AM demodulation.  am_demod takes |x| of everything in the
 * band, so a carrier, a switching spur or the DC spike of a zero-IF front end beats with the video signal and leaves stripes over
 * the whole frame; in IQ the interferer still sits in its own frequency band, where this filter removes it.  The response is one
 * pass band minus up to four stop bands, in Hz relative to the tuned centre.
 *
 * Spec (tsdrgpu_channel_t).  taps == 0: off.  Otherwise T = taps is odd with 9 <= T <= 257; every frequency f has |f| <=
 * TSDRGPU_CHANNEL_MAX_HZ; lo < hi for every band; every stop band lies inside the pass band (pass_lo <= lo, hi <= pass_hi);
 * 0 <= nstop <= 4 and the stop bands are pairwise disjoint (two bands may touch, max(lo) < min(hi) is an overlap).  A pure notch
 * is a pass band wider than the sample rate, e.g. pass:-250000000:250000000,stop:-20000:20000.
 *
 * Taps (tsdrgpu_channel_taps), in double throughout, for t = 0 .. T-1 and the integer d = t - (T-1)/2:
 *   every band edge is f/fs clamped to [-0.5, 0.5]; the stop band edges are then clamped into the clamped pass band [P0, P1];
 *   g_[a,b](0) = b - a, and for d != 0  Re g = (sin 2 pi b d - sin 2 pi a d) / (2 pi d),  Im g = (cos 2 pi a d - cos 2 pi b d) / (2 pi d)
 *   w(d) = I0(beta sqrt(1 - (2d/(T-1))^2)) / I0(beta),  beta = TSDRGPU_CHANNEL_BETA
 *   h[t] = w(d) (g_pass(d) - sum_k g_stop_k(d)),  Re and Im each rounded to float32 once.
 *   The taps depend on the spec and fs only.
 * Filter.  Output pair n is y[n] = sum_{t=0}^{T-1} x[n-t] h[t], float32 in tap order t = 0, 1, ... with no contraction:
 *   pr = xr hr - xi hi,  pi = xr hi + xi hr  (each product rounded, then the difference / sum);
 *   yr = pr, yi = pi at t = 0, then yr = yr + pr, yi = yi + pi.
 *   One pair out per pair in; the group delay is (T-1)/2 samples, so the picture moves by about (T-1)/2 * r pixels (r = pixels per
 *   sample), which AUTOSHIFT re-centres.
 * State.  x[n] for n < 0 of a run is the history: the last T-1 input pairs of the runs before, zero before the first sample.  It is
 * kept on the device (two buffers: a run reads one and writes the other) and zeroed at create, at reset and by a set that changes
 * the taps (a new spec or a new fs); a set that leaves the taps as they are keeps it. */
#define TSDRGPU_CHANNEL_MAX_STOPS     4
#define TSDRGPU_CHANNEL_MIN_TAPS      9
#define TSDRGPU_CHANNEL_MAX_TAPS      257
#define TSDRGPU_CHANNEL_DEFAULT_TAPS  65
#define TSDRGPU_CHANNEL_MAX_HZ        250000000LL      /* the host library's sample-rate limit / 2 */
#define TSDRGPU_CHANNEL_BETA          6.0
typedef struct {
	int32_t taps;                                    /* T; 0 = off */
	int32_t nstop;
	int64_t pass_lo_hz, pass_hi_hz;
	int64_t stop_lo_hz[TSDRGPU_CHANNEL_MAX_STOPS], stop_hi_hz[TSDRGPU_CHANNEL_MAX_STOPS];
} tsdrgpu_channel_t;
/* host-only: the spelling shared by the host library's TSDR_CHANNEL and Python.  "off", or "pass:<lo>:<hi>" followed by zero to
 * four ",stop:<a>:<b>" and optionally ",taps:<T>" (default TSDRGPU_CHANNEL_DEFAULT_TAPS).  Frequencies are decimal integers in Hz
 * with an optional leading '-'; nothing else (no blank, '+', exponent or unit).  The result must be a valid spec (above).
 * TSDRGPU_OK with *out set (all zero for "off"), else TSDRGPU_EINVAL and *out untouched. */
TSDRGPU_API int  tsdrgpu_channel_parse(const char *spec, tsdrgpu_channel_t *out);
/* host-only: the taps of a valid spec (taps != 0) at sample rate fs > 0, 2T floats re/im interleaved; taps may be NULL to query *T */
TSDRGPU_API int  tsdrgpu_channel_taps(const tsdrgpu_channel_t *spec, uint32_t fs, float *taps, int *T);
typedef struct tsdrgpu_chanfilt tsdrgpu_chanfilt_t;
TSDRGPU_API int  tsdrgpu_chanfilt_create(tsdrgpu_ctx_t *ctx, tsdrgpu_chanfilt_t **f);
TSDRGPU_API void tsdrgpu_chanfilt_destroy(tsdrgpu_chanfilt_t *f);
TSDRGPU_API int  tsdrgpu_chanfilt_reset(tsdrgpu_chanfilt_t *f, void *stream);           /* zeroes the history */
/* a valid spec (taps != 0) and fs > 0, used from the next run on */
TSDRGPU_API int  tsdrgpu_chanfilt_set(tsdrgpu_chanfilt_t *f, const tsdrgpu_channel_t *spec, uint32_t fs);
/* asynchronous: `pairs` IQ pairs from d_in to d_out (both 8-byte aligned, not overlapping), history carried.  Needs a set first. */
TSDRGPU_API int  tsdrgpu_chanfilt_run(tsdrgpu_chanfilt_t *f, void *stream, const float *d_in, uint64_t pairs, float *d_out);

/* ---------------------------------------------------------------------------- a19+  Welch power spectrum (beyond the reference)
 * An opt-in spectrum of the IQ stream, so that a user can find the carriers, spurs and the DC spike around a harmonic of the pixel
 * clock and place the channel filter's stop bands (Hz relative to the tuned centre) without a second program.
 *
 * Spec (tsdrgpu_welch_t).  n == 0: off.  Otherwise N = n is a power of two in [TSDRGPU_SPECTRUM_MIN_N, TSDRGPU_SPECTRUM_MAX_N] and
 * rate (reports per second of stream time) is an integer in [1, TSDRGPU_SPECTRUM_MAX_RATE].
 * Window: the periodic 4-term Blackman-Harris window of N points,
 *   w[n] = 0.35875 - 0.48829 cos(2 pi n/N) + 0.14128 cos(4 pi n/N) - 0.01168 cos(6 pi n/N),
 *   built in double (tsdrgpu_spectrum_window) and stored as float32; sidelobes at -92 dB.  There is no other window.
 * Segments.  A run is a stretch of the stream with no break in it.  Segment j of a run covers the pairs [j N/2, j N/2 + N) counted
 *   from the run's first pair (hop N/2, 50 % overlap).  A run ends at a discontinuity (tsdrgpu_spectrum_run with discontinuity != 0,
 *   the pipeline's samples_dropped != 0): only its partial segment is discarded, completed segments still count toward the next
 *   report.  A reset, or a set with a new spec or sample rate, also discards the completed segments of the report in progress.
 * Report.  Each report averages K consecutive completed segments, K = max(1, floor(fs / (rate N/2))) (tsdrgpu_spectrum_k):
 *   P[k] = (1/K) sum_seg |sum_n w[n] x[n] e^{-2 pi i k n/N}|^2 / (sum_n w[n])^2
 *   (w the float32 window, sum_n w[n] in double), in double, linear power: a complex tone of amplitude A at a bin centre reads A^2,
 *   full scale 1.0 (0 dBFS).  Value i of a report is bin k = i - N/2 (fftshift order), at (i - N/2) fs/N Hz from the tuned centre.
 * Computation: x[n] w[n] rounded to float32 (__fmul_rn), float32 FFT with the exact DFT's stage angles, |X|^2 and every sum in double.
 *   Agrees with a float64 evaluation of the definition to 1e-6 of the report's largest sqrt(P) in amplitude.  The same calls with the
 *   same blocks give the same bits (no atomics); another cut of the stream may change the last bits. */
#define TSDRGPU_SPECTRUM_MIN_N        256
#define TSDRGPU_SPECTRUM_MAX_N        65536
#define TSDRGPU_SPECTRUM_DEFAULT_RATE 10
#define TSDRGPU_SPECTRUM_MAX_RATE     100
typedef struct {
	int32_t n;                                       /* N; 0 = off */
	int32_t rate;                                    /* reports per second of stream time */
} tsdrgpu_welch_t;
/* host-only: the spelling shared by the host library's TSDR_SPECTRUM and Python.  "off" or "welch:<N>[:<rate>]" (rate default
 * TSDRGPU_SPECTRUM_DEFAULT_RATE); N and rate are decimal digits only (no sign, blank or leading '+').  TSDRGPU_OK with *out set
 * (zeros for "off"), else TSDRGPU_EINVAL and *out untouched. */
TSDRGPU_API int  tsdrgpu_spectrum_parse(const char *spec, tsdrgpu_welch_t *out);
/* host-only: the window of a valid N in double (before its rounding to float32), N values */
TSDRGPU_API int  tsdrgpu_spectrum_window(int n, double *w);
/* host-only: K of a valid spec (n != 0) at fs > 0; 0 for anything else */
TSDRGPU_API uint32_t tsdrgpu_spectrum_k(const tsdrgpu_welch_t *spec, uint32_t fs);
typedef struct tsdrgpu_spectrum tsdrgpu_spectrum_t;
TSDRGPU_API int  tsdrgpu_spectrum_create(tsdrgpu_ctx_t *ctx, tsdrgpu_spectrum_t **s);
TSDRGPU_API void tsdrgpu_spectrum_destroy(tsdrgpu_spectrum_t *s);
/* a valid spec (n != 0) and fs > 0, used from the next run on; a new spec or fs discards the open segment and the report in progress */
TSDRGPU_API int  tsdrgpu_spectrum_set(tsdrgpu_spectrum_t *s, const tsdrgpu_welch_t *spec, uint32_t fs);
/* discards the open segment and the report in progress */
TSDRGPU_API int  tsdrgpu_spectrum_reset(tsdrgpu_spectrum_t *s);
/* host-only: the number of reports the next run of `pairs` pairs would complete (state untouched) */
TSDRGPU_API int  tsdrgpu_spectrum_plan(const tsdrgpu_spectrum_t *s, uint64_t pairs, int discontinuity, uint32_t *nreports);
/* asynchronous: `pairs` IQ pairs from d_iq (8-byte aligned; discontinuity != 0: they do not follow the pairs of the last run).  The
 * reports this run completes go to d_reports, N doubles each, in order; *h_nreports is set on return from pair counts alone (no
 * synchronisation).  More than `capacity` reports: TSDRGPU_ECAPACITY, state untouched.  d_iq is read on `stream` only, until the
 * run's work there is done; the open segment (< N pairs) is kept in the object's own memory.  Needs a set first. */
TSDRGPU_API int  tsdrgpu_spectrum_run(tsdrgpu_spectrum_t *s, void *stream, const float *d_iq, uint64_t pairs, int discontinuity,
                                      double *d_reports, uint32_t capacity, uint32_t *h_nreports);

/* ---------------------------------------------------------------------------- a19+  spectral coherence at the line rate (beyond the reference)
 * An opt-in companion of the Welch spectrum that shows which of the power around a harmonic of the pixel clock is the picture.
 * Every line of the raster carries the same horizontal blanking, so the emanation is cyclostationary at the line rate alpha: each
 * frequency it occupies is correlated with the frequency alpha away from it.  Broadcast carriers, tones, switching spurs and receiver
 * noise have no such correlation.  The coherence reads about 0 for them (an estimator floor of about 1/sqrt(K)) and rises where the
 * picture's energy is.  Its axis is the spectrum's (plot 100), so the two overlay: pass the bands where it rises, stop the others.
 * How far it rises on real captures (sync pulses, TMDS control periods) has not been measured; on synthetic video with a weak
 * blanking level it is about 2.2 x the floor at K = 390 and 5 x at K = 3906 (DESIGN 5.5).
 *
 * Spec (tsdrgpu_coherence_t).  rate == 0: off.  Otherwise rate (reports per second of stream time) is an integer in
 *   [1, TSDRGPU_COHERENCE_MAX_RATE].
 * Cycle frequency.  alpha > 0 is the line rate in Hz: an argument of tsdrgpu_coherence_set; the pipeline uses height x refresh rate,
 *   read at the first segment of each report (PLL steps take effect from the next report).
 * N.  The smallest power of two with N >= 16 fs / alpha, and at least 256 (tsdrgpu_coherence_n): alpha lies 16 to 32 bins apart,
 *   clear of the window's +-4-bin main lobe, so U+ and U- below do not overlap.  Above 65536 the spec is unresolvable: set returns
 *   TSDRGPU_EINVAL (the pipeline delivers no coherence reports until the geometry or the sample rate changes).
 * Window and segments: the Welch spectrum's (Blackman-Harris w of N points, hop N/2).  Segment j starts at pair s_j = j N/2, counted
 *   from the first pair of the report in progress.
 * Transforms and sums, for segment j:
 *   U+-_j[k] = sum_n w+-[n] x[s_j + n] e^{-2 pi i k n/N},  w+[n] = w[n] e^{-i pi alpha n/fs},  w-[n] = conj(w+[n])
 *   C[k] = sum_j U+_j[k] conj(U-_j[k]) e^{-2 pi i alpha s_j/fs}   (the factor makes the average coherent across segments)
 *   P+-[k] = sum_j |U+-_j[k]|^2
 * Report.  Each report sums K = max(1, floor(fs / (rate N/2))) segments (the tsdrgpu_spectrum_k rule), then
 *   gamma[k] = |C[k]| / sqrt(P+[k] P-[k]) in double, 0 where P+ P- = 0.  Value i of a report is bin k = i - N/2 (fftshift order), at
 *   (i - N/2) fs/N Hz from the tuned centre: the axis of plot 100.
 * Discontinuities.  Unlike the Welch spectrum, a discontinuity (discontinuity != 0, the pipeline's samples_dropped != 0) discards the
 *   open segment AND the report in progress: a gap breaks the time reference of the phase factor.  A reset, or a set with a new rate,
 *   fs or N, also discards the report in progress; a set that changes only alpha takes effect at the next report.
 * Computation: w+ is built in double (tsdrgpu_coherence_window) and each component rounded once to float32; x w+- is a float32
 *   complex product with no contraction; float32 FFT with the exact DFT's stage angles; alpha s_j/fs is formed in double from the
 *   integer s_j and reduced mod 1 before its sincospi; products, sums and gamma in double.  The same calls with the same blocks give
 *   the same bits (no atomics). */
#define TSDRGPU_COHERENCE_DEFAULT_RATE 1
#define TSDRGPU_COHERENCE_MAX_RATE     100
typedef struct {
	int32_t rate;                                    /* reports per second of stream time; 0 = off */
} tsdrgpu_coherence_t;
/* host-only: the spelling shared by the host library's TSDR_COHERENCE and Python.  "off" or "line[:<rate>]" (rate default
 * TSDRGPU_COHERENCE_DEFAULT_RATE, decimal digits only as in tsdrgpu_spectrum_parse).  TSDRGPU_OK with *out set (rate 0 for "off"),
 * else TSDRGPU_EINVAL and *out untouched. */
TSDRGPU_API int  tsdrgpu_coherence_parse(const char *spec, tsdrgpu_coherence_t *out);
/* host-only: N at sample rate fs and line rate alpha (Hz); 0 when unresolvable (N > 65536) or fs == 0 or alpha is not > 0 */
TSDRGPU_API uint32_t tsdrgpu_coherence_n(uint32_t fs, double alpha);
/* host-only: w+ of a valid N (a power of two in [256, 65536]) in double before its rounding: 2 N values, (re, im) of each n */
TSDRGPU_API int  tsdrgpu_coherence_window(int n, double alpha, uint32_t fs, double *w2);
typedef struct tsdrgpu_coherence tsdrgpu_coherence_obj_t;
TSDRGPU_API int  tsdrgpu_coherence_create(tsdrgpu_ctx_t *ctx, tsdrgpu_coherence_obj_t **c);
TSDRGPU_API void tsdrgpu_coherence_destroy(tsdrgpu_coherence_obj_t *c);
/* a valid spec (rate != 0), fs > 0 and alpha with tsdrgpu_coherence_n(fs, alpha) != 0, used from the next run on (alpha alone: from
 * the next report on); a new rate, fs or N discards the open segment and the report in progress */
TSDRGPU_API int  tsdrgpu_coherence_set(tsdrgpu_coherence_obj_t *c, const tsdrgpu_coherence_t *spec, uint32_t fs, double alpha);
/* discards the open segment and the report in progress */
TSDRGPU_API int  tsdrgpu_coherence_reset(tsdrgpu_coherence_obj_t *c);
/* host-only: the number of reports the next run of `pairs` pairs would complete (state untouched) */
TSDRGPU_API int  tsdrgpu_coherence_plan(const tsdrgpu_coherence_obj_t *c, uint64_t pairs, int discontinuity, uint32_t *nreports);
/* asynchronous, with the contract of tsdrgpu_spectrum_run: d_iq 8-byte aligned, N doubles per report into d_reports, *h_nreports
 * from pair counts alone, more than `capacity` reports: TSDRGPU_ECAPACITY with the state untouched.  Needs a set first. */
TSDRGPU_API int  tsdrgpu_coherence_run(tsdrgpu_coherence_obj_t *c, void *stream, const float *d_iq, uint64_t pairs, int discontinuity,
                                       double *d_reports, uint32_t capacity, uint32_t *h_nreports);

/* ---------------------------------------------------------------------------- a6+  windowed-sinc resampler (beyond the reference)
 * An opt-in third kernel beside box (the default, above) and nearest-neighbour.  The reference chose the box integrator
 * to save CPU time; this mode evaluates the band-limited signal at the pixel instants instead.
 *
 * Timeline: the box mode's, unchanged.  tsdrgpu_plan_resample and the `offset` recurrence give every block the same
 * n_out pixels, so frame alignment, drop compensation, tsdr_sync and the PLL behave exactly as in box mode; only the
 * value of each pixel differs.  In box mode sample k of block b spans [k*r + phase, (k+1)*r + phase) on the pixel
 * axis, so pixel p's centre on the sample axis is tau = (p + 0.5 - phase)/r - 0.5.
 *
 * Pixel p of a block (descriptor fields r, phase, size, n_out) is, with T taps, L phases and the delay D below:
 *     q    = r_inv * ((p + 0.5) - phase) - (0.5 + D)     r_inv = 1/r; every operation one IEEE double rounding to nearest,
 *                                                         in this order: p + 0.5 (exact), - phase, * r_inv, - 8.5
 *     k0   = floor(q),  j = (int) ((q - k0) * L + 0.5)   (q - k0 and * L are exact; + 0.5 rounds once)
 *     if j == L:  j = 0, k0 += 1
 *     y    = x[k0 - (T/2 - 1)] * h[j][0],  then  y = y + x[k0 - (T/2 - 1) + t] * h[j][t]  for t = 1 .. T-1
 *            (float32; every product and sum rounded on its own: no FMA contraction)
 * where x[k] is the magnitude sqrtf(I*I + Q*Q) of sample k of the block (formed on load exactly as tsdrgpu_am_demod
 * does), k < 0 reaching back into earlier blocks of the run and, before the run's first sample, into the history.
 *
 * Delay D = T/2.  The newest tap is k0 + T/2.  Since n_out = (int)(size*r + phase) and phase = -offset*r lies in [0, 1)
 * (the recurrence keeps offset in (-1/r, 0]), the last pixel has tau < size - 0.5 - 0.5/r, so q + 0.5/L < size - D - 1
 * + (0.5 - 0.5/r + 0.5/L) < size - D and the rounded k0 is at most size - 1 - T/2: every tap lies inside the block's own
 * samples.  D = T/2 - 1 would reach one sample past the block for every r > 1.  The mode is therefore causal with no
 * look-ahead; the picture moves by a constant D*r pixels, which AUTOSHIFT re-centres.
 * History H.  The oldest tap is k0 - (T/2 - 1); the first pixel has tau > -0.5 - 0.5/r, so the taps reach back at most
 * T - 1 + ceil(0.5 + 0.5/r) samples before the block: 16 for r >= 1 (every geometry tsdrgpu_geometry produces has
 * 1 < r <= 2, because r = floor(2x)/x with x = fs/(fv*h)), 17 down to r = 1/3, 24 down to r = 1/16.  The resampler carries
 * H = 32 magnitudes; runs with r < TSDRGPU_SINC_MIN_RATIO are refused (TSDRGPU_EINVAL).
 *
 * Taps: a Kaiser-windowed sinc, beta = 5, cut-off 0.5*min(1, r) cycles per input sample (below the output's Nyquist
 * frequency when downsampling): h[j][t] = sinc(2 fc d) * I0(beta sqrt(1 - (d/(T/2))^2)) with d = t - (T/2 - 1) - j/L,
 * built in double, each phase normalised to sum 1 (flat fields stay flat under auto-gain), rounded to float32.  The
 * table depends on min(1, r) only, so it is rebuilt only when a run with r < 1 changes it.
 *
 * State: the last H magnitudes of the stream, on the device (two buffers: a run reads one and writes the other).
 * tsdrgpu_resampler_reset zeroes them, and so does switching the kernel from box to sinc.  A sinc run leaves the box
 * state `contrib` untouched (as a nearest-neighbour run does in the reference); `offset` advances as in every mode.
 * Box and nearest-neighbour runs leave the history untouched.  tsdrgpu_resampler_get_state / set_state keep their
 * box-only meaning: they do not include the history.
 */
#define TSDRGPU_SINC_TAPS      16
#define TSDRGPU_SINC_PHASES    256
#define TSDRGPU_SINC_DELAY     8                    /* T/2 */
#define TSDRGPU_SINC_HISTORY   32
#define TSDRGPU_SINC_BETA      5.0
#define TSDRGPU_SINC_MIN_RATIO 0.0625               /* 1/16: the taps then reach at most 24 <= H samples back */
enum { TSDRGPU_RS_BOX = 0, TSDRGPU_RS_SINC = 1 };
/* selects the kernel of the following runs; a run's nearest_neighbour != 0 still takes precedence */
TSDRGPU_API int  tsdrgpu_resampler_set_kernel(tsdrgpu_resampler_t *r, int kernel);
/* host-only: the tap table for ratio r in [j][t] order (L*T floats; taps may be NULL to query *T and *L only) */
TSDRGPU_API int  tsdrgpu_sinc_taps(double r, float *taps, int *T, int *L);
/* host-only: the pixels per CTA tile a sinc run at ratio r launches with (0 for r < TSDRGPU_SINC_MIN_RATIO); the tests
 * restate the kernel's tiling and check its shared-memory and history bounds with it */
TSDRGPU_API uint32_t tsdrgpu_sinc_tile_pixels(double r);

/* ---------------------------------------------------------------------------- a7-a15  frame stage
 * replaces dsp_post_process + dsp_postprocess_t (dsp.c:112-239), dsp_autogain_run (:41-94),
 * dsp_timelowpass_run (:22-33), dsp_average_v_h (:96-110), syncdetector_run / findthesweetspot / findbestfit /
 * frameratepll state (syncdetector.c:26-226) and gaussianblur (gaussian.c:18-79), for a BATCH of consecutive
 * frames.  Pixel outputs and all integer sync results are bit-exact; `snr` (never announced by the reference,
 * dsp.c:234) is computed with parallel double sums, ~1e-12 relative.
 * The PLL's write-back to refreshrate (syncdetector.c:141-152) is the HOST's job: the per-frame results carry
 * vx / avg_speed / state so the caller applies it between batches (geometry is constant inside one batch).
 */
typedef struct tsdrgpu_framestage tsdrgpu_framestage_t;

typedef struct {
	int32_t x_dx, x_vx, x_absvx, x_stripsize;     /* sweetspot_data_t db_x (syncdetector.h:16-22) */
	int32_t y_dx, y_vx, y_absvx, y_stripsize;     /* db_y */
	double  avg_speed;                            /* syncdetector_t.avg_speed after this frame */
	int32_t pll_state;                            /* 1 = locked */
	float   lastmax, lastmin, snr;                /* dsp_autogain_t after this frame */
	int32_t autogain_report;                      /* 1 when dsp.c:231-235 would announce min/max */
	int32_t reserved;
} tsdrgpu_frame_result_t;

enum {                                            /* flags for tsdrgpu_framestage_run */
	TSDRGPU_FS_AUTOSHIFT            = 1,          /* PARAM_INT_AUTOSHIFT */
	TSDRGPU_FS_LOWPASS_BEFORE_SYNC  = 2,          /* PARAM_LOW_PASS_BEFORE_SYNC */
	TSDRGPU_FS_AUTOGAIN_AFTER_PROC  = 4,          /* PARAM_AUTOGAIN_AFTER_PROCESSING */
	TSDRGPU_FS_SUPERRESOLUTION      = 8,          /* PARAM_AUTOCORR_SUPERRESOLUTION (suppresses the green lines) */
	TSDRGPU_FS_COMPUTE_SNR          = 16          /* also fill .snr (costs one more reduction) */
};

TSDRGPU_API int  tsdrgpu_framestage_create(tsdrgpu_ctx_t *ctx, tsdrgpu_framestage_t **fs);
TSDRGPU_API void tsdrgpu_framestage_destroy(tsdrgpu_framestage_t *fs);
TSDRGPU_API int  tsdrgpu_framestage_reset(tsdrgpu_framestage_t *fs, void *stream);          /* dsp_post_process_init */
/* d_frames_in / d_frames_out: nframes * width * height floats, frames back to back (in != out).
 * h_results (nframes entries, may be NULL) is filled when the call returns: this call synchronises `stream`
 * only if h_results != NULL. */
TSDRGPU_API int  tsdrgpu_framestage_run(tsdrgpu_framestage_t *fs, void *stream, const float *d_frames_in, int nframes,
                                        int width, int height, float motionblur, float lowpasscoeff, unsigned flags,
                                        float *d_frames_out, tsdrgpu_frame_result_t *h_results);

/* same, but never synchronises: h_results_pinned (page-locked, nframes entries, may be NULL) is valid once the
 * stream has passed this call; h_autogain_report (nframes ints, may be NULL) is filled on return. */
TSDRGPU_API int  tsdrgpu_framestage_run_async(tsdrgpu_framestage_t *fs, void *stream, const float *d_frames_in, int nframes,
                                              int width, int height, float motionblur, float lowpasscoeff, unsigned flags,
                                              float *d_frames_out, tsdrgpu_frame_result_t *h_results_pinned,
                                              int32_t *h_autogain_report);

/* Overlap mode (off by default).  When on, and for the default stage order (LOWPASS_BEFORE_SYNC set,
 * AUTOGAIN_AFTER_PROC clear), the latency-bound sync search and the re-centring of batch k run on an internal side
 * stream while `stream` already works on batch k+1.  d_frames_out / h_results_pinned of a run are then valid only
 * after tsdrgpu_framestage_join(fs, s) has made stream `s` wait for the side stream (or after a device sync). */
TSDRGPU_API int  tsdrgpu_framestage_set_overlap(tsdrgpu_framestage_t *fs, int on);
TSDRGPU_API int  tsdrgpu_framestage_join(tsdrgpu_framestage_t *fs, void *stream);

/* ---------------------------------------------------------------------------- a8+  percentile auto-gain (beyond the reference)
 * The reference stretches every frame between its smallest and its largest pixel (dsp.c:50-61), so a single noise tail or
 * impulsive sample sets the span.  Clip mode takes the levels a fixed fraction of the pixels inside each end instead.
 *
 *   TSDRGPU_AG_MINMAX (default): the reference's min/max, unchanged.
 *   TSDRGPU_AG_CLIP, ppm in [0, 250000] (parts per million clipped at each end).  Per frame of n pixels:
 *     V    = the pixels v with !(v > 250 || v < -250) (not a marker, dsp.c:57) and v == v (not NaN); n_v = |V| (64-bit)
 *     order: IEEE total order of the bit patterns (key(v) = bits ^ 0xffffffff for negative sign, bits | 0x80000000 for
 *            positive sign, compared as unsigned 32-bit integers), so -0.0 < +0.0 and ties are plain duplicates
 *     if n_v == 0:  lo = hi = pixel 0 of the frame (the reference's seed, dsp.c:50-51)
 *     else:         k = floor(n_v * ppm / 1000000) in 64-bit integers; lo = the k-th smallest element of V (0-based),
 *                   hi = the (n_v - 1 - k)-th smallest
 *   lo and hi then take the places of the reference's min and max: the lastmax/lastmin IIR, span, the normalisation
 *   (markers pass through), the SNR and the auto-gain report (dsp.c:63-94, 231-235) are unchanged, for both stage orders.
 *   ppm = 0 gives min and max of V, which equal the reference's whenever pixel 0 is in V.
 * The mode is a property of the frame stage, kept across tsdrgpu_framestage_reset; switching it leaves lastmin/lastmax as
 * they are (the IIR carries on).  Out-of-range ppm or an unknown mode: TSDRGPU_EINVAL.
 * Selection is exact (integer histogram counts only): a radix select on the 32-bit keys in three digit rounds. */
#define TSDRGPU_AG_MAX_PPM 250000
enum { TSDRGPU_AG_MINMAX = 0, TSDRGPU_AG_CLIP = 1 };
TSDRGPU_API int  tsdrgpu_framestage_set_autogain(tsdrgpu_framestage_t *fs, int mode, int ppm);
/* host-only: a percentage as the host library's TSDR_AUTOGAIN=clip:<percent> and Python's "clip:<percent>" spell it -> ppm.
 * percent = one or more decimal digits, optionally '.' and one or more digits (nothing else: no sign, blank, exponent or
 * hex), with value in [0, 25]; ppm = floor(percent * 1e4 + 0.5), the product and the sum each one IEEE double rounding.
 * Returns -1 for anything else. */
TSDRGPU_API int  tsdrgpu_autogain_ppm(const char *percent);
/* stage level (synchronises): lo / hi / n_v above for nframes frames of n pixels each, back to back from d_frames (any 4-byte
 * alignment), n <= TSDRGPU_MAX_FRAME_PIXELS.  h_lo, h_hi (floats) and h_valid (uint64) hold nframes entries; h_valid may be NULL. */
#define TSDRGPU_MAX_FRAME_PIXELS (4000 * 4000)
TSDRGPU_API int  tsdrgpu_frame_levels(tsdrgpu_ctx_t *ctx, void *stream, const float *d_frames, uint64_t n, int nframes, int ppm,
                                      float *h_lo, float *h_hi, uint64_t *h_valid);

/* ---------------------------------------------------------------------------- a8+  contrast-limited adaptive histogram equalisation
 * (beyond the reference).  Every auto-gain is one global linear stretch per frame, which cannot lift faint detail in the dim
 * parts of a frame without saturating the bright ones.  CLAHE maps each pixel through the clipped, equalised histograms of the
 * tiles around it.  It is the last step of the frame stage: it runs on each frame as delivered (after the auto-gain, IIR,
 * re-centring or green lines and auto-gain after processing) and never feeds back: d_screen, lastmin/lastmax, the sync state
 * and every tsdrgpu_frame_result_t field are unchanged.  Per frame of W x H pixels, clip_centi in [100, 25600] (clip x 100),
 * tiles tx, ty in [1, 64]:
 *   1. valid pixel: !(v > 250 || v < -250) && v == v.  Markers, NaN and +-inf pass through unchanged and are counted nowhere.
 *   2. bin of a valid v: 0 if v <= 0, 255 if v >= 1, else (int)(v * 256.0f).
 *   3. tiles: TX = min(tx, W), TY = min(ty, H); column bounds x_j = floor(j W / TX), j = 0..TX, rows likewise; tile (i, j)
 *      holds n_t valid pixels with histogram h[256].
 *   4. clip and redistribute (OpenCV's integer scheme): L = max(1, floor(clip_centi n_t / 25600)) in 64-bit;
 *      excess = sum max(h_b - L, 0), then h_b = min(h_b, L); q, r = divmod(excess, 256), every h_b += q; if r > 0:
 *      step = max(256 / r, 1) and h[k step] += 1 for k = 0, 1, ... while k < r and k step < 256.  The total stays n_t.
 *   5. LUT: lut_b = (float) cdf_b / (float) n_t, cdf_b the inclusive prefix sum (one IEEE division, both operands exact);
 *      an empty tile has lut_b = (float) b / 255.0f.
 *   6. interpolation: s_j = x_j + x_{j+1}, c = 2x + 1.  If c <= s_0 or c >= s_{TX-1} the nearest edge tile is used alone
 *      (j0 = j1, wx = 0); otherwise j0 is the last j with s_j <= c, j1 = j0 + 1, wx = (float)(c - s_j0) / (float)(s_j1 - s_j0).
 *      Rows likewise give i0, i1, wy.  With L_ab the LUT of tile (i_a, j_b) at the pixel's bin:
 *      top = L00 + wx (L01 - L00), bot = L10 + wx (L11 - L10), out = top + wy (bot - top), each operation rounded to float32
 *      with no contraction.
 * Valid pixels come out in [0, 1], so tsdrgpu_pixels_argb and the ARGB pipeline output apply unchanged.
 * Integer histograms only: the result is deterministic. */
enum { TSDRGPU_CONTRAST_OFF = 0, TSDRGPU_CONTRAST_CLAHE = 1 };
#define TSDRGPU_CLAHE_MIN_CLIP 100
#define TSDRGPU_CLAHE_MAX_CLIP 25600
#define TSDRGPU_CLAHE_MAX_TILES 64
/* the frame stage's contrast mode, applied from the next run on and kept across tsdrgpu_framestage_reset.  With
 * TSDRGPU_CONTRAST_OFF (the default) the other arguments are ignored.  Out-of-range values or an unknown mode: TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_framestage_set_contrast(tsdrgpu_framestage_t *fs, int mode, int clip_centi, int tx, int ty);
/* host-only: the spelling shared by the host library's TSDR_CONTRAST and Python.  "off", "clahe:<clip>" or
 * "clahe:<clip>:<tx>x<ty>"; clip = one or more digits, optionally '.' and one or two digits, value in [1, 256], converted to
 * hundredths with integer arithmetic; tx, ty = digits in [1, 64], default 8x8.  Nothing else (no sign, blank or exponent).
 * TSDRGPU_OK with the four outputs set (zeros for "off"), else TSDRGPU_EINVAL and the outputs untouched. */
TSDRGPU_API int  tsdrgpu_contrast_parse(const char *spec, int *mode, int *clip_centi, int *tx, int *ty);
/* stage level (synchronises): CLAHE of nframes frames of w x h (w, h <= 8192, w h <= TSDRGPU_MAX_FRAME_PIXELS), back to back
 * from d_in to d_out, both 4-byte aligned; d_in == d_out works in place, otherwise the two must not overlap. */
TSDRGPU_API int  tsdrgpu_clahe(tsdrgpu_ctx_t *ctx, void *stream, const float *d_in, float *d_out, int w, int h, int nframes,
                               int clip_centi, int tx, int ty);

/* ---------------------------------------------------------------------------- a8+  non-local means denoising (beyond the reference)
 * The reference's only noise reduction is the temporal IIR, which smears anything that moves and does nothing for a picture
 * shown briefly.  Non-local means replaces each pixel by a weighted mean of the pixels in a search window around it; a
 * neighbour's weight falls with the distance between its patch and the centre pixel's patch, so flat areas are averaged hard
 * while edges and glyph strokes keep their shape.  It runs on each frame as delivered (after every branch's last step) and
 * before CLAHE, so CLAHE equalises the denoised frame, and never feeds back: d_screen, lastmin/lastmax, the sync state and
 * every tsdrgpu_frame_result_t field are unchanged.  Per frame of W x H pixels, h_milli in [1, 1000] (h = h_milli / 1000 in
 * the units of the normalised frame), search radius R in [1, 10], patch radius P in [1, 3]:
 *   1. valid pixel: !(v > 250 || v < -250) && v == v.  Markers, NaN and +-inf pass through unchanged.
 *   2. guide: g = valid ? min(max(v, 0), 1) : 0; g_c(y, x) is g at the coordinates clamped into the frame.  Every patch
 *      lookup goes through g_c, so a patch is defined at every pixel, the frame edges included.
 *   3. patch distance for offset (dy, dx): e(y, x) = (g_c(y, x) - g_c(y + dy, x + dx))^2 (one subtraction, one
 *      multiplication); s(y, x) = ((e(y, x-P) + e(y, x-P+1)) + ...) + e(y, x+P), left to right;
 *      d = ((s(y-P, x) + s(y-P+1, x)) + ...) + s(y+P, x), top to bottom.  Every operation is rounded to float32 (no
 *      sliding-window sums, which round differently).
 *   4. weight: inv = (float) (1e6 / (4.0 h_milli^2 (2P+1)^2)), computed once in double and rounded once;
 *      t = min(d inv, 1), u = 1 - t, w = u u (a compact bisquare kernel: 1 at d = 0, no exp, no table).
 *   5. accumulation: offsets in raster order, dy from -R to R outer, dx from -R to R inner, the centre offset included as an
 *      ordinary offset (it gets w = 1).  Neighbour (y+dy, x+dx) contributes only when it lies inside the frame (no clamping
 *      here) and is valid: acc_w = acc_w + w, acc_v = acc_v + (w v_n), each product and sum rounded, no contraction, both
 *      accumulators starting at +0.  The output is acc_v / acc_w (one IEEE division; acc_w >= 1 because of the centre).
 * The output of a valid pixel is a convex combination of valid pixels of its window, so it stays within their range and
 * tsdrgpu_pixels_argb and the ARGB pipeline output apply unchanged.  A valid -0.0 whose neighbours all get weight 0 comes
 * out as +0.0. */
enum { TSDRGPU_DENOISE_OFF = 0, TSDRGPU_DENOISE_NLM = 1 };
#define TSDRGPU_NLM_MAX_H 1000
#define TSDRGPU_NLM_MAX_R 10
#define TSDRGPU_NLM_MAX_P 3
/* the frame stage's denoise mode, applied from the next run on and kept across tsdrgpu_framestage_reset.  With
 * TSDRGPU_DENOISE_OFF (the default) the other arguments are ignored.  Out-of-range values or an unknown mode: TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_framestage_set_denoise(tsdrgpu_framestage_t *fs, int mode, int h_milli, int r, int p);
/* host-only: the spelling shared by the host library's TSDR_DENOISE and Python.  "off", "nlm:<h>" or "nlm:<h>:<R>:<P>";
 * h = one or more digits, optionally '.' and one to three digits, value in [0.001, 1], converted to thousandths with integer
 * arithmetic; R, P = digits in [1, 10] and [1, 3], default 5 and 1.  Nothing else (no sign, blank or exponent).
 * TSDRGPU_OK with the four outputs set (zeros for "off"), else TSDRGPU_EINVAL and the outputs untouched. */
TSDRGPU_API int  tsdrgpu_denoise_parse(const char *spec, int *mode, int *h_milli, int *r, int *p);
/* stage level (synchronises): non-local means of nframes frames of w x h (w h <= TSDRGPU_MAX_FRAME_PIXELS), back to back
 * from d_in to d_out, both 4-byte aligned.  It cannot run in place: overlapping buffers are refused with TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_nlm(tsdrgpu_ctx_t *ctx, void *stream, const float *d_in, float *d_out, int w, int h, int nframes,
                             int h_milli, int r, int p);

/* ---------------------------------------------------------------------------- a8+  Richardson-Lucy deconvolution along the lines (beyond the reference)
 * Every geometry decodes at about two pixels per IQ sample (W = (int)(2 fs / (fv h))), and the front end has already averaged the
 * signal over the sample period, so a one-pixel stroke comes out as a bump about three pixels wide.  On one frame that is aliasing
 * as well as blur, but an average of frames whose sampling phase drifts (the stack, or motion blur > 0) is the picture convolved
 * with a fixed line-spread function, which deconvolution can undo.  It runs on each frame as delivered, after the stack and before
 * NLM and CLAHE (stack -> deblur -> NLM -> CLAHE; RL assumes a linear blur, which NLM's weights are not), and never feeds back:
 * d_screen, lastmin/lastmax, the sync state and every tsdrgpu_frame_result_t field are unchanged.
 * Each line y of a frame is processed on its own (lines are separate in time; after the re-centring the blanking sits at the line
 * ends, so there is no vertical blur to undo).  sigma = sigma_centi / 100 in [0.25, 4] pixels, iterations I in [1, 64]:
 *   1. taps: R = ceil(3 sigma) = (3 sigma_centi + 99) / 100 in integers; k_j = exp(-j^2 / (2 sigma^2)) / sum, j in [-R, R], the sum
 *      over the same j, all in double, each tap rounded once to float (tsdrgpu_deblur_taps).
 *   2. inputs: valid(v) is !(v > 250 || v < -250) && v == v; m(x) = valid as 0 / 1, and a position outside the line counts as
 *      invalid, so line ends and markers follow one rule.  d(x) = m ? (v > 0 ? min(v, 1) : 0) : 0 (the clamp to [0, 1], with -0
 *      taken to +0).
 *   3. masked correlation: B(a)(x) = sum_j k_j (m(x+j) a(x+j)), j from -R to R, left to right, each product and sum rounded to
 *      float32.  rn(x) = 1.0f / B(1)(x), one IEEE division, once per line, where m = 1 (there B(1) >= k_0 > 0).
 *   4. iterations: u_0 = d; each iteration, per pixel: b = B(u) rn; q = m ? d / max(b, eps) : 0; u <- m ? u (B(q) rn) : 0, with
 *      eps = TSDRGPU_DEBLUR_EPS (2^-30), every operation rounded to float32, no contraction, IEEE division.
 *   5. output: out = valid(v) ? min(u_I, 1.0f) : v.  Markers, NaN and +-inf pass through in place; valid outputs lie in [0, 1],
 *      so NLM, CLAHE, tsdrgpu_pixels_argb and the ARGB pipeline output apply unchanged.
 * A valid pixel further than 2 R I pixels from every invalid pixel and line end is unaffected by them.
 * Guidance: sigma near 1 fits the box resampler (its ratio r = pixelrate / fs is within 0.2 % of 2, and the two r-pixel boxes of
 * integration and hold give r / sqrt(6) = 0.82, to which the front end's own roll-off adds); the sinc resampler wants less.  The
 * step is meant for averaged frames (the stack, or motion blur > 0): on a single noisy frame it amplifies noise and aliasing. */
enum { TSDRGPU_DEBLUR_OFF = 0, TSDRGPU_DEBLUR_RL = 1 };
#define TSDRGPU_DEBLUR_MIN_SIGMA 25           /* sigma_centi */
#define TSDRGPU_DEBLUR_MAX_SIGMA 400
#define TSDRGPU_DEBLUR_MAX_ITER  64
#define TSDRGPU_DEBLUR_MAX_R     12           /* ceil(3 * 4) */
#define TSDRGPU_DEBLUR_EPS       0x1p-30f
/* host-only: the taps of step 1.  *R (may be NULL) receives R; taps (may be NULL) receives the 2R + 1 taps k_{-R} .. k_R.
 * TSDRGPU_EINVAL for sigma_centi outside [25, 400]. */
TSDRGPU_API int  tsdrgpu_deblur_taps(int sigma_centi, float *taps, int *R);
/* the frame stage's deblur mode, applied from the next run on and kept across tsdrgpu_framestage_reset.  With
 * TSDRGPU_DEBLUR_OFF (the default) the other arguments are ignored.  Out-of-range values or an unknown mode: TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_framestage_set_deblur(tsdrgpu_framestage_t *fs, int mode, int sigma_centi, int iterations);
/* host-only: the spelling shared by the host library's TSDR_DEBLUR and Python.  "off", "rl:<sigma>" or "rl:<sigma>:<I>";
 * sigma = one to six digits, optionally '.' and one or two digits, value in [0.25, 4], converted to hundredths with integer
 * arithmetic; I = one to six digits in [1, 64], default 20.  Nothing else (no sign, blank or exponent).
 * TSDRGPU_OK with the three outputs set (zeros for "off"), else TSDRGPU_EINVAL and the outputs untouched. */
TSDRGPU_API int  tsdrgpu_deblur_parse(const char *spec, int *mode, int *sigma_centi, int *iterations);
/* stage level (synchronises): deblur of nframes frames of w x h (w h <= TSDRGPU_MAX_FRAME_PIXELS) back to back from d_in to
 * d_out, both 4-byte aligned.  It cannot run in place: overlapping buffers are refused with TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_deblur(tsdrgpu_ctx_t *ctx, void *stream, const float *d_in, float *d_out, int w, int h, int nframes,
                                int sigma_centi, int iterations);

/* ---------------------------------------------------------------------------- a8+  drift-registered frame averaging (beyond the reference)
 * Averaging many frames is how faint text is read, but the reference's temporal IIR (motionblur, dsp.c:22-33) averages in raster
 * coordinates before the sync search re-centres the frame, so any drift of the picture between frames is averaged in as smear.
 * Stacking finds where each frame sits relative to a running average, to a fraction of a pixel, resamples the frame into the
 * average's coordinates, blends it in and delivers the average moved to where the current frame is.  It runs on each frame as
 * delivered (after every branch's last step), before NLM and CLAHE, and never feeds back: d_screen, lastmin/lastmax, the sync
 * state and every tsdrgpu_frame_result_t field are unchanged, so the PLL keeps seeing the drift it corrects.
 * Depth N in [2, 1024], search radius rx in [1, 32] pixels along a line (default 8) and ry in [0, 8] whole lines (default 2).
 * Motion model: drift is a circular shift of the flattened W x H raster (n = W H pixels) by a real number of pixels; a whole-line
 * jump is a shift by a multiple of W.  Indices below are taken mod n; valid(v) is !(v > 250 || v < -250) && v == v.
 * State: accumulator A (n floats), m = frames taken since the last restart, the last two offsets o1, o2 (double, unwrapped);
 * R(x) = floor(x + 0.5) in double.  Per frame F:
 *   1. quantise: Q(v) = (int)(min(max(v, 0), 1) * 255.0f + 0.5f) in float32; qF[p] = valid(F[p]) ? Q(F[p]) : 0, qA[q] = Q(A[q]).
 *   2. restart frame (m == 0): A[p] = valid(F[p]) ? F[p] : 0, o = 0, m = 1; the output is F bit for bit.
 *   3. search: b = R(o1) + (m >= 2 ? R(o1) - R(o2) : 0) (constant velocity); candidates s = b + dy W + dx, dy from -ry to ry
 *      (outer), dx from -rx to rx (inner); score S(s) = sum_q qF[q + s] qA[q] in 64-bit integers (exact, order-free); s* is the
 *      largest S, the first in loop order on a tie.
 *   4. sub-pixel fit, only when -rx < dx* < rx: a = S(s* - 1), c = S(s* + 1), M = S(s*) as doubles, den = (a - 2M) + c;
 *      delta = den < 0 ? clamp((a - c) / (2 den), -0.5, 0.5) : 0.  o = s* + delta.
 *   5. warp: I = floor(o), t = (float)(o - I); Catmull-Rom weights in float32, no contraction:
 *      wm1 = ((-0.5t + 1)t - 0.5)t, w0 = ((1.5t - 2.5)t)t + 1, w1 = ((-1.5t + 2)t + 0.5)t, w2 = ((0.5t - 0.5)t)t;
 *      x[q] = ((wm1 F[q+I-1] + w0 F[q+I]) + w1 F[q+I+1]) + w2 F[q+I+2].
 *   6. blend, only where all four taps are valid (elsewhere A[q] keeps its value): k = min(m + 1, N), wn = (float)(1.0 / k),
 *      wo = (float)(1.0 - 1.0 / k); A[q] = A[q] wo + x[q] wn in float32, no contraction.  Then m += 1.  The first frames form a
 *      true running mean; from then on this is an exponential average with time constant N.
 *   7. output: out[p] = valid(F[p]) ? A[p - R(o)] : F[p] (markers, NaN and +-inf pass through in place).  Then o2 = o1, o1 = o.
 * Every frame yields a tsdrgpu_stack_record_t.  Restarts (m = 0) happen at create, at reset, when W or H changes and when a set
 * changes the mode, N, rx or ry.  The definition is frame-sequential: any cut of a frame sequence into batches gives the same bits. */
/* The change-adaptive mode (TSDRGPU_STACK_ADAPT, "adapt:<N>[:<rx>x<ry>]", the same ranges and defaults) restarts the average
 * tile by tile where the picture changes, so a typed word or a new dialog is not buried under a fading ghost of the old content
 * for N frames.  Steps 1-5 and 7 are align's, unchanged (step 3's m >= 2 is still the global m); step 6 becomes:
 *   tiles: the accumulator's raster in fixed tiles of TSDRGPU_STACK_TILE x TSDRGPU_STACK_TILE pixels, pixel q in tile
 *      ((q mod W) div 16, (q div W) div 16); the last column and row of tiles may be partial.  Per tile t: a count m_t and a
 *      residual level e_t (unsigned, mean square in 8-bit levels with 4 fraction bits, or "none").  A restart frame sets every
 *      m_t = 1 and e_t = none; every restart of align (create, reset, W or H, set) restarts these too.
 *   6a. statistic, over the pixels q of tile t whose four taps are valid: d = Q(x[q]) - Q(A[q]) (A before this frame's blend;
 *      Q of any finite x clamps as in step 1), D_t = sum d^2 and C_t = their count, in exact integers.
 *   6b. decision: changed_t = C_t > 0 && e_t != none && 16 D_t > RATIO e_t C_t && D_t > FLOOR C_t (exact 64-bit integers), with
 *      RATIO = TSDRGPU_STACK_ADAPT_RATIO and FLOOR = TSDRGPU_STACK_ADAPT_FLOOR.  Tile t restarts when changed_t holds for t or
 *      one of its 8 neighbours (not wrapping at the edges), so an edge that falls across a tile border is caught on both sides.
 *   6c. state: a restarting tile takes m_t = 0 and e_t = none; any other tile with C_t > 0 takes r = floor(16 D_t / C_t) and
 *      e_t = (e_t == none ? r : floor((7 e_t + r) / 8)).
 *   6d. blend, only where all four taps are valid: k_t = min(m_t + 1, N), wn and wo from k_t as in align, A[q] = A[q] wo + x[q] wn
 *      with the weights of q's tile.  Then m_t = min(m_t + 1, N) for every tile, and m += 1 as in align.
 * Each tile is measured against its own running level, not the frame's: tiles holding one-pixel strokes carry a warp residual
 * that flat tiles do not, and a frame-wide normaliser either restarts them on static frames or misses changes under heavy
 * noise.  A restarted tile starts a new level with its new content, so it does not restart again on its own fresh average.
 * RATIO = 3 and FLOOR = 64 (an rms residual of 8 levels, which keeps noise-free tiles with e_t near 0 from restarting) are fixed;
 * DESIGN.md section 5.5 gives the quality they were chosen for.  When no tile restarts, every m_t follows the global m's
 * sequence capped at N, so the output and records equal align's bit for bit; the record's `changed` counts the tiles restarted
 * in that frame (always 0 for align and on restart frames). */
/* The motion-tracking mode (TSDRGPU_STACK_TRACK, "track:<N>[:<rx>x<ry>]", the same ranges and defaults) carries the average
 * tile by tile with content that moves inside the picture: a terminal that scrolls, a page scrolled in a browser, a window being
 * dragged.  To adapt, every tile such motion crosses has changed, so the average restarts there at every move.  Here a changed
 * tile first looks in the old average for where its content came from and, when it finds it, takes its average and counts
 * from there; only what is newly exposed starts again.  Steps 1-5 and 7 are align's and 6a is adapt's, unchanged: D_t(0) = D_t,
 * C_t(0) = C_t and changed_t against the tile's level e_t.  The counts are per pixel: c[p] <= N (16 bits), and A and c are
 * double-buffered, since a moving tile gathers from other tiles' old values.  Pixel p = (X, Y), X = p mod W, Y = p div W.
 *   6t. local search, only for tiles with changed_t (the tile's own flag, before the neighbour rule): for every integer
 *      v = (vx, vy) != (0, 0) with |vx| <= LX = TSDRGPU_STACK_TRACK_LX and |vy| <= LY = TSDRGPU_STACK_TRACK_LY, over the tile's
 *      pixels p whose four taps are valid and whose source s = (X - vx, Y - vy) lies inside the W x H raster (no wrap):
 *      d = Q(x[p]) - Q(A[s]), D_t(v) = sum d^2 and C_t(v) = their count, exact integers.  v is admissible when C_t(v) > 0 and
 *      2 C_t(v) >= C_t(0).  v* is the admissible v with the least D/C, compared as D(v) C(v') against D(v') C(v) exactly in
 *      64 bits; ties go to the smaller |vx| + |vy|, then to the first in loop order (vy outer, vx inner, both ascending).
 *      moved_t holds when v* exists and passes 6b's change test at the tile's own level: not (16 D(v*) > RATIO e_t C(v*) and
 *      D(v*) > FLOOR C(v*)).
 *   6b. a tile restarts when changed_t && !moved_t holds for it or one of its 8 neighbours (no wrap); a moved tile that a
 *      neighbour restarts does restart; moved tiles do not spread restarts.
 *   6c. a restarting tile takes e_t = none; a moved tile that does not restart takes r* = floor(16 D(v*) / C(v*)) and
 *      e_t = floor((7 e_t + r*) / 8); every other tile follows adapt's 6c.
 *   6d. blend into the second accumulator A' and counts c': the source is s = p - v* in a moved tile that does not restart and
 *      s = p elsewhere; in a restarting tile, and for a pixel of a moved tile whose s falls outside the raster, s = p and c[s]
 *      counts as 0.  k = min(c[s] + 1, N), with wn and wo from k as in align; A'[p] = A[s] wo + x[p] wn where all four taps
 *      are valid, A'[p] = A[s] elsewhere; c'[p] = k in every case.  Then A' and c' are the state, and m += 1 as in align.
 *   A restart frame sets every c = 1 and e_t = none; every restart of align restarts the counts, the levels and both planes.
 * The record's `changed` counts the tiles restarted in the frame, as in adapt; tsdrgpu_stack_vectors reads where each tile
 * moved.  LX and LY are fixed: 32 lines cover a one-line scroll of any usual font.  When no tile moves in a sequence, a tile's
 * pixels share one count equal to adapt's m_t, so every output and record equals adapt's bit for bit. */
/* The glitch-tolerant mode (TSDRGPU_STACK_ROBUST, "robust:<N>[:<rx>x<ry>]", the same ranges and defaults) is track with three
 * additions that keep a disturbance lasting one frame out of the average: a frame torn around dropped samples, a re-centring step
 * or a PLL correction that moves one frame against the next, impulsive interference over a few lines.  In adapt and track every
 * tile such a frame touches restarts with that one noisy frame as its content, and the average takes N frames to rebuild.  Here
 * a change must last two frames before a tile restarts.  Steps 1-5 and 7, 6a, 6t, the move test, and 6c for tiles that blend are
 * track's, unchanged, and so are the per-pixel counts, except that bit 15 of c[p] holds a flag g[p] and the count is c[p] & 0x7fff
 * (still <= N).  Per tile one more bit, pend_t; a restart frame, and so every restart of align, sets every pend_t = 0 and g = 0.
 *   6r. debounce: new_t = changed_t && !moved_t (the tile's own flag of track's 6b), confirmed_t = new_t && pend_t.  A tile
 *      restarts when confirmed_t holds for it or one of its 8 neighbours (no wrap); a moved tile that a neighbour restarts does
 *      restart.  A tile is held when new_t && !pend_t and no neighbour restarts it.
 *   6h. frame hold: with `held` the number of held tiles, the frame is a glitch frame when 2 held > ntiles.  Then o = b (step 3's
 *      prediction) replaces the found offset in step 7 and in the history (o2 = o1, o1 = b); no tile blends, moves or restarts;
 *      A, c and every e_t stay as they were.  The record reports offset = b, score, dx and dy as found, and changed = 0.
 *   6c. a held tile keeps e_t; a restarting tile takes e_t = none; every other tile follows track's 6c.
 *   6d. a held tile keeps A and c (g included).  Every other tile blends as in track with k = min((c[s] & 0x7fff) + 1, N), except
 *      that the gate applies in a tile that neither restarts nor is held and whose level before this frame's 6c is e_t != none:
 *      for a pixel p whose four taps are valid and whose source s lies inside the raster, d = Q(x[p]) - Q(A[s]), and p is gated
 *      when d^2 > max(e_t, GATE_MIN) (more than 4 rms of the tile's residual and more than 32 levels; GATE_MIN =
 *      TSDRGPU_STACK_ROBUST_GATE_MIN = 16 FLOOR).  A gated p with g[s] = 0 keeps A'[p] = A[s] and c'[p] = (c[s] & 0x7fff) | 0x8000;
 *      a gated p with g[s] = 1 restarts, A'[p] = x[p] and c'[p] = 1.  Every pixel not gated takes track's 6d with g cleared.
 *   After every frame, glitch frames included, pend_t = new_t for every tile.
 * A region that keeps changing restarts every third frame (restart, fresh level, held, restart), where adapt and track restart
 * it every second frame: the frame after a restart measures against e_t = none, so it is never new.  A lasting change is taken
 * one frame later than in track, and a lone bad frame never reaches the average.  The constants are fixed.  When no tile is
 * held and no pixel gated over a sequence, no tile is ever new (the first would have been held), so every output and record
 * equals track's bit for bit.  tsdrgpu_stack_robust_counts reads the last frame's held tiles, gated pixels and hold. */
/* the stack's modes; any other value, 2, 3 and 5 included, is refused with TSDRGPU_EINVAL */
enum { TSDRGPU_STACK_OFF = 0, TSDRGPU_STACK_ALIGN = 1, TSDRGPU_STACK_ADAPT = 4, TSDRGPU_STACK_TRACK = 8, TSDRGPU_STACK_ROBUST = 16 };
#define TSDRGPU_STACK_MIN_N  2
#define TSDRGPU_STACK_MAX_N  1024
#define TSDRGPU_STACK_MAX_RX 32
#define TSDRGPU_STACK_MAX_RY 8
#define TSDRGPU_STACK_TILE   16
#define TSDRGPU_STACK_ADAPT_RATIO 3
#define TSDRGPU_STACK_ADAPT_FLOOR 64
#define TSDRGPU_STACK_TRACK_LX 16
#define TSDRGPU_STACK_TRACK_LY 32
#define TSDRGPU_STACK_ROBUST_GATE_MIN (16 * TSDRGPU_STACK_ADAPT_FLOOR)
typedef struct {
	double  offset;                               /* o (unwrapped; 0 on a restart frame) */
	int64_t score;                                /* S(s*) (0 on a restart frame) */
	int32_t dx, dy;                               /* the best candidate's place in the window */
	int32_t restarted;                            /* 1 on a restart frame */
	int32_t changed;                              /* adapt, track, robust: the tiles restarted in this frame (0 for align) */
} tsdrgpu_stack_record_t;
/* host-only: the spelling shared by the host library's TSDR_STACK and Python.  "off", "align:<N>", "align:<N>:<rx>x<ry>", and
 * the same with "adapt:", "track:" or "robust:"; N, rx, ry = one to six digits in the ranges above, rx and ry defaulting to 8, 2.
 * Nothing else (no sign, blank or point).  TSDRGPU_OK with the four outputs set (zeros for "off"), else TSDRGPU_EINVAL and the
 * outputs untouched. */
TSDRGPU_API int  tsdrgpu_stack_parse(const char *spec, int *mode, int *depth, int *rx, int *ry);
/* stage level: one stack's state on the device.  run takes nframes frames of w x h (w h <= TSDRGPU_MAX_FRAME_PIXELS) back to back
 * from d_in to d_out (4-byte aligned, not overlapping), never synchronises, and fills h_records_pinned (page-locked, nframes
 * entries, may be NULL) once the stream has passed the call.  With TSDRGPU_STACK_OFF a run copies d_in to d_out. */
typedef struct tsdrgpu_stack tsdrgpu_stack_t;
TSDRGPU_API int  tsdrgpu_stack_create(tsdrgpu_ctx_t *ctx, tsdrgpu_stack_t **st);
TSDRGPU_API void tsdrgpu_stack_destroy(tsdrgpu_stack_t *st);
TSDRGPU_API int  tsdrgpu_stack_reset(tsdrgpu_stack_t *st);
TSDRGPU_API int  tsdrgpu_stack_set(tsdrgpu_stack_t *st, int mode, int depth, int rx, int ry);
TSDRGPU_API int  tsdrgpu_stack_run(tsdrgpu_stack_t *st, void *stream, const float *d_in, float *d_out, int w, int h, int nframes,
                                   tsdrgpu_stack_record_t *h_records_pinned);
/* track and robust modes (synchronises): where each tile of the last frame moved.  h_v receives 2 ntiles values, (vx, vy) of
 * tile t at h_v[2t], h_v[2t + 1] with t = (Y div 16) ceil(W / 16) + X div 16: v* for a tile that moved and did not restart (nor,
 * in robust mode, was held), (0, 0) (never a candidate) for every other tile, on a restart frame and on a glitch frame.
 * TSDRGPU_EINVAL unless the mode is track or robust, a frame has been taken since the last restart and ntiles is the tile count
 * of its geometry. */
TSDRGPU_API int  tsdrgpu_stack_vectors(tsdrgpu_stack_t *st, int32_t *h_v, int ntiles);
/* robust mode (synchronises): the last frame's held tiles (6r), gated pixels (6d) and whether it was a glitch frame (6h, 0 or
 * 1); all three 0 on a restart frame.  TSDRGPU_EINVAL unless the mode is robust and a frame has been taken since the last
 * restart. */
TSDRGPU_API int  tsdrgpu_stack_robust_counts(tsdrgpu_stack_t *st, int32_t *held_tiles, uint64_t *gated_pixels, int32_t *frame_held);
/* the frame stage's stack mode, applied from the next run on.  The mode is kept across tsdrgpu_framestage_reset; the accumulator
 * is not (the reset restarts it).  Out-of-range values or an unknown mode: TSDRGPU_EINVAL. */
TSDRGPU_API int  tsdrgpu_framestage_set_stack(tsdrgpu_framestage_t *fs, int mode, int depth, int rx, int ry);
/* the records of the frame stage's last run with the stack on (nframes <= that run's frames); synchronises the device */
TSDRGPU_API int  tsdrgpu_framestage_stack_records(tsdrgpu_framestage_t *fs, tsdrgpu_stack_record_t *h_records, int nframes);

/* stage-level entry points (same arithmetic as the kernels inside tsdrgpu_framestage_run) */
TSDRGPU_API int tsdrgpu_autogain(tsdrgpu_ctx_t *ctx, void *stream, float *h_lastmax, float *h_lastmin, float *h_snr,
                                 int n, const float *d_in, float *d_out, float norm);        /* synchronises */
TSDRGPU_API int tsdrgpu_timelowpass(tsdrgpu_ctx_t *ctx, void *stream, float coeff, int n, const float *d_in, float *d_screen);
TSDRGPU_API int tsdrgpu_average_v_h(tsdrgpu_ctx_t *ctx, void *stream, int width, int height, const float *d_in,
                                    float *d_wbuf, float *d_hbuf);
TSDRGPU_API int tsdrgpu_gaussianblur(tsdrgpu_ctx_t *ctx, void *stream, float *d_data, int n);

/* ---------------------------------------------------------------------------- a16 host pixel rule (next-row item)
 * the JNI glue's float->ARGB mapping (JavaGUI/jni/TSDRLibraryNDK.c:222-283), bit-exact; transparent (2048.0f)
 * pixels keep the previous content of d_argb. */
TSDRGPU_API int tsdrgpu_pixels_argb(tsdrgpu_ctx_t *ctx, void *stream, const float *d_frame, int n, int inverted, int32_t *d_argb);
/* a batch of frames converted IN PLACE (float frame f becomes its n int32 pixels); d_last (n int32, caller-zeroed at start)
 * is the host's persistent pixel buffer carried across frames and calls, so transparent samples behave as in the GUI */
TSDRGPU_API int tsdrgpu_pixels_argb_batch(tsdrgpu_ctx_t *ctx, void *stream, float *d_frames_inout, uint64_t n, int nframes, int inverted, int32_t *d_last);

/* ---------------------------------------------------------------------------- a19/a20  FFT and correlations
 * replace fft_perform, fft_autocorrelation, fft_crosscorrelation (fft.c:49-176).  Same definitions as the
 * reference (forward divides by N, inverse does not; N = largest power of two <= size; "autocorrelation" is
 * IFFT(|FFT(x)|/N)), computed by a float32 Stockham FFT with double-derived twiddles: results agree with the
 * reference's float-storage/double-arithmetic radix-2 code to ~1e-6 of the spectrum's peak (tolerance-based).
 */
TSDRGPU_API uint32_t tsdrgpu_fft_getrealsize(uint32_t size);                                   /* fft.c:5-11 */
TSDRGPU_API int tsdrgpu_fft(tsdrgpu_ctx_t *ctx, void *stream, float *d_iq, uint32_t size, int inverse);   /* in place */
TSDRGPU_API int tsdrgpu_autocorrelation(tsdrgpu_ctx_t *ctx, void *stream, float *d_answer, const float *d_real, uint32_t size);
/* `batch` independent autocorrelations in one set of launches: input b at d_reals + b*real_stride (floats), output b at
 * d_answers + b*2*size (floats).  size must be even. */
TSDRGPU_API int tsdrgpu_autocorrelation_batch(tsdrgpu_ctx_t *ctx, void *stream, float *d_answers, const float *d_reals, uint32_t size,
                                              uint32_t batch, uint64_t real_stride);
TSDRGPU_API int tsdrgpu_crosscorrelation(tsdrgpu_ctx_t *ctx, void *stream, float *d_a_out, float *d_b_tmp, uint32_t samples);

/* ---------------------------------------------------------------------------- a17/a18  frame-rate detector
 * replaces frameratedetector_runontodata / accummulate (frameratedetector.c:34-126) and the two extbuffer
 * running means: one capture in, the two lag-window plots out. */
typedef struct tsdrgpu_frd tsdrgpu_frd_t;
TSDRGPU_API int  tsdrgpu_frd_create(tsdrgpu_ctx_t *ctx, tsdrgpu_frd_t **frd);
TSDRGPU_API void tsdrgpu_frd_destroy(tsdrgpu_frd_t *frd);
/* Overlapped mode: a run's kernels go to an internal stream (behind what `stream` held at the call) with work buffers of the
 * detector's own, so the transforms share the chip with what the caller enqueues next; the capture must stay untouched until
 * tsdrgpu_frd_join(frd, s) has put stream s behind the run (plots / peaks readers join by themselves). */
TSDRGPU_API int  tsdrgpu_frd_set_overlap(tsdrgpu_frd_t *frd, int on);
TSDRGPU_API int  tsdrgpu_frd_join(tsdrgpu_frd_t *frd, void *stream);
TSDRGPU_API int  tsdrgpu_frd_reset(tsdrgpu_frd_t *frd);                      /* extbuffer_cleartozero on all three */
TSDRGPU_API uint32_t tsdrgpu_frd_capture_size(uint32_t samplerate);          /* frameratedetector.c:160 */
TSDRGPU_API void tsdrgpu_frd_windows(uint32_t samplerate, int *frame_min, int *frame_max, int *line_min, int *line_max);
/* d_capture: `size` demodulated samples.  The running means stay on the device; pass h_* (may be NULL) to copy
 * them out (then the call synchronises).  *calls = captures accumulated so far. */
TSDRGPU_API int  tsdrgpu_frd_run(tsdrgpu_frd_t *frd, void *stream, uint32_t samplerate, const float *d_capture, uint32_t size,
                                 double *h_frame_plot, int frame_cap, double *h_line_plot, int line_cap, uint64_t *calls);
/* same without the final synchronisation; the h_* buffers must be page-locked */
TSDRGPU_API int  tsdrgpu_frd_run_async(tsdrgpu_frd_t *frd, void *stream, uint32_t samplerate, const float *d_capture, uint32_t size,
                                       double *h_frame_plot_pinned, int frame_cap, double *h_line_plot_pinned, int line_cap, uint64_t *calls);
/* `batch` consecutive captures (capture b at d_captures + b*capture_stride floats) accumulated in order, as if
 * tsdrgpu_frd_run had been called batch times; asynchronous, plots stay on the device. */
TSDRGPU_API int  tsdrgpu_frd_run_batch(tsdrgpu_frd_t *frd, void *stream, uint32_t samplerate, const float *d_captures, uint32_t size,
                                       uint32_t batch, uint64_t capture_stride, uint64_t *calls);
/* copies the current running means (device-resident) to host buffers; synchronises */
/* dump_autocorrect (frameratedetector.c:64-85): CSV of (lag in ms, 10 log10 |r|) of one capture's autocorrelation; synchronises */
TSDRGPU_API int  tsdrgpu_frd_dump_csv(tsdrgpu_frd_t *frd, void *stream, uint32_t samplerate, const float *d_capture, uint32_t size, const char *path);
TSDRGPU_API int  tsdrgpu_frd_get_plots(tsdrgpu_frd_t *frd, void *stream, uint32_t samplerate, double *h_frame_plot, int frame_cap,
                                       double *h_line_plot, int line_cap);
/* SURVEY 8f-3 on the device: index of the first strict maximum of each plot (PlotVisualizer.java:203-236), reduced on the GPU
 * right behind the running means of every run.  h_peaks[0] = frame plot, [1] = line plot.  _async: page-locked destination. */
TSDRGPU_API int  tsdrgpu_frd_peaks(tsdrgpu_frd_t *frd, void *stream, int32_t *h_peaks);                  /* synchronises */
TSDRGPU_API int  tsdrgpu_plot_peaks(tsdrgpu_ctx_t *ctx, void *stream, const double *d_frame_plot, int frame_len, const double *d_line_plot, int line_len,
                                    int32_t *h_peaks);                                                     /* synchronises */
TSDRGPU_API int  tsdrgpu_frd_peaks_async(tsdrgpu_frd_t *frd, void *stream, int32_t *h_peaks_pinned);
TSDRGPU_API int  tsdrgpu_accumulate(tsdrgpu_ctx_t *ctx, void *stream, double *d_out, uint64_t calls,
                                    const float *d_in_complex, int startid, int length);

/* ---------------------------------------------------------------------------- a22  superbandwidth
 * replace complex_to_abs_diff, superb_bestfit, superb_ondataready (superbandwidth.c:67-152). */
TSDRGPU_API int tsdrgpu_complex_to_abs_diff(tsdrgpu_ctx_t *ctx, void *stream, float *d_data, int size_floats);
/* alignment lag in floats (2 * argmax over the first half of |xcorr|), exact integer.  synchronises */
TSDRGPU_API int tsdrgpu_superb_bestfit(tsdrgpu_ctx_t *ctx, void *stream, const float *d_hop0, const float *d_hopi,
                                       int size_floats, int samples_in_frame, int *h_best_offset);
/* single-GPU stitch of nhops hops (each count_pairs IQ pairs, d_hops[i] device pointers in a HOST array);
 * d_out holds nhops * N * 2 floats, N = fft_getrealsize(count_pairs).  synchronises (lags are read back). */
TSDRGPU_API int tsdrgpu_superb_stitch(tsdrgpu_ctx_t *ctx, void *stream, float *const *d_hops, int nhops, int count_pairs,
                                      int samples_in_frame, float *d_out, int *h_best_offsets, int *h_total_samples);
/* multi-GPU building blocks: round 1's one-all-gather formulation (one hop per rank, DESIGN.md section 6), kept as
 * bench.py's NCCL all-gather baseline for the sharded stitch below.  Every rank sends [FFT_N(raw hop) | FFT_nd(first
 * difference of |hop|)] (n + nd complex, returned in *h_n / *h_nd), the caller runs one all-gather, then every rank
 * derives the integer alignment lags itself (tsdrgpu_superb_lags, exact) and produces its strided residue s of the
 * H*N-point inverse (y[H*p + s], p < N), applying the lags as spectral phase ramps while mixing. */
TSDRGPU_API int tsdrgpu_superb_local_spectra(tsdrgpu_ctx_t *ctx, void *stream, const float *d_hop, int count_pairs, int samples_in_frame,
                                             float *d_block, uint32_t *h_n, uint32_t *h_nd);
TSDRGPU_API int tsdrgpu_superb_lags(tsdrgpu_ctx_t *ctx, void *stream, const float *d_gathered, int nhops, uint64_t block_stride_complex,
                                    uint32_t n, uint32_t nd, int *h_lags);
TSDRGPU_API int tsdrgpu_superb_residue_ifft_lag(tsdrgpu_ctx_t *ctx, void *stream, const float *d_gathered, int nhops,
                                                uint64_t block_stride_complex, uint32_t n, int residue, const int *h_lags, float *d_out_residue);

/* ---- one hop per GPU, behind the C-ABI (SURVEY section 8e, DESIGN.md section 6; csrc/superb_mgpu.cu) ----------------------
 * superb_ondataready sharded over the GPUs of one node: rank q owns hop q.  Local spectra -> this rank's alignment lag (hop 0's
 * difference spectrum read from rank 0 over NVLink) -> an all-to-all mix (bins pulled from the peers, residues pushed to
 * them) -> one N-point inverse per rank -> |.| pushed into the root's window -> the root interleaves the time-contiguous
 * MAGNITUDE stream (what am_demod makes of superb_run's output, TSDRLibrary.c:271-274).  No host synchronisation, no
 * collective library: flags in peer memory order the phases.  A group object exists once per rank; the windows are tied
 * together either through CUDA IPC handles (one process per GPU: export -> exchange by any means -> connect_ipc) or directly
 * (all ranks in one process: connect_local).  nranks in {2, 4, 8} (a node has at most eight GPUs). */
typedef struct tsdrgpu_superb_mgpu tsdrgpu_superb_mgpu_t;
TSDRGPU_API int  tsdrgpu_superb_mgpu_create(tsdrgpu_ctx_t *ctx, int nranks, int rank, int root, uint32_t max_pairs_per_hop, tsdrgpu_superb_mgpu_t **g);
TSDRGPU_API void tsdrgpu_superb_mgpu_destroy(tsdrgpu_superb_mgpu_t *g);
TSDRGPU_API int  tsdrgpu_superb_mgpu_export(tsdrgpu_superb_mgpu_t *g, uint8_t handle[64]);
TSDRGPU_API int  tsdrgpu_superb_mgpu_connect_ipc(tsdrgpu_superb_mgpu_t *g, const uint8_t *handles /* nranks x 64 bytes, rank-major */);
TSDRGPU_API int  tsdrgpu_superb_mgpu_connect_local(tsdrgpu_superb_mgpu_t *const *all_ranks, int nranks);
/* unmap the peers' windows; with one process per GPU: all ranks disconnect, synchronise among themselves, then destroy */
TSDRGPU_API int  tsdrgpu_superb_mgpu_disconnect(tsdrgpu_superb_mgpu_t *g);
/* every rank calls this once per stitch (same count_pairs / samples_in_frame), each on a stream of its own device; asynchronous.
 * d_hop: this rank's hop.  d_hop0: a copy of hop 0 (the alignment reference, superbandwidth.c:133) on THIS device, or NULL --
 * then its difference spectrum is read from rank 0 over NVLink after one more barrier; either all ranks pass it or none.
 * The root's d_stream_out receives nranks * N magnitudes, N = fft_getrealsize(count_pairs) returned in *h_n. */
TSDRGPU_API int  tsdrgpu_superb_mgpu_stitch(tsdrgpu_superb_mgpu_t *g, void *stream, const float *d_hop, const float *d_hop0, int count_pairs,
                                            int samples_in_frame, float *d_stream_out, uint32_t *h_n);
/* lags (complex samples) of the last stitch as every rank published them, and the status word (0 = fine); synchronises `stream` */
/* the root's stream inside its window: valid after a stitch called with d_stream_out = NULL, until the root's next stitch */
TSDRGPU_API int  tsdrgpu_superb_mgpu_stream_window(tsdrgpu_superb_mgpu_t *g, float **d_stream);
TSDRGPU_API int  tsdrgpu_superb_mgpu_lags(tsdrgpu_superb_mgpu_t *g, void *stream, int *h_lags, uint32_t *h_status);

/* ---------------------------------------------------------------------------- a22+  coherent superbandwidth (beyond the reference)
 * The reference's mode above records hop 0 wherever the front end was left (two of its four hops share a tuning), copies each
 * hop's spectrum in FFT order to bins that have nothing to do with its tuning, and aligns the hops by an integer lag only.  The
 * coherent mode records H hops at known, overlapping tunings, places each hop's bins at their true frequencies, and matches
 * every hop to its neighbour in delay (to 1/1024 sample), phase and gain over their common bins.  It assumes the screen shows
 * the same picture over the whole round (as the reference's own alignment does): the joins are fitted on that common content.
 *
 * Spec (tsdrgpu_superband_t).  mode TSDRGPU_SUPERBAND_REFERENCE (0, the default): the reference's path, unchanged.  mode
 *   TSDRGPU_SUPERBAND_COHERENT (1): H = hops in {2, 4, 8}, overlap o = overlap_pct in [10, 50] percent.
 * Schedule (tsdrgpu_superband_schedule).  N = fft_getrealsize(10 floor(fs / fv)) pairs of each hop are used (the reference's
 *   10 frames).  Hop spacing D = 2 round((1 - o/100) N/2) bins (even; round half away from zero), overlap M = N - D.  Hop i is
 *   centred at c_i = (i - (H-1)/2) D bins of the stitched band and recorded at offset round(c_i fs / N) Hz through the retune
 *   callback.  Every hop, hop 0 included, is recorded after a retune and the 0.5 s pause.  A drop restarts the hop in progress.
 * Stitch (tsdrgpu_superb_stitch_coherent), with centred bin indices.  Hop r = floor((H-1)/2) is the reference; the joins chain
 *   outward from it (r+1, ..., H-1, then r-1, ..., 0): each newly placed hop b is matched to its corrected neighbour a.
 *   1. X_i = FFT_N(hop_i) / N (float32, exact stage angles).  Stitched bin kappa of hop i is its bin k = kappa - c_i.
 *   2. Overlap of a and b: M bins from kappa0 = c_upper - N/2, m = 0 .. M-1.  A_m, B_m the two hops' bins there (A corrected),
 *      C_m = A_m conj(B_m), u_m = sin^2 theta_m cos^2 theta_m, theta_m = pi (m + 1/2) / M (the crossfade weights' product).
 *   3. S(tau) = sum_m u_m C_m e^{2 pi i m tau / N}, in double.  tau0 = the first maximum of |S| over integers, from the N-point
 *      inverse transform of u C and the first-max argmax, mapped to (-N/2, N/2].  tau1 = the best of tau0 + j/32, tau^ the best of
 *      tau1 + j/1024 (j = -32 .. 32, S evaluated directly, ties to the smallest j).  g = S(tau^) / sum u |B|^2;
 *      rho = |S(tau^)| / sqrt(sum u |A|^2 sum u |B|^2) in [0, 1].  If sum u |B|^2 = 0: g = 0, tau^ = 0, rho = 0.
 *   4. B'_kappa = g B_kappa e^{-2 pi i (kappa - kappa0) tau^ / N} for every bin of hop b (a delay is a ramp over the whole band).
 *   5. Y over L = H N bins: in an overlap the lower hop weighs cos^2 theta_m, the upper sin^2 theta_m, elsewhere in a hop's band
 *      1; bins no hop covers are 0.  The hops span N + (H-1) D <= L bins, centred.
 *   6. y = IFFT_L(Y), unscaled (a tone of amplitude A in a hop keeps amplitude A): L pairs at H fs.
 *   Phases are formed in double from integers reduced mod 1 before sincospi (tau^ = T / 1024 with T an integer); every sum is in
 *   double with a fixed order (no atomics): the same inputs give the same bits.  The pipeline hands y to the decimator at H fs
 *   as the one-GPU reference path does. */
enum { TSDRGPU_SUPERBAND_REFERENCE = 0, TSDRGPU_SUPERBAND_COHERENT = 1 };
#define TSDRGPU_SUPERBAND_DEFAULT_HOPS    4
#define TSDRGPU_SUPERBAND_DEFAULT_OVERLAP 25
#define TSDRGPU_SUPERBAND_MIN_OVERLAP     10
#define TSDRGPU_SUPERBAND_MAX_OVERLAP     50
#define TSDRGPU_SUPERBAND_MAX_HOPS        8
typedef struct {
	int32_t mode;                                    /* TSDRGPU_SUPERBAND_* */
	int32_t hops;                                    /* H (coherent) */
	int32_t overlap_pct;                             /* o (coherent) */
} tsdrgpu_superband_t;
/* one join of a coherent stitch (48 bytes) */
typedef struct {
	int32_t hop, neighbour;                          /* b, a */
	int32_t tau0;                                    /* integer lag, in (-N/2, N/2] */
	int32_t kappa0;                                  /* lowest stitched bin of the overlap */
	int64_t tau_1024;                                /* tau^ x 1024, exact */
	double  tau;                                     /* tau^ in samples at fs */
	double  g_re, g_im;                              /* g */
	double  rho;                                     /* join quality, 0 .. 1 */
} tsdrgpu_superband_est_t;
/* host-only: the spelling shared by the host library's TSDR_SUPERBAND and Python.  "reference", or "coherent[:<H>[:<o>]]" (default
 * coherent:4:25); H and o are one to six decimal digits in the ranges above, nothing else.  TSDRGPU_OK with *out set, else
 * TSDRGPU_EINVAL and *out untouched. */
TSDRGPU_API int  tsdrgpu_superband_parse(const char *spec, tsdrgpu_superband_t *out);
/* host-only: the schedule of a coherent spec at fs > 0 and refresh rate fv > 0: *n = N, *d = D and offsets[i] (H values, may be
 * NULL) the retune offsets in Hz.  TSDRGPU_EINVAL for a spec that is not coherent and valid, N < 16, 10 floor(fs / fv) beyond 32 bits, or
 * an offset outside int32 (which no fs up to the host library's 500 MS/s reaches: |offset| <= 3.15 fs). */
TSDRGPU_API int  tsdrgpu_superband_schedule(const tsdrgpu_superband_t *spec, uint32_t fs, double refreshrate, uint32_t *n, uint32_t *d,
                                            int32_t *offsets);
/* asynchronous, never synchronises the host: the coherent stitch of `nhops` hops (d_hops: device pointers in a HOST array, each at
 * least count_pairs pairs) with hop spacing d (even, N/2 <= d < N, N = fft_getrealsize(count_pairs)).  d_out receives L = nhops N
 * interleaved pairs; d_est (device memory) nhops - 1 records, that of hop b at index b - (b > r).  Work memory is the context's
 * scratch: once a call of a size has run, the next call of that size allocates nothing. */
TSDRGPU_API int  tsdrgpu_superb_stitch_coherent(tsdrgpu_ctx_t *ctx, void *stream, float *const *d_hops, int nhops, int count_pairs, int d,
                                                float *d_out, tsdrgpu_superband_est_t *d_est);

/* ---------------------------------------------------------------------------- a1, a3, a5, a16, a17  streaming pipeline
 * replaces the body of process() (TSDRLibrary.c:264-298), decimatingthread / postprocessingthread /
 * videodecodingthread (TSDRLibrary.c:300-418) with their three rings (circbuff.c), dsp_dropped_compensation_*
 * (dsp.c:313-368) and the frame-rate detector's capture loop (frameratedetector.c:128-187, 215-230).
 * HOST buffers in (the plugin's), HOST frame / plot buffers out (valid during the callback only), callbacks on an
 * internal delivery thread.  The C host library (tempestsdr_b200/host) forwards the reference's process() here.
 * The setters (all but set_superb_devices), tsdrgpu_pipeline_sync and get_geometry may be called from any thread, also while
 * process() runs on another; each call takes effect whole, from the next process() call or group of decimator blocks on.
 */
typedef struct tsdrgpu_pipeline tsdrgpu_pipeline_t;

enum {                                   /* indices of params_int: TSDRLibrary.h:32-41 */
	TSDRGPU_PARAM_INT_AUTOSHIFT = 0, TSDRGPU_PARAM_INT_FRAMERATE_PLL = 1, TSDRGPU_PARAM_AUTOCORR_PLOTS_RESET = 2,
	TSDRGPU_PARAM_AUTOCORR_PLOTS_OFF = 3, TSDRGPU_PARAM_AUTOCORR_SUPERRESOLUTION = 4,
	TSDRGPU_PARAM_NEAREST_NEIGHBOUR_RESAMPLING = 5, TSDRGPU_PARAM_LOW_PASS_BEFORE_SYNC = 6,
	TSDRGPU_PARAM_AUTOGAIN_AFTER_PROCESSING = 7, TSDRGPU_PARAM_AUTOCORR_DUMP = 8
};

typedef struct {
	uint32_t samplerate;                 /* tsdrplugin_getsamplerate() */
	int      height;                     /* tsdr_setresolution */
	double   refreshrate;
	float    motionblur;                 /* tsdr_motionblur */
	uint32_t params_int[9];              /* tsdr_setparameter_int */
	int      batch_frames;               /* frames per frame-stage launch (>= 1; 1 = lowest latency) */
	int      batch_blocks;               /* decimator blocks (0.1 frame each) per resampler launch (>= 1; default 10) */
	int      block_when_busy;            /* 1: wait for the frame callback instead of dropping a batch */
} tsdrgpu_pipeline_config_t;

typedef struct {
	uint64_t samples_in, samples_dropped_upstream, samples_resampled;
	uint64_t frames_processed, frames_delivered, frames_dropped, captures, plots_delivered;
	uint64_t h2d_bytes, d2h_bytes, gpu_launches, stitches;
	uint64_t host_buffers_registered;   /* plugin buffers page-locked in place (cudaHostRegister) after they kept coming back */
	uint64_t spectra_delivered, spectra_skipped;   /* spectrum reports handed to plot_cb / skipped because every report slot was busy */
	uint64_t coherence_delivered, coherence_skipped;   /* the same for coherence reports */
} tsdrgpu_pipeline_stats_t;

typedef void (*tsdrgpu_frame_cb)(float *buf, int width, int height, void *user);                  /* tsdr_readasync_function */
typedef void (*tsdrgpu_value_cb)(int value_id, double arg0, double arg1, void *user);             /* tsdr_value_changed_callback */
typedef void (*tsdrgpu_plot_cb)(int plot_id, int offset, double *values, int size, uint32_t samplerate, void *user);
typedef void (*tsdrgpu_retune_cb)(int32_t offset_hz, void *user);        /* shiftfreq (TSDRLibrary.c:208): tune to centre + offset */

TSDRGPU_API int  tsdrgpu_pipeline_create(tsdrgpu_ctx_t *ctx, const tsdrgpu_pipeline_config_t *cfg, tsdrgpu_frame_cb frame_cb,
                                         tsdrgpu_value_cb value_cb, tsdrgpu_plot_cb plot_cb, void *user, tsdrgpu_pipeline_t **p);
TSDRGPU_API void tsdrgpu_pipeline_destroy(tsdrgpu_pipeline_t *p);
/* == process(buf, items_count, ctx, samples_dropped): returns once h_iq has been read (it may then be reused) */
TSDRGPU_API int  tsdrgpu_pipeline_process(tsdrgpu_pipeline_t *p, const float *h_iq, uint64_t items_count, int64_t samples_dropped);
/* The same with the samples still in the front end's wire format (SURVEY section 8f-1): the block crosses PCIe as 1 or 2
 * bytes per component and is converted on the device to exactly the floats TSDRPlugin_RawFile.c:241-261 would have
 * produced on the host.  fmt uses the RawFile plugin's own numbering (TSDRPlugin_RawFile.c:29-33). */
enum { TSDRGPU_FMT_FLOAT = 0, TSDRGPU_FMT_INT8 = 1, TSDRGPU_FMT_INT16 = 2, TSDRGPU_FMT_UINT8 = 3, TSDRGPU_FMT_UINT16 = 4 };
/* the conversion alone, device to device (d_raw: items_count samples of `fmt`; d_out: items_count floats) */
TSDRGPU_API int  tsdrgpu_convert_samples(tsdrgpu_ctx_t *ctx, void *stream, const void *d_raw, int fmt, uint64_t items_count, float *d_out);
TSDRGPU_API int  tsdrgpu_pipeline_process_raw(tsdrgpu_pipeline_t *p, const void *h_samples, int fmt, uint64_t items_count, int64_t samples_dropped);
/* For a front end with a ring of page-locked buffers: returns once everything is enqueued; the buffer must stay untouched until
 * tsdrgpu_pipeline_sync_input() returns.  Consecutive blocks then cross the link back to back. */
TSDRGPU_API int  tsdrgpu_pipeline_process_raw_async(tsdrgpu_pipeline_t *p, const void *h_pinned_samples, int fmt, uint64_t items_count, int64_t samples_dropped);
TSDRGPU_API int  tsdrgpu_pipeline_sync_input(tsdrgpu_pipeline_t *p);
TSDRGPU_API int  tsdrgpu_pipeline_flush(tsdrgpu_pipeline_t *p);            /* waits for the GPU and for every pending callback */
TSDRGPU_API int  tsdrgpu_pipeline_set_param_int(tsdrgpu_pipeline_t *p, int id, uint32_t value);
TSDRGPU_API int  tsdrgpu_pipeline_set_resolution(tsdrgpu_pipeline_t *p, int height, double refreshrate);
TSDRGPU_API int  tsdrgpu_pipeline_set_samplerate(tsdrgpu_pipeline_t *p, uint32_t samplerate);
/* superbandwidth mode (PARAM_AUTOCORR_SUPERRESOLUTION = 1; superb_run, superbandwidth.c:179-254) retunes the front end
 * between hops through this callback; without it the hops are recorded at one frequency */
TSDRGPU_API int  tsdrgpu_pipeline_set_retune(tsdrgpu_pipeline_t *p, tsdrgpu_retune_cb cb);
/* superbandwidth with ONE HOP PER GPU (tsdrgpu_superb_mgpu_*): devices[0] = the pipeline's own device, n in {2, 4, 8} hops =
 * devices of this node with peer access; hop i is recorded into device i's memory and transformed there, device 0 receives the
 * stitched magnitude stream and makes the frames.  n <= 1: back to 4 hops on one GPU (the reference's SUPER_HOPS_TO_MAKE). */
TSDRGPU_API int  tsdrgpu_pipeline_set_superb_devices(tsdrgpu_pipeline_t *p, const int *devices, int n);
/* superbandwidth stitch (see tsdrgpu_superb_stitch_coherent; NULL: TSDRGPU_SUPERBAND_REFERENCE, the default), taking effect at the
 * next round.  The coherent mode runs on one GPU: a coherent spec while set_superb_devices holds n > 1 devices is refused with
 * TSDRGPU_EINVAL, and so is set_superb_devices with n > 1 while the spec is coherent. */
TSDRGPU_API int  tsdrgpu_pipeline_set_superband(tsdrgpu_pipeline_t *p, const tsdrgpu_superband_t *spec);
/* the last coherent round's joins (synchronises): *n = H - 1 records into out (capacity cap), in tsdrgpu_superb_stitch_coherent's
 * order; *n = 0 before the first coherent stitch.  Call it between process() calls. */
TSDRGPU_API int  tsdrgpu_pipeline_superband_estimates(tsdrgpu_pipeline_t *p, tsdrgpu_superband_est_t *out, int cap, int *n);
/* Page-lock the caller's sample buffers in place (cudaHostRegister) once the same buffer has been handed to process() three
 * times, so that pageable plugin memory crosses PCIe by direct DMA.  Off by default: only for callers that keep their buffer
 * mapped for the whole run (the reference's plugins malloc once per tsdrplugin_readasync); released at destroy. */
TSDRGPU_API int  tsdrgpu_pipeline_set_host_registration(tsdrgpu_pipeline_t *p, int on);
TSDRGPU_API int  tsdrgpu_pipeline_set_motionblur(tsdrgpu_pipeline_t *p, float coeff);
/* SURVEY section 8f-2: deliver final pixels.  mode 1: the frame callback's buffer holds w*h int32 pixels of the JNI glue's
 * float->ARGB rule (TSDRLibraryNDK.c:222-283) instead of floats (same size, so the callback type is unchanged: cast it);
 * inverted as the GUI's "inverted colours".  mode 0 (default): floats, as the reference. */
TSDRGPU_API int  tsdrgpu_pipeline_set_output_argb(tsdrgpu_pipeline_t *p, int mode, int inverted);
/* SURVEY section 8f-4 / 8f-3, both off by default because the reference announces neither:
 *  report_snr:  value callback id 4 (VALUE_ID_SNR, TSDRLibrary.h:52) with dsp_autogain_t.snr next to every auto-gain report
 *               (the announce dsp.c:234 leaves commented out);
 *  detect_mode: after every pair of plots, value callback id TSDRGPU_VALUE_ID_DETECTED_MODE with (fps, height) computed
 *               like the GUI's auto-resolution (tsdrgpu_detect_videomode). */
#define TSDRGPU_VALUE_ID_DETECTED_MODE 100
TSDRGPU_API int  tsdrgpu_pipeline_set_reports(tsdrgpu_pipeline_t *p, int report_snr, int detect_mode);
/* resampling kernel (TSDRGPU_RS_BOX, the default, or TSDRGPU_RS_SINC; see tsdrgpu_resampler_set_kernel), taking effect at the
 * next group of decimator blocks like set_param_int; PARAM_NEAREST_NEIGHBOUR_RESAMPLING = 1 still wins */
TSDRGPU_API int  tsdrgpu_pipeline_set_resampler(tsdrgpu_pipeline_t *p, int kernel);
/* auto-gain levels (TSDRGPU_AG_MINMAX, the default, or TSDRGPU_AG_CLIP with ppm; see tsdrgpu_framestage_set_autogain), taking
 * effect at the next frame-stage batch */
TSDRGPU_API int  tsdrgpu_pipeline_set_autogain(tsdrgpu_pipeline_t *p, int mode, int ppm);
/* contrast mode (TSDRGPU_CONTRAST_OFF, the default, or TSDRGPU_CONTRAST_CLAHE; see tsdrgpu_framestage_set_contrast), taking
 * effect at the next frame-stage batch */
TSDRGPU_API int  tsdrgpu_pipeline_set_contrast(tsdrgpu_pipeline_t *p, int mode, int clip_centi, int tx, int ty);
/* denoise mode (TSDRGPU_DENOISE_OFF, the default, or TSDRGPU_DENOISE_NLM; see tsdrgpu_framestage_set_denoise), taking effect
 * at the next frame-stage batch */
TSDRGPU_API int  tsdrgpu_pipeline_set_denoise(tsdrgpu_pipeline_t *p, int mode, int h_milli, int r, int p_radius);
/* deblur mode (TSDRGPU_DEBLUR_OFF, the default, or TSDRGPU_DEBLUR_RL; see tsdrgpu_framestage_set_deblur), taking effect at the
 * next frame-stage batch */
TSDRGPU_API int  tsdrgpu_pipeline_set_deblur(tsdrgpu_pipeline_t *p, int mode, int sigma_centi, int iterations);
/* stack mode (TSDRGPU_STACK_OFF, the default, TSDRGPU_STACK_ALIGN, TSDRGPU_STACK_ADAPT, TSDRGPU_STACK_TRACK or TSDRGPU_STACK_ROBUST; see tsdrgpu_framestage_set_stack),
 * taking effect at the next frame-stage batch.  tsdrgpu_pipeline_sync restarts the stack at the next frame-stage batch.  While
 * the stack is on, every frame with an auto-gain report (dsp.c:231-235) also announces value id TSDRGPU_VALUE_ID_STACK_DRIFT with arg0 = the mean drift
 * in px/frame since the last announcement or restart ((o - o_last) / frames, 0 right after a restart) and arg1 = the frame's
 * offset o mod W H, in [0, W H).  The drift is the refresh-rate error the PLL has left: a picture that drifts by d px/frame
 * over W H delivered pixels per frame has its refresh rate off by about -d / (W H) relative. */
#define TSDRGPU_VALUE_ID_STACK_DRIFT 101
TSDRGPU_API int  tsdrgpu_pipeline_set_stack(tsdrgpu_pipeline_t *p, int mode, int depth, int rx, int ry);
/* channel filter (see tsdrgpu_chanfilt_*; NULL or taps == 0: off, the default), taking effect at the next process().  Each block is
 * filtered on the device right after its H2D copy and raw-format conversion, so the resampler (every kernel) and the frame-rate
 * detector both see the filtered stream.  The taps follow the samplerate.  The history is zeroed before a block when the call
 * reports samples_dropped != 0, when the previous block with samples was not filtered (drop compensation discarded all of it and no
 * capture needed it, or the filter was off) and after superbandwidth mode: that mode records its hops unfiltered, because the
 * bands refer to one tuning. */
TSDRGPU_API int  tsdrgpu_pipeline_set_channel(tsdrgpu_pipeline_t *p, const tsdrgpu_channel_t *spec);
/* Welch spectrum of the IQ stream (see tsdrgpu_spectrum_*; NULL or n == 0: off, the default), taking effect at the next process().
 * It taps each block right after its H2D copy and raw-format conversion, before the channel filter, on a low-priority stream of its
 * own, and changes nothing else.  Every report goes to plot_cb(TSDRGPU_PLOT_ID_SPECTRUM, -N/2, values, N, fs) on the delivery thread,
 * in order; when every report slot is still held by the host that delivery is skipped (stats.spectra_skipped).  A call with
 * samples_dropped != 0 starts a new run; a new samplerate and superbandwidth mode (suspended for the whole mode: its hops are
 * recorded at different tunings) discard the report in progress. */
#define TSDRGPU_PLOT_ID_SPECTRUM 100
TSDRGPU_API int  tsdrgpu_pipeline_set_spectrum(tsdrgpu_pipeline_t *p, const tsdrgpu_welch_t *spec);
/* Spectral coherence of the IQ stream at the line rate (see tsdrgpu_coherence_*; NULL or rate == 0: off, the default), taking effect
 * at the next process().  It taps where the spectrum does (after the raw-format conversion, before the channel filter, whose bands it
 * helps to place), runs on the spectrum's low-priority stream and changes nothing else.  alpha = height x refresh rate and fs = the
 * samplerate, read per call.  Every report goes to plot_cb(TSDRGPU_PLOT_ID_COHERENCE, -N/2, gamma, N, fs) on the delivery thread, in
 * order; when every report slot is still held by the host that delivery is skipped (stats.coherence_skipped).  A call with
 * samples_dropped != 0, a new samplerate or N, and superbandwidth mode (suspended for the whole mode) discard the report in
 * progress.  While the geometry is unresolvable (tsdrgpu_coherence_n == 0) no reports are made. */
#define TSDRGPU_PLOT_ID_COHERENCE 101
TSDRGPU_API int  tsdrgpu_pipeline_set_coherence(tsdrgpu_pipeline_t *p, const tsdrgpu_coherence_t *spec);
TSDRGPU_API int  tsdrgpu_pipeline_sync(tsdrgpu_pipeline_t *p, int pixels);   /* tsdr_sync: syncoffset += pixels */
TSDRGPU_API int  tsdrgpu_pipeline_get_geometry(tsdrgpu_pipeline_t *p, int *width, int *height, double *refreshrate);
TSDRGPU_API int  tsdrgpu_pipeline_stats(tsdrgpu_pipeline_t *p, tsdrgpu_pipeline_stats_t *out);

#ifdef __cplusplus
}
#endif
#endif
