/* host_plan.c -- host-side scalar planning for libtsdrgpu.  Plain C on purpose ("host code stays C"): these are
 * the data-independent scalar recurrences of the reference, replayed with the reference's operand types and
 * operation order so the device kernels receive bit-identical parameters. */
#include "host_plan.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

uint64_t tsdrgpu_plan_resample(double *offset, const uint32_t *sizes, uint32_t uniform, uint32_t nblocks,
                               double upsample_by, double downsample_by, tsdrgpu_rs_block_t *blocks) {
	const double r = upsample_by / downsample_by;          /* dsp.c:258 */
	const double rinv = downsample_by / upsample_by;       /* dsp.c:259 */
	double off = *offset;
	uint64_t in_pos = 0, out_pos = 0;
	for (uint32_t b = 0; b < nblocks; b++) {
		const uint32_t size = sizes ? sizes[b] : uniform;
		const uint32_t n_out = (uint32_t) (int) ((size - off) * r);      /* dsp.c:262 */
		if (n_out == 0) return UINT64_MAX;
		if (blocks) {
			blocks[b].in_start = in_pos; blocks[b].out_start = out_pos;
			blocks[b].size = size; blocks[b].n_out = n_out;
			blocks[b].r = r; blocks[b].phase = -off * r;                  /* dsp.c:272 */
		}
		off += n_out * rinv - size;                                       /* dsp.c:306 */
		in_pos += size; out_pos += n_out;
	}
	*offset = off;
	return out_pos;
}

void tsdrgpu_geometry(uint32_t samplerate, int height, double refreshrate, int *width, double *pixelrate,
                      double *pixeltimeoversampletime) {
	const double real_width = samplerate / (refreshrate * height);
	const int w = (int) (2 * real_width);
	const double pr = w * height * refreshrate;
	*width = w; *pixelrate = pr;
	*pixeltimeoversampletime = (samplerate != 0 && pr != 0) ? ((double) samplerate) / pr : 0.0;
}

/* frameratepll's write-back (syncdetector.c:141-152): `refreshrate -= vx * 1e-5` while unlocked, `avg_speed * 1e-6` once
 * locked, only when the frame moved (vx != 0).  The averages themselves come from the frame stage (fs_sync). */
int tsdrgpu_pll_step(double *refreshrate, int32_t x_vx, int32_t pll_state, double avg_speed) {
	if (x_vx == 0) return 0;
	const double diff = (pll_state == 0) ? x_vx * 0.00001 : avg_speed * 0.000001;
	*refreshrate -= diff;
	return 1;
}

void tsdrgpu_gauss_taps(float taps[5]) {
	/* CALC_GAUSSCOEFF(N,i) = expf(-2.0f*ALPHA*ALPHA*i*i/(N*N)) with textual i in {-2,-1,0,1,2}, N = 5 */
	const float e2 = expf(-2.0f * 1.0f * 1.0f * -2 * -2 / (5 * 5));
	const float e1 = expf(-2.0f * 1.0f * 1.0f * -1 * -1 / (5 * 5));
	const float e0 = expf(-2.0f * 1.0f * 1.0f * 0 * 0 / (5 * 5));
	const float norm = e2 + e1 + e0 + e1 + e2;
	taps[0] = e2 / norm; taps[1] = e1 / norm; taps[2] = e0 / norm; taps[3] = e1 / norm; taps[4] = e2 / norm;
}

/* I0, the modified Bessel function of the first kind, by its power series (converges for every x; beta = 5 needs ~20 terms) */
static double bessel_i0(double x) {
	double sum = 1.0, term = 1.0;
	for (int k = 1; k < 200; k++) {
		const double f = x / (2.0 * k);
		term *= f * f;
		sum += term;
		if (term < 1e-17 * sum) break;
	}
	return sum;
}

/* the windowed-sinc resampler's taps (definition in tsdrgpu.h) */
int tsdrgpu_sinc_taps(double r, float *taps, int *T, int *L) {
	const int nt = TSDRGPU_SINC_TAPS, nl = TSDRGPU_SINC_PHASES;
	if (T) *T = nt;
	if (L) *L = nl;
	if (!taps) return TSDRGPU_OK;
	if (!(r > 0)) return TSDRGPU_EINVAL;
	const double pi = 3.14159265358979323846;
	const double fc = 0.5 * (r < 1.0 ? r : 1.0), half = 0.5 * nt;
	for (int j = 0; j < nl; j++) {
		double h[TSDRGPU_SINC_TAPS], sum = 0.0;
		for (int t = 0; t < nt; t++) {
			const double d = (double) (t - (nt / 2 - 1)) - (double) j / nl;
			const double x = pi * 2.0 * fc * d;
			const double s = (x == 0.0) ? 1.0 : sin(x) / x;
			const double z = d / half, a = 1.0 - z * z;
			h[t] = s * bessel_i0(TSDRGPU_SINC_BETA * sqrt(a > 0.0 ? a : 0.0));
			sum += h[t];
		}
		for (int t = 0; t < nt; t++) taps[j * nt + t] = (float) (h[t] / sum);
	}
	return TSDRGPU_OK;
}

/* ---- channel filter (definition in tsdrgpu.h) */
static int channel_valid(const tsdrgpu_channel_t *s) {
	const int64_t M = TSDRGPU_CHANNEL_MAX_HZ;
	if (s->taps < TSDRGPU_CHANNEL_MIN_TAPS || s->taps > TSDRGPU_CHANNEL_MAX_TAPS || (s->taps & 1) == 0) return 0;
	if (s->nstop < 0 || s->nstop > TSDRGPU_CHANNEL_MAX_STOPS) return 0;
	if (s->pass_lo_hz < -M || s->pass_hi_hz > M || !(s->pass_lo_hz < s->pass_hi_hz)) return 0;
	for (int k = 0; k < s->nstop; k++) {
		const int64_t a = s->stop_lo_hz[k], b = s->stop_hi_hz[k];
		if (!(a < b) || a < s->pass_lo_hz || b > s->pass_hi_hz) return 0;
		for (int j = 0; j < k; j++) {
			const int64_t lo = a > s->stop_lo_hz[j] ? a : s->stop_lo_hz[j], hi = b < s->stop_hi_hz[j] ? b : s->stop_hi_hz[j];
			if (lo < hi) return 0;
		}
	}
	return 1;
}

/* a decimal integer with an optional leading '-': at most 12 digits (so no overflow; the range check follows) */
static int channel_int(const char **c, int64_t *v) {
	const char *p = *c;
	const int neg = (*p == '-');
	if (neg) p++;
	int64_t x = 0;
	int n = 0;
	while (*p >= '0' && *p <= '9') { if (++n > 12) return 0; x = 10 * x + (*p++ - '0'); }
	if (n == 0) return 0;
	*v = neg ? -x : x;
	*c = p;
	return 1;
}

int tsdrgpu_channel_parse(const char *spec, tsdrgpu_channel_t *out) {
	if (!spec || !out) return TSDRGPU_EINVAL;
	tsdrgpu_channel_t s;
	memset(&s, 0, sizeof s);
	if (strcmp(spec, "off") == 0) { *out = s; return TSDRGPU_OK; }
	const char *c = spec;
	if (strncmp(c, "pass:", 5) != 0) return TSDRGPU_EINVAL;
	c += 5;
	if (!channel_int(&c, &s.pass_lo_hz) || *c++ != ':' || !channel_int(&c, &s.pass_hi_hz)) return TSDRGPU_EINVAL;
	while (strncmp(c, ",stop:", 6) == 0) {
		if (s.nstop == TSDRGPU_CHANNEL_MAX_STOPS) return TSDRGPU_EINVAL;
		c += 6;
		if (!channel_int(&c, &s.stop_lo_hz[s.nstop]) || *c++ != ':' || !channel_int(&c, &s.stop_hi_hz[s.nstop])) return TSDRGPU_EINVAL;
		s.nstop++;
	}
	s.taps = TSDRGPU_CHANNEL_DEFAULT_TAPS;
	if (strncmp(c, ",taps:", 6) == 0) {
		c += 6;
		int64_t t;
		if (*c == '-' || !channel_int(&c, &t) || t > TSDRGPU_CHANNEL_MAX_TAPS) return TSDRGPU_EINVAL;
		s.taps = (int32_t) t;
	}
	if (*c || !channel_valid(&s)) return TSDRGPU_EINVAL;
	*out = s;
	return TSDRGPU_OK;
}

/* ---- the Welch spectrum's spelling, window and K (definitions in tsdrgpu.h) */
static int spectrum_valid(const tsdrgpu_welch_t *s) {
	return s->n >= TSDRGPU_SPECTRUM_MIN_N && s->n <= TSDRGPU_SPECTRUM_MAX_N && (s->n & (s->n - 1)) == 0 && s->rate >= 1 &&
	       s->rate <= TSDRGPU_SPECTRUM_MAX_RATE;
}

/* one to six decimal digits, *c moved past them; 0 for none or more than six */
static int spectrum_digits(const char **c, int32_t *v) {
	int32_t x = 0;
	int n = 0;
	while (**c >= '0' && **c <= '9') { if (++n > 6) return 0; x = 10 * x + (*(*c)++ - '0'); }
	*v = x;
	return n > 0;
}

int tsdrgpu_spectrum_parse(const char *spec, tsdrgpu_welch_t *out) {
	if (!spec || !out) return TSDRGPU_EINVAL;
	tsdrgpu_welch_t s = {0, 0};
	if (strcmp(spec, "off") == 0) { *out = s; return TSDRGPU_OK; }
	const char *c = spec;
	if (strncmp(c, "welch:", 6) != 0) return TSDRGPU_EINVAL;
	c += 6;
	if (!spectrum_digits(&c, &s.n)) return TSDRGPU_EINVAL;
	s.rate = TSDRGPU_SPECTRUM_DEFAULT_RATE;
	if (*c == ':') { c++; if (!spectrum_digits(&c, &s.rate)) return TSDRGPU_EINVAL; }
	if (*c || !spectrum_valid(&s)) return TSDRGPU_EINVAL;
	*out = s;
	return TSDRGPU_OK;
}

int tsdrgpu_spectrum_window(int n, double *w) {
	const tsdrgpu_welch_t s = {n, 1};
	if (!w || !spectrum_valid(&s)) return TSDRGPU_EINVAL;
	const double pi = 3.14159265358979323846;
	for (int i = 0; i < n; i++) {
		const double x = 2.0 * pi * i / n;
		w[i] = 0.35875 - 0.48829 * cos(x) + 0.14128 * cos(2.0 * x) - 0.01168 * cos(3.0 * x);
	}
	return TSDRGPU_OK;
}

uint32_t tsdrgpu_spectrum_k(const tsdrgpu_welch_t *spec, uint32_t fs) {
	if (!spec || fs == 0 || !spectrum_valid(spec)) return 0;
	const uint64_t k = (uint64_t) fs / ((uint64_t) spec->rate * (uint64_t) (spec->n / 2));
	return k > 0 ? (uint32_t) k : 1u;
}

/* ---- the coherence's spelling, N and window (definitions in tsdrgpu.h) */
int tsdrgpu_coherence_parse(const char *spec, tsdrgpu_coherence_t *out) {
	if (!spec || !out) return TSDRGPU_EINVAL;
	tsdrgpu_coherence_t s = {0};
	if (strcmp(spec, "off") == 0) { *out = s; return TSDRGPU_OK; }
	const char *c = spec;
	if (strncmp(c, "line", 4) != 0) return TSDRGPU_EINVAL;
	c += 4;
	s.rate = TSDRGPU_COHERENCE_DEFAULT_RATE;
	if (*c == ':') { c++; if (!spectrum_digits(&c, &s.rate)) return TSDRGPU_EINVAL; }
	if (*c || s.rate < 1 || s.rate > TSDRGPU_COHERENCE_MAX_RATE) return TSDRGPU_EINVAL;
	*out = s;
	return TSDRGPU_OK;
}

uint32_t tsdrgpu_coherence_n(uint32_t fs, double alpha) {
	if (fs == 0 || !(alpha > 0.0) || alpha > 1e300) return 0;
	const double need = 16.0 * (double) fs / alpha;
	uint32_t n = TSDRGPU_SPECTRUM_MIN_N;
	while ((double) n < need) { if (n >= TSDRGPU_SPECTRUM_MAX_N) return 0; n *= 2; }
	return n;
}

int tsdrgpu_coherence_window(int n, double alpha, uint32_t fs, double *w2) {
	const tsdrgpu_welch_t s = {n, 1};
	if (!w2 || !spectrum_valid(&s) || fs == 0 || !(alpha > 0.0) || alpha > 1e300) return TSDRGPU_EINVAL;
	const double pi = 3.14159265358979323846;
	tsdrgpu_spectrum_window(n, w2 + n);                /* the real window in the upper half, read before it is overwritten */
	for (int i = 0; i < n; i++) {
		const double w = w2[n + i], a = -pi * fmod(alpha * (double) i / (double) fs, 2.0);
		w2[2 * i] = w * cos(a);
		w2[2 * i + 1] = w * sin(a);
	}
	return TSDRGPU_OK;
}

/* ---- auto-gain, contrast, denoise, stack and deblur options (definitions in tsdrgpu.h) */
int autogain_ok(int mode, int ppm) {
	return (mode == TSDRGPU_AG_MINMAX || mode == TSDRGPU_AG_CLIP) && ppm >= 0 && ppm <= TSDRGPU_AG_MAX_PPM;
}

int contrast_ok(int mode, int clip_centi, int tx, int ty) {
	return mode == TSDRGPU_CONTRAST_OFF || (mode == TSDRGPU_CONTRAST_CLAHE && clip_centi >= TSDRGPU_CLAHE_MIN_CLIP &&
	       clip_centi <= TSDRGPU_CLAHE_MAX_CLIP && tx >= 1 && tx <= TSDRGPU_CLAHE_MAX_TILES && ty >= 1 && ty <= TSDRGPU_CLAHE_MAX_TILES);
}

int denoise_ok(int mode, int h_milli, int r, int p) {
	return mode == TSDRGPU_DENOISE_OFF || (mode == TSDRGPU_DENOISE_NLM && h_milli >= 1 && h_milli <= TSDRGPU_NLM_MAX_H && r >= 1 &&
	       r <= TSDRGPU_NLM_MAX_R && p >= 1 && p <= TSDRGPU_NLM_MAX_P);
}

int stack_ok(int mode, int depth, int rx, int ry) {
	return mode == TSDRGPU_STACK_OFF || ((mode == TSDRGPU_STACK_ALIGN || mode == TSDRGPU_STACK_ADAPT || mode == TSDRGPU_STACK_TRACK ||
	                                      mode == TSDRGPU_STACK_ROBUST) && depth >= TSDRGPU_STACK_MIN_N &&
	       depth <= TSDRGPU_STACK_MAX_N && rx >= 1 && rx <= TSDRGPU_STACK_MAX_RX && ry >= 0 && ry <= TSDRGPU_STACK_MAX_RY);
}

int deblur_ok(int mode, int sigma_centi, int iterations) {
	return mode == TSDRGPU_DEBLUR_OFF || (mode == TSDRGPU_DEBLUR_RL && sigma_centi >= TSDRGPU_DEBLUR_MIN_SIGMA &&
	       sigma_centi <= TSDRGPU_DEBLUR_MAX_SIGMA && iterations >= 1 && iterations <= TSDRGPU_DEBLUR_MAX_ITER);
}

/* one to six decimal digits -> their value, *c moved past them; -1 for none or more than six */
static int option_digits(const char **c) {
	int v = 0, d = 0;
	while (**c >= '0' && **c <= '9' && d < 7) { v = 10 * v + (**c - '0'); (*c)++; d++; }
	return (d == 0 || d == 7) ? -1 : v;
}

/* the contrast and denoise spellings: "off" -> 0 with v = {0, 0, 0}; "<prefix><x>" or "<prefix><x>:<a><sep><b>" -> 1 with
 * v = {x, a, b}, a and b defaulting to da and db.  x = a whole part of one to six digits, then optionally '.' and one to k
 * digits, read as the integer x 10^k.  -1 if malformed; the ranges are the caller's. */
static int option_parse(const char *spec, const char *prefix, int k, char sep, int da, int db, int v[3]) {
	if (strcmp(spec, "off") == 0) { v[0] = v[1] = v[2] = 0; return 0; }
	const size_t np = strlen(prefix);
	if (strncmp(spec, prefix, np) != 0) return -1;
	const char *c = spec + np;
	if ((v[0] = option_digits(&c)) < 0) return -1;
	for (int i = 0; i < k; i++) v[0] *= 10;
	if (*c == '.') {
		const char *f = ++c;
		int frac = option_digits(&c);
		const int nd = (int) (c - f);
		if (frac < 0 || nd > k) return -1;
		for (int i = nd; i < k; i++) frac *= 10;
		v[0] += frac;
	}
	v[1] = da; v[2] = db;
	if (*c == ':') {
		c++; v[1] = option_digits(&c);
		if (*c != sep) return -1;
		c++; v[2] = option_digits(&c);
	}
	return *c ? -1 : 1;
}

int tsdrgpu_contrast_parse(const char *spec, int *mode, int *clip_centi, int *tx, int *ty) {
	int v[3], on;
	if (!spec || !mode || !clip_centi || !tx || !ty || (on = option_parse(spec, "clahe:", 2, 'x', 8, 8, v)) < 0) return TSDRGPU_EINVAL;
	const int m = on ? TSDRGPU_CONTRAST_CLAHE : TSDRGPU_CONTRAST_OFF;
	if (!contrast_ok(m, v[0], v[1], v[2])) return TSDRGPU_EINVAL;
	*mode = m; *clip_centi = v[0]; *tx = v[1]; *ty = v[2];
	return TSDRGPU_OK;
}

int tsdrgpu_denoise_parse(const char *spec, int *mode, int *h_milli, int *r, int *p) {
	int v[3], on;
	if (!spec || !mode || !h_milli || !r || !p || (on = option_parse(spec, "nlm:", 3, ':', 5, 1, v)) < 0) return TSDRGPU_EINVAL;
	const int m = on ? TSDRGPU_DENOISE_NLM : TSDRGPU_DENOISE_OFF;
	if (!denoise_ok(m, v[0], v[1], v[2])) return TSDRGPU_EINVAL;
	*mode = m; *h_milli = v[0]; *r = v[1]; *p = v[2];
	return TSDRGPU_OK;
}

int tsdrgpu_stack_parse(const char *spec, int *mode, int *depth, int *rx, int *ry) {
	int v[3], on, m = TSDRGPU_STACK_ALIGN;
	if (!spec || !mode || !depth || !rx || !ry) return TSDRGPU_EINVAL;
	if ((on = option_parse(spec, "align:", 0, 'x', 8, 2, v)) < 0) { on = option_parse(spec, "adapt:", 0, 'x', 8, 2, v); m = TSDRGPU_STACK_ADAPT; }
	if (on < 0) { on = option_parse(spec, "track:", 0, 'x', 8, 2, v); m = TSDRGPU_STACK_TRACK; }
	if (on < 0) { on = option_parse(spec, "robust:", 0, 'x', 8, 2, v); m = TSDRGPU_STACK_ROBUST; }
	if (on < 0) return TSDRGPU_EINVAL;
	if (!on) m = TSDRGPU_STACK_OFF;
	if (!stack_ok(m, v[0], v[1], v[2])) return TSDRGPU_EINVAL;
	*mode = m; *depth = v[0]; *rx = v[1]; *ry = v[2];
	return TSDRGPU_OK;
}

/* ---- the coherent superbandwidth mode's spelling and schedule (definitions in tsdrgpu.h) */
int superband_ok(const tsdrgpu_superband_t *s) {
	return s->mode == TSDRGPU_SUPERBAND_REFERENCE || (s->mode == TSDRGPU_SUPERBAND_COHERENT && (s->hops == 2 || s->hops == 4 || s->hops == 8) &&
	       s->overlap_pct >= TSDRGPU_SUPERBAND_MIN_OVERLAP && s->overlap_pct <= TSDRGPU_SUPERBAND_MAX_OVERLAP);
}

int tsdrgpu_superband_parse(const char *spec, tsdrgpu_superband_t *out) {
	if (!spec || !out) return TSDRGPU_EINVAL;
	tsdrgpu_superband_t s = {TSDRGPU_SUPERBAND_REFERENCE, 0, 0};
	if (strcmp(spec, "reference") != 0) {
		const char *c = spec;
		if (strncmp(c, "coherent", 8) != 0) return TSDRGPU_EINVAL;
		c += 8;
		s.mode = TSDRGPU_SUPERBAND_COHERENT; s.hops = TSDRGPU_SUPERBAND_DEFAULT_HOPS; s.overlap_pct = TSDRGPU_SUPERBAND_DEFAULT_OVERLAP;
		if (*c == ':') {
			c++; if ((s.hops = option_digits(&c)) < 0) return TSDRGPU_EINVAL;
			if (*c == ':') { c++; if ((s.overlap_pct = option_digits(&c)) < 0) return TSDRGPU_EINVAL; }
		}
		if (*c) return TSDRGPU_EINVAL;
	}
	if (!superband_ok(&s)) return TSDRGPU_EINVAL;
	*out = s;
	return TSDRGPU_OK;
}

int tsdrgpu_superband_schedule(const tsdrgpu_superband_t *spec, uint32_t fs, double refreshrate, uint32_t *n, uint32_t *d, int32_t *offsets) {
	if (!spec || !n || !d || !superband_ok(spec) || spec->mode != TSDRGPU_SUPERBAND_COHERENT || fs == 0 || !(refreshrate > 0.0)) return TSDRGPU_EINVAL;
	const double per_frame = floor((double) fs / refreshrate);
	if (!(per_frame >= 1.0) || 10.0 * per_frame > 4294967295.0) return TSDRGPU_EINVAL;
	const uint32_t N = tsdrgpu_fft_getrealsize((uint32_t) (10.0 * per_frame));
	if (N < 16) return TSDRGPU_EINVAL;
	const uint32_t D = 2u * (uint32_t) llround((1.0 - spec->overlap_pct / 100.0) * (double) N / 2.0);
	const int H = spec->hops;
	for (int i = 0; i < H; i++) {
		const double c = (double) (2 * i - (H - 1)) * (double) D / 2.0;       /* exact: D is even */
		const double hz = (double) llround(c * (double) fs / (double) N);
		if (hz < -2147483648.0 || hz > 2147483647.0) return TSDRGPU_EINVAL;
		if (offsets) offsets[i] = (int32_t) hz;
	}
	*n = N; *d = D;
	return TSDRGPU_OK;
}

/* its own small rule, as it takes one optional value: "rl:<sigma>[:<I>]", sigma with at most two fraction digits */
int tsdrgpu_deblur_parse(const char *spec, int *mode, int *sigma_centi, int *iterations) {
	if (!spec || !mode || !sigma_centi || !iterations) return TSDRGPU_EINVAL;
	if (strcmp(spec, "off") == 0) { *mode = TSDRGPU_DEBLUR_OFF; *sigma_centi = 0; *iterations = 0; return TSDRGPU_OK; }
	if (strncmp(spec, "rl:", 3) != 0) return TSDRGPU_EINVAL;
	const char *c = spec + 3;
	int s = option_digits(&c), it = 20;
	if (s < 0) return TSDRGPU_EINVAL;
	s *= 100;
	if (*c == '.') {
		const char *f = ++c;
		int frac = option_digits(&c);
		const int nd = (int) (c - f);
		if (frac < 0 || nd > 2) return TSDRGPU_EINVAL;
		s += nd == 1 ? 10 * frac : frac;
	}
	if (*c == ':') { c++; if ((it = option_digits(&c)) < 0) return TSDRGPU_EINVAL; }
	if (*c || !deblur_ok(TSDRGPU_DEBLUR_RL, s, it)) return TSDRGPU_EINVAL;
	*mode = TSDRGPU_DEBLUR_RL; *sigma_centi = s; *iterations = it;
	return TSDRGPU_OK;
}

/* the deblur taps (definition in tsdrgpu.h) */
int tsdrgpu_deblur_taps(int sigma_centi, float *taps, int *R) {
	if (!deblur_ok(TSDRGPU_DEBLUR_RL, sigma_centi, 1)) return TSDRGPU_EINVAL;
	const int r = (3 * sigma_centi + 99) / 100;
	if (R) *R = r;
	if (!taps) return TSDRGPU_OK;
	const double s = sigma_centi / 100.0;
	double e[2 * TSDRGPU_DEBLUR_MAX_R + 1], sum = 0.0;
	for (int j = -r; j <= r; j++) { e[j + r] = exp(-(double) (j * j) / (2.0 * s * s)); sum += e[j + r]; }
	for (int j = 0; j <= 2 * r; j++) taps[j] = (float) (e[j] / sum);
	return TSDRGPU_OK;
}

/* its own rule, not option_parse's: any number of digits, and the value is rounded from the correctly rounded double */
int tsdrgpu_autogain_ppm(const char *percent) {
	if (!percent) return -1;
	const char *c = percent + strspn(percent, "0123456789");
	if (c == percent) return -1;
	if (*c == '.') { const char *f = c + 1; c = f + strspn(f, "0123456789"); if (c == f) return -1; }
	if (*c) return -1;
	const double v = strtod(percent, NULL);          /* a plain decimal: correctly rounded, as Python's float() */
	if (!(v <= 25.0)) return -1;
	return (int) floor(v * 1e4 + 0.5);
}

static double clampd(double v, double lo, double hi) { return v < lo ? lo : (v > hi ? hi : v); }

int tsdrgpu_channel_taps(const tsdrgpu_channel_t *spec, uint32_t fs, float *taps, int *T) {
	if (!spec || fs == 0 || !channel_valid(spec)) return TSDRGPU_EINVAL;
	const int nt = spec->taps;
	if (T) *T = nt;
	if (!taps) return TSDRGPU_OK;
	const double pi = 3.14159265358979323846, half = 0.5 * (nt - 1), i0b = bessel_i0(TSDRGPU_CHANNEL_BETA);
	const double p0 = clampd((double) spec->pass_lo_hz / fs, -0.5, 0.5), p1 = clampd((double) spec->pass_hi_hz / fs, -0.5, 0.5);
	double lo[1 + TSDRGPU_CHANNEL_MAX_STOPS], hi[1 + TSDRGPU_CHANNEL_MAX_STOPS];
	lo[0] = p0; hi[0] = p1;
	for (int k = 0; k < spec->nstop; k++) {
		lo[1 + k] = clampd(clampd((double) spec->stop_lo_hz[k] / fs, -0.5, 0.5), p0, p1);
		hi[1 + k] = clampd(clampd((double) spec->stop_hi_hz[k] / fs, -0.5, 0.5), p0, p1);
	}
	for (int t = 0; t < nt; t++) {
		const int d = t - (nt - 1) / 2;
		double re = 0.0, im = 0.0, sr = 0.0, si = 0.0;          /* g_pass, then the sum of the g_stop */
		for (int k = 0; k <= spec->nstop; k++) {
			const double a = lo[k], b = hi[k];
			double gr, gi;
			if (d == 0) { gr = b - a; gi = 0.0; }
			else {
				const double den = 2.0 * pi * d;
				gr = (sin(2.0 * pi * b * d) - sin(2.0 * pi * a * d)) / den;
				gi = (cos(2.0 * pi * a * d) - cos(2.0 * pi * b * d)) / den;
			}
			if (k == 0) { re = gr; im = gi; } else { sr += gr; si += gi; }
		}
		const double z = d / half, arg = 1.0 - z * z;
		const double w = bessel_i0(TSDRGPU_CHANNEL_BETA * sqrt(arg > 0.0 ? arg : 0.0)) / i0b;
		taps[2 * t] = (float) (w * (re - sr));
		taps[2 * t + 1] = (float) (w * (im - si));
	}
	return TSDRGPU_OK;
}

/* Stage-angle errors of the reference's FFT.  fft_perform (fft.c:132-165) derives the stage twiddle c_l = (c1, c2)
 * by the half-angle recurrence c2 = sqrt((1-c1)/2), c1 = sqrt((1+c1)/2), which cancels catastrophically for small
 * angles: the angle of c_l is (pi / 2^l) * (1 + eps[l]) with |eps| growing to ~1e-6 at l = 20 and ~1e-4 at l = 23.
 * Replaying the recurrence with the same double arithmetic gives eps exactly; the CUDA FFT can then use the same
 * (wrong) angles so that its results track the reference's instead of the true DFT.  eps[0] = eps[1] = 0. */
void tsdrgpu_fft_reference_eps(int stages, int inverse, double *eps) {
	double c1 = -1.0, c2 = 0.0;
	for (int l = 0; l < stages; l++) {
		if (l == 0) eps[l] = 0.0;                      /* c = (-1, 0): only k = 0 is ever used */
		else {
			const long double ideal = 3.14159265358979323846264338327950288L / (long double) (1ull << l);
			const long double got = atan2l(fabsl((long double) c2), (long double) c1);
			eps[l] = (double) (got / ideal - 1.0L);
		}
		double n2 = sqrt((1.0 - c1) / 2.0);
		if (!inverse) n2 = -n2;
		const double n1 = sqrt((1.0 + c1) / 2.0);
		c1 = n1; c2 = n2;
	}
}

/* Auto video-mode detection (SURVEY section 8f-3), the arithmetic the GUI does on the two autocorrelation plots:
 * PlotVisualizer.java:203-236 takes the index of the first strict maximum of a plot (starting from element 0),
 * Main.java:1301-1303 turns the frame plot's into fps = samplerate / (offset + index), Main.java:1346-1350 + 1041-1043 the
 * line plot's into height = round((frame offset + index) / (line offset + index)), Java's Math.round = floor(x + 0.5). */
static int first_max(const double *v, int n) {
	int best = 0;
	double top = v[0];
	for (int i = 1; i < n; i++) if (v[i] > top) { top = v[i]; best = i; }
	return best;
}
/* the same arithmetic from peak indices that were picked elsewhere (on the device: k_plot_peaks) */
int tsdrgpu_videomode_from_peaks(int frame_offset, int frame_index, int line_offset, int line_index, uint32_t samplerate, double *fps, int *height) {
	const double frame_length = (double) (frame_offset + frame_index), line_length = (double) (line_offset + line_index);
	if (frame_length <= 0 || line_length <= 0) return TSDRGPU_EINVAL;
	if (fps) *fps = (double) (long long) samplerate / frame_length;
	if (height) *height = (int) floor(frame_length / line_length + 0.5);
	return TSDRGPU_OK;
}
int tsdrgpu_detect_videomode(const double *frame_plot, int frame_offset, int frame_len, const double *line_plot, int line_offset, int line_len,
                             uint32_t samplerate, double *fps, int *height, int *frame_index, int *line_index) {
	if (!frame_plot || !line_plot || frame_len <= 0 || line_len <= 0) return TSDRGPU_EINVAL;
	const int fi = first_max(frame_plot, frame_len), li = first_max(line_plot, line_len);
	const double frame_length = (double) (frame_offset + fi), line_length = (double) (line_offset + li);
	if (frame_length <= 0 || line_length <= 0) return TSDRGPU_EINVAL;
	if (fps) *fps = (double) (long long) samplerate / frame_length;
	if (height) *height = (int) floor(frame_length / line_length + 0.5);
	if (frame_index) *frame_index = fi;
	if (line_index) *line_index = li;
	return TSDRGPU_OK;
}
