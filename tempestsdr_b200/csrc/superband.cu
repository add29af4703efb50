// superband.cu -- a22+: the coherent superbandwidth stitch (definition in tsdrgpu.h, tsdrgpu_superb_stitch_coherent).
//
// Per round: H forward N-point transforms (the project's exact-angle plans), then per join, chaining outward from the reference hop:
//   sb_cross          u C into a zeroed N-point buffer (float32, for the integer search) and u C in double (for the refinement), and
//                     per-CTA double partials of sum u |A|^2 and sum u |B|^2; the neighbour's correction is applied as A is loaded
//   N-point inverse   of u C (the same plans), then the first-max argmax -> tau0
//   sb_refine x 2     S at 65 candidates per stage, per-CTA double partials; sb_refine_finish (one CTA) sums them in order and picks
//                     the best (ties to the smallest j); the second finish also forms g and rho from the norm partials
// then sb_assemble writes every bin of the L-point spectrum once (gains, ramps, crossfades, zeros) and one L-point inverse makes y.
// The estimates never leave the device, nothing synchronises the host, and no sum uses atomics: the same inputs give the same bits.
#include "common.cuh"
#include <math.h>

namespace {

constexpr int SB_THREADS = 256;
constexpr unsigned SB_CHUNK = 1024;            // bins of u C per shared-memory chunk of sb_refine
constexpr unsigned SB_MAX_PARTS = 512;         // CTAs of sb_cross and sb_refine (a function of the size only, not of the device)
constexpr int SB_CAND = 65;                    // candidates per refinement stage, j = -32 .. 32

struct SbHop {
	long long c;                                // c_i, centre in stitched bins
	long long kappa0;                           // kappa0 of the hop's own join (its ramp's origin); unused for the reference hop
	const tsdrgpu_superband_est_t *est;         // the hop's correction, NULL for the reference hop
};
struct SbPlan {
	SbHop hop[TSDRGPU_SUPERBAND_MAX_HOPS];
	int H; unsigned long long N, M, L;
	const float2 *X;                            // H spectra X_i = FFT_N(hop_i) / N, N apart, FFT order
};

inline unsigned sb_parts(unsigned long long n) {
	const unsigned long long p = (n + SB_CHUNK - 1) / SB_CHUNK;
	return (unsigned) (p < 1 ? 1 : (p > SB_MAX_PARTS ? SB_MAX_PARTS : p));
}

// e^{-2 pi i x T / (1024 N)} for integers x and T: the product reduced mod 1024 N (a power of two) before the sincospi
__device__ __forceinline__ double2 sb_unit(long long x, long long T, unsigned long long N, double sign) {
	const unsigned long long Q = N << 10, e = ((unsigned long long) x * (unsigned long long) T) & (Q - 1);
	double s, c;
	sincospi(2.0 * ((double) e / (double) Q), &s, &c);
	return make_double2(c, sign * s);
}
__device__ __forceinline__ double2 zmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// hop i's bin at stitched bin kappa, with its correction g e^{-2 pi i (kappa - kappa0) tau^ / N}
__device__ __forceinline__ double2 sb_bin(const SbPlan &P, int i, long long kappa) {
	const SbHop &h = P.hop[i];
	const float2 x = __ldg(P.X + (unsigned long long) i * P.N + ((unsigned long long) (kappa - h.c) & (P.N - 1)));
	double2 v = make_double2((double) x.x, (double) x.y);
	if (h.est) v = zmul(zmul(make_double2(h.est->g_re, h.est->g_im), v), sb_unit(kappa - h.kappa0, h.est->tau_1024, P.N, -1.0));
	return v;
}

// theta_m = pi (m + 1/2) / M: (sin theta, cos theta)
__device__ __forceinline__ double2 sb_theta(unsigned long long m, unsigned long long M) {
	double s, c;
	sincospi((double) (2 * m + 1) / (double) (2 * M), &s, &c);
	return make_double2(s, c);
}

template <class T> __device__ __forceinline__ T sb_block_sum2(T v, T *s) {      // fixed-order block sum of a double2; result in thread 0
	for (int o = 16; o > 0; o >>= 1) { v.x += __shfl_down_sync(0xffffffffu, v.x, o); v.y += __shfl_down_sync(0xffffffffu, v.y, o); }
	if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
	__syncthreads();
	if (threadIdx.x == 0) for (int w = 1; w < (int) (blockDim.x >> 5); w++) { v.x += s[w].x; v.y += s[w].y; }
	return v;
}

// join (a, b): Z[m] = u_m A_m conj(B_m) for m < M and 0 up to N (float32), Cd[m] the same in double, norm partials per CTA
__global__ void __launch_bounds__(SB_THREADS) sb_cross(SbPlan P, int a, int b, long long kappa0, float2 *__restrict__ Z,
                                                      double2 *__restrict__ Cd, double2 *__restrict__ norms) {
	__shared__ double2 s_red[SB_THREADS / 32];
	double2 acc = make_double2(0.0, 0.0);
	for (unsigned long long m = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; m < P.N; m += (unsigned long long) gridDim.x * blockDim.x) {
		if (m >= P.M) { Z[m] = make_float2(0.0f, 0.0f); continue; }
		const long long kappa = kappa0 + (long long) m;
		const double2 A = sb_bin(P, a, kappa), B = sb_bin(P, b, kappa), t = sb_theta(m, P.M);
		const double u = (t.x * t.x) * (t.y * t.y);
		const double2 C = make_double2(u * (A.x * B.x + A.y * B.y), u * (A.y * B.x - A.x * B.y));
		Z[m] = make_float2((float) C.x, (float) C.y);
		Cd[m] = C;
		acc.x += u * (A.x * A.x + A.y * A.y);
		acc.y += u * (B.x * B.x + B.y * B.y);
	}
	acc = sb_block_sum2(acc, s_red);
	if (threadIdx.x == 0) norms[blockIdx.x] = acc;
}

// the candidates' base T and step: stage 1 from the argmax (tau0 mapped to (-N/2, N/2]), stage 2 from stage 1's pick
__device__ __forceinline__ long long sb_base(int stage, const int *idx, const tsdrgpu_superband_est_t *est, unsigned long long N) {
	if (stage == 2) return est->tau_1024;
	long long t = (long long) *idx;
	if ((unsigned long long) t > N / 2) t -= (long long) N;
	return 1024 * t;
}

// S(T_j / 1024) for T_j = base + step (j - 32): each warp owns the candidates j = warp, warp + 8, ...; lanes walk a shared-memory
// chunk of u C; per-CTA partials part[j * gridDim.x + cta]
__global__ void __launch_bounds__(SB_THREADS) sb_refine(const double2 *__restrict__ Cd, unsigned long long M, unsigned long long N, int stage,
                                                       const int *idx, const tsdrgpu_superband_est_t *est, double2 *__restrict__ part) {
	__shared__ double2 s_c[SB_CHUNK];
	constexpr int PER = (SB_CAND + SB_THREADS / 32 - 1) / (SB_THREADS / 32);
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const long long base = sb_base(stage, idx, est, N), step = stage == 2 ? 1 : 32;
	double2 acc[PER];
	#pragma unroll
	for (int q = 0; q < PER; q++) acc[q] = make_double2(0.0, 0.0);
	const unsigned long long chunks = (M + SB_CHUNK - 1) / SB_CHUNK;
	for (unsigned long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
		const unsigned long long m0 = ch * SB_CHUNK, n = (M - m0 < SB_CHUNK) ? M - m0 : SB_CHUNK;
		__syncthreads();
		for (unsigned k = threadIdx.x; k < n; k += blockDim.x) s_c[k] = Cd[m0 + k];
		__syncthreads();
		#pragma unroll
		for (int q = 0; q < PER; q++) {
			const int j = warp + q * (SB_THREADS / 32);
			if (j >= SB_CAND) break;
			const long long T = base + step * (j - 32);
			for (unsigned k = lane; k < n; k += 32) {
				const double2 v = s_c[k], e = sb_unit((long long) (m0 + k), T, N, 1.0);
				acc[q].x += v.x * e.x - v.y * e.y;
				acc[q].y += v.x * e.y + v.y * e.x;
			}
		}
	}
	#pragma unroll
	for (int q = 0; q < PER; q++) {
		const int j = warp + q * (SB_THREADS / 32);
		if (j >= SB_CAND) break;
		double2 v = acc[q];
		for (int o = 16; o > 0; o >>= 1) { v.x += __shfl_down_sync(0xffffffffu, v.x, o); v.y += __shfl_down_sync(0xffffffffu, v.y, o); }
		if (lane == 0) part[(size_t) j * gridDim.x + blockIdx.x] = v;
	}
}

// one CTA: S_j = the partials of candidate j in CTA order; the first largest |S_j| wins.  Stage 1 records tau0 and T1, stage 2 T, g
// and rho (the norm partials summed in CTA order as well)
__global__ void __launch_bounds__(128) sb_refine_finish(const double2 *__restrict__ part, unsigned parts, int stage, const int *idx,
                                                       const double2 *__restrict__ norms, unsigned nnorm, unsigned long long N,
                                                       int hop, int neighbour, long long kappa0, tsdrgpu_superband_est_t *est) {
	__shared__ double2 s_S[SB_CAND];
	const int j = threadIdx.x;
	if (j < SB_CAND) {
		double2 S = make_double2(0.0, 0.0);
		for (unsigned p = 0; p < parts; p++) { const double2 v = part[(size_t) j * parts + p]; S.x += v.x; S.y += v.y; }
		s_S[j] = S;
	}
	__syncthreads();
	if (threadIdx.x != 0) return;
	int best = 0; double bm = -1.0;
	for (int k = 0; k < SB_CAND; k++) { const double m = sqrt(s_S[k].x * s_S[k].x + s_S[k].y * s_S[k].y); if (m > bm) { bm = m; best = k; } }
	const long long T = sb_base(stage, idx, est, N) + (stage == 2 ? 1 : 32) * (long long) (best - 32);
	if (stage == 1) {
		long long t0 = (long long) *idx;
		if ((unsigned long long) t0 > N / 2) t0 -= (long long) N;
		est->hop = hop; est->neighbour = neighbour; est->tau0 = (int32_t) t0; est->kappa0 = (int32_t) kappa0;
		est->tau_1024 = T;
		return;
	}
	double na = 0.0, nb = 0.0;
	for (unsigned p = 0; p < nnorm; p++) { na += norms[p].x; nb += norms[p].y; }
	const double2 S = s_S[best];
	if (nb == 0.0) { est->tau_1024 = 0; est->tau = 0.0; est->g_re = est->g_im = 0.0; est->rho = 0.0; return; }
	est->tau_1024 = T; est->tau = (double) T / 1024.0;
	est->g_re = S.x / nb; est->g_im = S.y / nb;
	const double den = sqrt(na * nb);
	est->rho = den > 0.0 ? bm / den : 0.0;
}

// every bin of the L-point spectrum, in FFT order: the weighted sum of the (one or two) corrected hops that cover it, else 0
__global__ void __launch_bounds__(SB_THREADS) sb_assemble(SbPlan P, float2 *__restrict__ Y) {
	const long long half = (long long) (P.N / 2);
	for (unsigned long long n = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; n < P.L; n += (unsigned long long) gridDim.x * blockDim.x) {
		const long long kappa = n < P.L / 2 ? (long long) n : (long long) n - (long long) P.L;
		double2 y = make_double2(0.0, 0.0);
		for (int i = 0; i < P.H; i++) {
			const long long lo = P.hop[i].c - half;
			if (kappa < lo || kappa >= P.hop[i].c + half) continue;
			double w = 1.0;
			const unsigned long long m_lo = (unsigned long long) (kappa - lo);
			if (i > 0 && m_lo < P.M) { const double2 t = sb_theta(m_lo, P.M); w = t.x * t.x; }          // upper hop of the overlap below
			else if (i + 1 < P.H && kappa >= P.hop[i + 1].c - half) {                                // lower hop of the overlap above
				const double2 t = sb_theta((unsigned long long) (kappa - (P.hop[i + 1].c - half)), P.M); w = t.y * t.y;
			}
			const double2 v = sb_bin(P, i, kappa);
			y.x += w * v.x; y.y += w * v.y;
		}
		Y[n] = make_float2((float) y.x, (float) y.y);
	}
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t) 255; }

}  // namespace

extern "C" int tsdrgpu_superb_stitch_coherent(tsdrgpu_ctx_t *ctx, void *stream_, float *const *d_hops, int nhops, int count_pairs, int d,
                                              float *d_out, tsdrgpu_superband_est_t *d_est) {
	BIND(ctx);
	ARG_TRY(ctx, d_hops && d_out && d_est && (nhops == 2 || nhops == 4 || nhops == 8) && count_pairs >= 16);
	for (int i = 0; i < nhops; i++) ARG_TRY(ctx, d_hops[i] != NULL);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = tsdrgpu_fft_getrealsize((uint32_t) count_pairs), L = N * (unsigned long long) nhops;
	ARG_TRY(ctx, d > 0 && (d & 1) == 0 && (unsigned long long) d >= N / 2 && (unsigned long long) d < N);
	const unsigned long long M = N - (unsigned long long) d;
	const int H = nhops, r = (H - 1) / 2;
	// work memory: slot 1 the H spectra (also the L-point inverse's scratch); slot 2 the N-point transforms' scratch, u C in float and
	// double, the partials, the argmax's partials and its result
	const unsigned pc = sb_parts(N), pr = sb_parts(M);
	const size_t o_z = align256(sizeof(float2) * N), o_cd = o_z + align256(sizeof(float2) * N), o_nrm = o_cd + align256(sizeof(double2) * M),
	             o_part = o_nrm + align256(sizeof(double2) * pc), o_am = o_part + align256(sizeof(double2) * SB_CAND * pr),
	             o_idx = o_am + align256(8 * TSDRGPU_ARGMAX_PARTS), total = o_idx + 256;
	void *s1, *s2; int rc;
	if ((rc = tsdrgpu_scratch(ctx, 1, sizeof(float2) * L, &s1))) return rc;
	if ((rc = tsdrgpu_scratch(ctx, 2, total, &s2))) return rc;
	char *w = (char *) s2;
	float2 *X = (float2 *) s1, *fscr = (float2 *) w, *Z = (float2 *) (w + o_z);
	double2 *Cd = (double2 *) (w + o_cd), *nrm = (double2 *) (w + o_nrm), *part = (double2 *) (w + o_part);
	int *idx = (int *) (w + o_idx);
	SbPlan P; memset(&P, 0, sizeof P);
	P.H = H; P.N = N; P.M = M; P.L = L; P.X = X;
	for (int i = 0; i < H; i++) {
		P.hop[i].c = (long long) (2 * i - (H - 1)) * d / 2;
		if ((rc = tsdrgpu_fft_exact_internal(ctx, stream, reinterpret_cast<const float2 *>(d_hops[i]), X + (size_t) i * N, fscr, N, 0))) return rc;
	}
	auto slot = [&](int b) { return d_est + (b - (b > r ? 1 : 0)); };
	const unsigned gc = pc;
	for (int k = 0; k < H - 1; k++) {
		const int b = k < H - 1 - r ? r + 1 + k : r - 1 - (k - (H - 1 - r)), a = b > r ? b - 1 : b + 1;
		const long long kappa0 = P.hop[b > a ? b : a].c - (long long) (N / 2);
		tsdrgpu_superband_est_t *e = slot(b);
		KL(ctx, "sb_cross", stream, sb_cross<<<gc, SB_THREADS, 0, stream>>>(P, a, b, kappa0, Z, Cd, nrm));
		if ((rc = tsdrgpu_fft_exact_internal(ctx, stream, Z, Z, fscr, N, 1))) return rc;
		if ((rc = tsdrgpu_argmax_mag_internal(ctx, stream, Z, (unsigned) N, w + o_am, idx))) return rc;
		for (int stage = 1; stage <= 2; stage++) {
			KL(ctx, "sb_refine", stream, sb_refine<<<pr, SB_THREADS, 0, stream>>>(Cd, M, N, stage, idx, e, part));
			KL(ctx, "sb_refine_finish", stream, sb_refine_finish<<<1, 128, 0, stream>>>(part, pr, stage, idx, nrm, gc, N, b, a, kappa0, e));
		}
		P.hop[b].est = e; P.hop[b].kappa0 = kappa0;
	}
	unsigned long long want = (L + SB_THREADS - 1) / SB_THREADS, cap = (unsigned long long) ctx->sm_count * 8;
	KL(ctx, "sb_assemble", stream, sb_assemble<<<(unsigned) (want < cap ? want : cap), SB_THREADS, 0, stream>>>(P, reinterpret_cast<float2 *>(d_out)));
	return tsdrgpu_fft_exact_internal(ctx, stream, reinterpret_cast<float2 *>(d_out), reinterpret_cast<float2 *>(d_out), X, L, 1);
}
