// framestage.cu -- a7..a15: the per-frame stage of the reference, for a batch of consecutive frames.
//
// Replaces dsp_post_process (dsp.c:134-239) and everything it calls: dsp_autogain_run (:41-94),
// dsp_timelowpass_run (:22-33), dsp_average_v_h (:96-110), syncdetector_run / findthesweetspot / findbestfit /
// frameratepll (syncdetector.c:26-226), gaussianblur (gaussian.c:18-79).
//
// The reference processes one frame at a time; frames depend on each other only through
//   (1) two scalars of the auto-gain IIR (lastmin/lastmax),
//   (2) the per-pixel temporal IIR (screenbuffer),
//   (3) the sync detector's small integer state.
// So a batch of F frames is processed stage by stage with F as an extra (parallel) grid dimension, the scalar
// recurrences run in one-thread epilogues, and of the sync search only the CHOICE of the strip size walks the frames one
// after another (one 8-CTA cluster): its sliding double-precision sums are replaced, under a per-strip exactness
// certificate, by prefix sums prepared for all frames in parallel (fs_sync_prep / fs_sync below).
// All pixel values and all integer results are bit-identical to the reference: every float/double operation is
// issued as an individual IEEE round-to-nearest instruction in the reference's order; the order-sensitive
// single-precision row/column sums are accumulated in exactly the reference's order (one owner thread per
// row / per column).  Only `snr` (dead in the reference, dsp.c:234) uses tree-ordered double sums.
//
// Every other kernel here is HBM-bound elementwise/reduction work: coalesced (vectorised where aligned) loads, rings in shared
// memory (tensor-map or cp.async copies) for the order-bound row/column sums, grid sized by pixels x frames.
#include "common.cuh"
#include "host_plan.h"
#include <stdlib.h>
#include <cuda_pipeline.h>
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace {

constexpr int FS_SMEM_STRIPS = 2 * 8192 + 2;   // doubles of strip buffers (w + h + 2) the sync search keeps in shared memory at most
constexpr int FS_MM_CHUNKS = 64;       // partial reductions per frame
constexpr int FS_SYNC_THREADS = 512;       // half an SM's registers: it must find room beside the main stream's CTAs

struct SyncState {                      // device-resident syncdetector_t + dsp_autogain_t
	int x_dx, x_vx, x_absvx, x_strip;
	int y_dx, y_vx, y_absvx, y_strip;
	double avg_speed;
	int pll_state;
	float lastmax, lastmin, snr;
};

struct FrameParams {                    // per frame, produced by the auto-gain epilogue
	float lastmin, span, lastmax, snr;
	double mean;
};

// ---------------------------------------------------------------- auto-gain pass 1: min / max / sum (dsp.c:50-61)
template <bool SNR>
__global__ void __launch_bounds__(256) fs_minmax(const float *__restrict__ in, size_t n, float *__restrict__ pmin,
                                                 float *__restrict__ pmax, double *__restrict__ psum) {
	const int f = blockIdx.y;
	const float *src = in + (size_t) f * n;
	float lo = INFINITY, hi = -INFINITY;
	double sum = 0.0;
	// 16-byte loads on the ADDRESS: frames of an odd number of pixels (1481 x 1125, 507 x 525) start at any of the four alignments,
	// so every frame is cut into a scalar head up to the next 16-byte boundary, a float4 body and a scalar tail (min / max and the
	// SNR's tree-ordered sum do not care about the order)
	auto take = [&](float v) {
		if (px_is_marker(v)) return;
		hi = (v > hi) ? v : hi;
		lo = (v < lo) ? v : lo;
		if (SNR) sum += (double) v;
	};
	{
		const size_t gtid = (size_t) blockIdx.x * blockDim.x + threadIdx.x, gsz = (size_t) gridDim.x * blockDim.x;
		const F4Split s(src, n);
		if (gtid < s.head) take(__ldg(src + gtid));
		if (gtid < n - s.tail0) take(__ldg(src + s.tail0 + gtid));
		const float4 *src4 = reinterpret_cast<const float4 *>(src + s.head);
		for (size_t i = gtid; i < s.nbody; i += gsz) {
			const float4 q = __ldg(src4 + i);
			take(q.x); take(q.y); take(q.z); take(q.w);
		}
	}
	__shared__ float s_lo[8], s_hi[8];
	__shared__ double s_sum[8];
	for (int o = 16; o > 0; o >>= 1) {
		const float olo = __shfl_xor_sync(0xffffffffu, lo, o), ohi = __shfl_xor_sync(0xffffffffu, hi, o);
		lo = (olo < lo) ? olo : lo; hi = (ohi > hi) ? ohi : hi;
		if (SNR) sum += __shfl_xor_sync(0xffffffffu, sum, o);
	}
	if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; if (SNR) s_sum[threadIdx.x >> 5] = sum; }
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int w = 1; w < 8; w++) { lo = (s_lo[w] < lo) ? s_lo[w] : lo; hi = (s_hi[w] > hi) ? s_hi[w] : hi; if (SNR) sum += s_sum[w]; }
		pmin[f * gridDim.x + blockIdx.x] = lo; pmax[f * gridDim.x + blockIdx.x] = hi;
		if (SNR) psum[f * gridDim.x + blockIdx.x] = sum;
	}
}

// epilogue: finish the reductions, then run the lastmin/lastmax IIR over the frames in order (dsp.c:63-68)
__global__ void __launch_bounds__(256) fs_autogain_iir(const float *__restrict__ in, size_t n, int nframes, int chunks,
                                                       const float *__restrict__ pmin, const float *__restrict__ pmax,
                                                       const double *__restrict__ psum, bool snr, float norm,
                                                       SyncState *state, FrameParams *params, const float2 *__restrict__ levels) {
	__shared__ float s_lo[1024], s_hi[1024];
	__shared__ double s_mean[1024];
	for (int base = 0; base < nframes; base += 1024) {
		const int cnt = min(1024, nframes - base);
		for (int t = threadIdx.x; t < cnt; t += blockDim.x) {
			const int f = base + t;
			float lo, hi;
			double sum = 0.0;
			if (levels) {                                // clip mode: the selected levels (fs_select_scan)
				lo = levels[f].x; hi = levels[f].y;
				if (snr) for (int c = 0; c < chunks; c++) sum += psum[f * chunks + c];
			} else {
				const float first = in[(size_t) f * n];  // min = max = screenbuffer[0], marker or not (dsp.c:50-51)
				lo = first; hi = first;
				for (int c = 0; c < chunks; c++) {
					const float a = pmin[f * chunks + c], b = pmax[f * chunks + c];
					lo = (a < lo) ? a : lo; hi = (b > hi) ? b : hi;
					if (snr) sum += psum[f * chunks + c];
				}
			}
			s_lo[t] = lo; s_hi[t] = hi; s_mean[t] = sum / (double) n;
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			float lastmax = state->lastmax, lastmin = state->lastmin;
			const float keep = __fsub_rn(1.0f, norm);
			for (int t = 0; t < cnt; t++) {
				lastmax = __fadd_rn(__fmul_rn(keep, lastmax), __fmul_rn(norm, s_hi[t]));
				lastmin = __fadd_rn(__fmul_rn(keep, lastmin), __fmul_rn(norm, s_lo[t]));
				FrameParams p;
				p.lastmin = lastmin; p.lastmax = lastmax;
				p.span = (lastmax == lastmin) ? 1.0f : __fsub_rn(lastmax, lastmin);
				p.mean = s_mean[t]; p.snr = state->snr;
				params[base + t] = p;
			}
			state->lastmax = lastmax; state->lastmin = lastmin;
		}
		__syncthreads();
	}
}

// auto-gain pass 2: normalise (dsp.c:72-79).  Optionally the SNR sums of the same loop.
template <bool SNR>
__global__ void __launch_bounds__(256) fs_normalise(const float *__restrict__ in, float *__restrict__ out, size_t n,
                                                    const FrameParams *__restrict__ params, double *__restrict__ psq,
                                                    double *__restrict__ plin) {
	const int f = blockIdx.y;
	const FrameParams P = params[f];
	const float *src = in + (size_t) f * n;
	float *dst = out + (size_t) f * n;
	double sq = 0.0, lin = 0.0;
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
		const float v = __ldg(src + i);
		dst[i] = px_is_marker(v) ? v : __fdiv_rn(__fsub_rn(v, P.lastmin), P.span);
		if (SNR) { const double d = (double) v - P.mean; sq += d * d; lin += d; }
	}
	if (SNR) {
		__shared__ double s_a[8], s_b[8];
		for (int o = 16; o > 0; o >>= 1) { sq += __shfl_xor_sync(0xffffffffu, sq, o); lin += __shfl_xor_sync(0xffffffffu, lin, o); }
		if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = sq; s_b[threadIdx.x >> 5] = lin; }
		__syncthreads();
		if (threadIdx.x == 0) {
			for (int w = 1; w < 8; w++) { sq += s_a[w]; lin += s_b[w]; }
			psq[f * gridDim.x + blockIdx.x] = sq; plin[f * gridDim.x + blockIdx.x] = lin;
		}
	}
}

__global__ void fs_snr_finish(int nframes, int chunks, size_t n, const double *__restrict__ psq, const double *__restrict__ plin,
                              FrameParams *params, SyncState *state) {
	for (int f = threadIdx.x; f < nframes; f += blockDim.x) {
		double sq = 0.0, lin = 0.0;
		for (int c = 0; c < chunks; c++) { sq += psq[f * chunks + c]; lin += plin[f * chunks + c]; }
		const double stdev = sqrt((sq - lin * lin / (double) n) / (double) (n - 1));   // dsp.c:91
		params[f].snr = (float) (params[f].mean / stdev);
		if (f == nframes - 1) state->snr = params[f].snr;
	}
}

// ---------------------------------------------------------------- clip-mode auto-gain levels (tsdrgpu.h, TSDRGPU_AG_CLIP)
// Exact per-frame order statistics by radix select on order-preserving 32-bit keys, three digit rounds of 11 / 11 / 10 bits.
// Each round: fs_select_hist counts (per CTA in shared memory, merged with one global atomic per non-empty bin) the valid pixels
// whose key matches the prefix found so far, by their next digit; fs_select_scan (one CTA per frame) then fixes that digit of
// the lo and the hi target.  Round 1 has one histogram for both targets (no prefix yet) and its total is n_v; later rounds have
// one per target, or one shared when both targets still have the same prefix.
constexpr int SEL_BINS = 2048;                        // 2^11

struct SelState {                                     // per frame, between the rounds
	unsigned prefix[2];                               // key bits fixed so far (lo, hi target), zero below
	unsigned rank[2];                                 // rank of the target among the keys with that prefix
	unsigned long long nvalid;
};

__device__ __forceinline__ unsigned sel_key(float v) {
	const unsigned u = __float_as_uint(v);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float sel_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// round R's digit: bits [shift, shift + width) of the key; the prefix to match is everything above it
template <int R> struct SelDigit {
	static constexpr int shift = R == 1 ? 21 : (R == 2 ? 10 : 0);
	static constexpr int prefix_shift = R == 1 ? 0 : (R == 2 ? 21 : 10);     // bits above the digit (round 1 has no prefix)
};

// one increment per group of lanes with the same bin (frames of a narrow range put most pixels of a warp into one bin);
// bin == ~0u counts nothing.  All 32 lanes of the warp must make the call (warp-uniform control flow around it).
__device__ __forceinline__ void sel_count(unsigned *h, unsigned bin) {
	if (!__any_sync(0xffffffffu, bin != ~0u)) return;      // rounds 2 and 3: most warps hold no candidate at all
	const unsigned peers = __match_any_sync(0xffffffffu, bin);
	if (bin != ~0u && (threadIdx.x & 31) == (unsigned) (__ffs(peers) - 1)) atomicAdd(h + bin, (unsigned) __popc(peers));
}

template <int R, bool SNR>
__global__ void __launch_bounds__(256) fs_select_hist(const float *__restrict__ in, size_t n, const SelState *__restrict__ sel,
                                                      unsigned *__restrict__ hist, double *__restrict__ psum) {
	constexpr int NB = R == 1 ? SEL_BINS : 2 * SEL_BINS;
	__shared__ unsigned s_h[NB];
	const int f = blockIdx.y;
	const float *src = in + (size_t) f * n;
	unsigned plo = 0, phi = 0;
	if (R > 1) {
		const SelState S = sel[f];
		if (S.nvalid == 0) return;                     // levels already fixed (pixel 0); uniform over the CTA
		plo = S.prefix[0] >> SelDigit<R>::prefix_shift; phi = S.prefix[1] >> SelDigit<R>::prefix_shift;
	}
	for (int b = threadIdx.x; b < NB; b += blockDim.x) s_h[b] = 0;
	__syncthreads();
	double sum = 0.0;
	auto take = [&](float v, bool inside) {           // every lane calls this; `inside` = v is a pixel of the frame
		const bool marker = px_is_marker(v);
		if (SNR && inside && !marker) sum += (double) v;   // the SNR's mean keeps the reference's terms (NaN included, dsp.c:58-60)
		unsigned bin = ~0u;
		if (inside && !marker && v == v) {            // px_valid(v), reusing the marker test above
			const unsigned k = sel_key(v);
			if (R == 1) bin = k >> 21;
			else {
				const unsigned p = k >> SelDigit<R>::prefix_shift;
				const unsigned d = (k >> SelDigit<R>::shift) & (R == 3 ? 1023u : 2047u);
				if (p == plo) bin = d;
				else if (p == phi) bin = SEL_BINS + d;
			}
		}
		sel_count(s_h, bin);
	};
	{   // 16-byte loads on the address, scalar head and tail (as fs_minmax); loop trip counts are warp-uniform
		const size_t gtid = (size_t) blockIdx.x * blockDim.x + threadIdx.x, gsz = (size_t) gridDim.x * blockDim.x;
		const size_t lane = threadIdx.x & 31;
		const F4Split s(src, n);
		take(gtid < s.head ? __ldg(src + gtid) : 0.0f, gtid < s.head);
		take(gtid < n - s.tail0 ? __ldg(src + s.tail0 + gtid) : 0.0f, gtid < n - s.tail0);
		const float4 *src4 = reinterpret_cast<const float4 *>(src + s.head);
		for (size_t i0 = gtid - lane; i0 < s.nbody; i0 += gsz) {
			const size_t i = i0 + lane;
			const bool inside = i < s.nbody;
			const float4 q = inside ? __ldg(src4 + i) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			take(q.x, inside); take(q.y, inside); take(q.z, inside); take(q.w, inside);
		}
	}
	__syncthreads();
	unsigned *g = hist + (size_t) f * 2 * SEL_BINS;
	for (int b = threadIdx.x; b < NB; b += blockDim.x) if (s_h[b]) atomicAdd(g + b, s_h[b]);
	if (SNR && R == 1) {
		__shared__ double s_sum[8];
		for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
		if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = sum;
		__syncthreads();
		if (threadIdx.x == 0) {
			for (int w = 1; w < 8; w++) sum += s_sum[w];
			psum[f * gridDim.x + blockIdx.x] = sum;
		}
	}
}

// the bin holding rank r of a 2048-bin histogram (256 threads, 8 bins each); returns the bin, *below = count of smaller bins
__device__ unsigned sel_find(const unsigned *h, unsigned r, unsigned *below) {
	__shared__ unsigned s_warp[8];
	__shared__ unsigned s_bin, s_below;
	unsigned c[8], local = 0;
	for (int j = 0; j < 8; j++) { c[j] = h[threadIdx.x * 8 + j]; local += c[j]; }
	unsigned incl = local;
	for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= (unsigned) o) incl += y; }
	if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = incl;
	__syncthreads();
	unsigned base = 0;
	for (int w = 0; w < (int) (threadIdx.x >> 5); w++) base += s_warp[w];
	unsigned start = base + incl - local;
	if (r >= start && r < start + local) {             // exactly one thread owns rank r
		for (int j = 0; j < 8; j++) {
			if (r < start + c[j]) { s_bin = threadIdx.x * 8 + j; s_below = start; break; }
			start += c[j];
		}
	}
	__syncthreads();
	*below = s_below;
	const unsigned bin = s_bin;
	__syncthreads();                                   // s_bin / s_warp are reused by the next call
	return bin;
}

template <int R>
__global__ void __launch_bounds__(256) fs_select_scan(const float *__restrict__ in, size_t n, int ppm, SelState *sel,
                                                      unsigned *hist, float2 *__restrict__ levels) {
	const int f = blockIdx.x;
	unsigned *g = hist + (size_t) f * 2 * SEL_BINS;
	SelState S;
	if (R == 1) {
		__shared__ unsigned long long s_total;
		if (threadIdx.x == 0) s_total = 0;
		__syncthreads();
		unsigned long long part = 0;
		for (int b = threadIdx.x; b < SEL_BINS; b += blockDim.x) part += g[b];
		atomicAdd(&s_total, part);
		__syncthreads();
		S.nvalid = s_total;
		S.prefix[0] = S.prefix[1] = 0;
		const unsigned long long k = S.nvalid * (unsigned long long) ppm / 1000000ull;
		S.rank[0] = (unsigned) k; S.rank[1] = (unsigned) (S.nvalid - 1 - k);
	} else S = sel[f];
	if (S.nvalid == 0) {
		if (R == 1 && threadIdx.x == 0) {
			const float first = in[(size_t) f * n];    // min = max = screenbuffer[0] (dsp.c:50-51)
			levels[f] = make_float2(first, first);
			sel[f] = S;
		}
	} else {
		constexpr int shift = SelDigit<R>::shift;
		const bool same = R == 1 || S.prefix[0] == S.prefix[1];
		for (int t = 0; t < 2; t++) {
			unsigned below;
			const unsigned d = sel_find(g + ((same || t == 0) ? 0 : SEL_BINS), S.rank[t], &below);
			S.prefix[t] |= d << shift; S.rank[t] -= below;
		}
		if (threadIdx.x == 0) {
			sel[f] = S;
			if (R == 3) levels[f] = make_float2(sel_value(S.prefix[0]), sel_value(S.prefix[1]));
		}
	}
	__syncthreads();
	for (int b = threadIdx.x; b < 2 * SEL_BINS; b += blockDim.x) g[b] = 0;      // clean for the next round / batch
}

// ---------------------------------------------------------------- temporal IIR over the batch (dsp.c:22-33)
// one thread per pixel carries the screen value through the F frames in order
__global__ void __launch_bounds__(256) fs_timelowpass(const float *__restrict__ in, float *out, float *screen,
                                                      size_t n, int nframes, float coeff, double fresh) {
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
		float s = screen[i];
		#pragma unroll 4
		for (int f = 0; f < nframes; f++) {
			const float v = __ldg(in + (size_t) f * n + i);
			const float old = __fmul_rn(s, coeff);
			s = __double2float_rn(__dadd_rn((double) old, __dmul_rn((double) v, fresh)));
			out[(size_t) f * n + i] = s;
		}
		screen[i] = s;
	}
}

// the normalised pixel v (dsp.c:72-79).  The quotient is formed for markers too and then dropped: without a branch around the
// division, the compiler keeps the divisor's reciprocal across unrolled pixels and their loads in flight together.
__device__ __forceinline__ float norm_px(float x, float lastmin, float span) {
	const float q = __fdiv_rn(__fsub_rn(x, lastmin), span);
	return px_is_marker(x) ? x : q;
}
__device__ __forceinline__ bool finite_px(float s) { return (__float_as_uint(s) & 0x7f800000u) != 0x7f800000u; }
// the values of v for which a motion blur of 0 does not pass v through unchanged (fs_collapse_tiles<true>): NaN, +-inf, -0.0f
__device__ __forceinline__ unsigned norm_px_bad(float v) { return !finite_px(v) | (__float_as_uint(v) == 0x80000000u); }

// auto-gain pass 2 fused with the temporal IIR (default stage order): out[f][i] = screen_f[i] where
// screen_f = lowpass(screen_{f-1}, normalise_f(in[f][i])).  Saves one write + one read of the normalised frames.
// REDO: after the collapse that normalised on load (motion blur 0, fs_collapse_tiles<true> / fs_collapse<true>), `out` already holds
// v.  A thread whose start-of-batch screen values are finite, in a batch whose certificate word is clear, then only carries the
// last frame into the screen (out[F-1] == screen_F); every other thread runs the literal update for its pixels, and one whose
// screen was not finite sets the word, so that the gated collapse after this kernel redoes the sums from `out`.
template <bool VEC, bool REDO>
__global__ void __launch_bounds__(256) fs_norm_lowpass(const float *__restrict__ in, float *out, float *screen, size_t n, int nframes,
                                                       const FrameParams *__restrict__ params, float coeff, double fresh, unsigned *cert) {
	extern __shared__ float2 s_par[];                    // (lastmin, span) per frame
	for (int f = threadIdx.x; f < nframes; f += blockDim.x) s_par[f] = make_float2(params[f].lastmin, params[f].span);
	__syncthreads();
	const bool redo_all = REDO && *cert != 0;
	int set = 0;                                         // REDO: a screen value was not finite
	if (VEC) {                                           // 4 pixels per thread, 16-byte loads and stores (n % 4 == 0, aligned bases: checked by the host)
		const size_t n4 = n >> 2;
		for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t) gridDim.x * blockDim.x) {
			float4 sc = reinterpret_cast<float4 *>(screen)[i];
			if (REDO && !redo_all) {
				if (finite_px(sc.x) && finite_px(sc.y) && finite_px(sc.z) && finite_px(sc.w)) {
					reinterpret_cast<float4 *>(screen)[i] = reinterpret_cast<const float4 *>(out + (size_t) (nframes - 1) * n)[i];
					continue;
				}
				set = 1;
			}
			float s4[4] = {sc.x, sc.y, sc.z, sc.w};
			for (int f0 = 0; f0 < nframes; f0 += 4) {         // 4 frames of loads in flight, then the ordered updates
				float4 q4[4];
				#pragma unroll
				for (int g = 0; g < 4; g++) if (f0 + g < nframes) q4[g] = __ldg(reinterpret_cast<const float4 *>(in + (size_t) (f0 + g) * n) + i);
				#pragma unroll
				for (int g = 0; g < 4; g++) {
					const int f = f0 + g;
					if (f >= nframes) break;
					const float raw[4] = {q4[g].x, q4[g].y, q4[g].z, q4[g].w};
					const float2 p = s_par[f];
					#pragma unroll
					for (int u = 0; u < 4; u++) {
						const float v = norm_px(raw[u], p.x, p.y);
						const float old = __fmul_rn(s4[u], coeff);
						s4[u] = __double2float_rn(__dadd_rn((double) old, __dmul_rn((double) v, fresh)));
					}
					reinterpret_cast<float4 *>(out + (size_t) f * n)[i] = make_float4(s4[0], s4[1], s4[2], s4[3]);
				}
			}
			reinterpret_cast<float4 *>(screen)[i] = make_float4(s4[0], s4[1], s4[2], s4[3]);
		}
	} else {
		// frames of an odd number of pixels (1481 x 1125, 507 x 525) start at every alignment: one pixel per thread, and because a
		// thread then has only 4 bytes per frame to ask for, SIXTEEN frames of loads are in flight before the ordered updates run
		// (with four the kernel falls far behind the 16-byte path in the share of the HBM roofline it reaches)
		for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
			float s = screen[i];
			if (REDO && !redo_all) {
				if (finite_px(s)) { screen[i] = out[(size_t) (nframes - 1) * n + i]; continue; }
				set = 1;
			}
			for (int f0 = 0; f0 < nframes; f0 += 16) {
				float raw[16];
				#pragma unroll
				for (int g = 0; g < 16; g++) if (f0 + g < nframes) raw[g] = ldg_stream_f1(in + (size_t) (f0 + g) * n + i);
				#pragma unroll
				for (int g = 0; g < 16; g++) {
					const int f = f0 + g;
					if (f >= nframes) break;
					const float2 p = s_par[f];
					const float v = norm_px(raw[g], p.x, p.y);
					const float old = __fmul_rn(s, coeff);
					s = __double2float_rn(__dadd_rn((double) old, __dmul_rn((double) v, fresh)));
					out[(size_t) f * n + i] = s;
				}
			}
			screen[i] = s;
		}
	}
	if (REDO && __syncthreads_or(set) && threadIdx.x == 0) atomicOr(cert, 1u);
}

// ---------------------------------------------------------------- row / column collapse (dsp.c:96-110)
// Sequential single-precision accumulation in raster order == per column: top to bottom; per row: left to right.
// grid.x = column CTAs followed by row CTAs; grid.y = frame.
// Both sums are chains of dependent additions (1125 per column, 740 per row at cfg2) that may not be re-associated, so
// the only parallelism is across chains; what has to be hidden is the memory latency inside a chain.  A CTA streams its
// slab of the frame through a ring of stages in shared memory (the next stages are in flight while one is summed), the
// owner threads read their operands from shared memory.  The frame is read twice; the second read comes from L2 only if it
// follows the first closely (see fs_collapse_tiles).
//
// fs_collapse_tiles: rows on 16-byte boundaries (w % 4 == 0, aligned base).  The ring is filled by 2-D tensor copies
// (cp.async.bulk.tensor, one request per box of the 3-D tensor map x = column, y = row, z = frame), issued by one thread and
// counted in bytes on the stage's mbarrier: nobody spends issue slots on copies or their addresses, and every thread owns a chain.
// A CTA is one warp:
//   column CTA: 32 columns x all rows, boxes of 32 columns x 64 rows (8 KB, 8 stages), lane c owns column c;
//   row CTA:    32 rows x all columns, boxes of 32 columns (128 B, 128-byte swizzle) x 32 rows (4 KB, 8 stages), lane r owns row r.
// Narrow CTAs make many per frame (24 + 36 at cfg2), so the resident ones (3 per SM by shared memory) cover ~7 frames at a time:
// a column CTA sweeps its frame top to bottom while the row CTAs of that frame run, so less is read in between and more of the
// second read is served by the L2.
// With CTAs of 128 columns / 128 rows (15 per frame, ~35 frames open) the second read mostly missed: 0.157 against 0.119 ms per
// 64-frame cfg2 launch on an H100 SXM at a 400 W power limit (smaller rings, 4 CTAs per SM: 0.121).
// The tensor map fills what lies beyond the frame's last column / row with zeros; those slots never enter a chain (x + 0.0f is
// not x when x = -0.0f): the loops are bounded by the columns / rows that exist.
constexpr int CT_THREADS = 32;
constexpr int CT_COLS = 32, CT_CROWS = 64, CT_CSTAGES = 8;      // column CTA box: 8 KB
constexpr int CT_RCOLS = 32, CT_ROWS = 32, CT_RSTAGES = 8;      // row CTA box: 4 KB
constexpr int CT_RING = CT_CSTAGES * CT_COLS * CT_CROWS * 4 > CT_RSTAGES * CT_RCOLS * CT_ROWS * 4 ? CT_CSTAGES * CT_COLS * CT_CROWS * 4
                                                                                                  : CT_RSTAGES * CT_RCOLS * CT_ROWS * 4;
constexpr int CT_SMEM = CT_RING + 1024;                 // + slack to put the ring on the 1024-byte boundary the swizzle repeats on

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
	asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
	             :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_box3(unsigned dst_smem, const CUtensorMap *map, int x, int y, int z, unsigned bar) {
	asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
	             :: "r"(dst_smem), "l"(reinterpret_cast<unsigned long long>(map)), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
}

__device__ __forceinline__ void tma_store_box3(const CUtensorMap *map, int x, int y, int z, unsigned src_smem) {
	asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
	             :: "l"(reinterpret_cast<unsigned long long>(map)), "r"(x), "r"(y), "r"(z), "r"(src_smem) : "memory");
	asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N> __device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory"); }

// ---- normalise on load (default stage order, motion blur 0)
// With motion blur c = 0 the temporal IIR is the identity: fs_norm_lowpass forms s' = (double) (s * c) + (double) v rounded to
// float, and s * c is a signed zero for every finite screen value s, so s' == v bit for bit unless v is NaN, +-inf or -0.0f
// (+0.0f + -0.0f is +0.0f).  The collapse then normalises the raw pixels as it loads them, sums v, and its column CTAs (which see
// every pixel once) write v as the low-passed frames and set the batch's certificate word when any v of the batch is one of those
// values.  fs_norm_lowpass<REDO> and the gated collapse after it redo the batch literally when the word is set.

// NORM = false: the literal collapse of `cmap`/`rmap` (one warp per CTA); with `gate`, only when *gate is set.
// NORM = true: the collapse of the raw frames normalised on load (CT_NTHREADS per CTA).  All warps normalise each landed box in
// place (the division makes that issue-bound for one warp), then warp 0's owner lanes sum it as above; a column CTA stores
// its normalised box through `smap` (the low-passed frames) and checks it for the certificate.  A slot is refilled two stages
// after its store was issued, once the store has read it.
constexpr int CT_NTHREADS = 128;
template <bool NORM>
__global__ void __launch_bounds__(NORM ? CT_NTHREADS : CT_THREADS) fs_collapse_tiles(const __grid_constant__ CUtensorMap cmap, const __grid_constant__ CUtensorMap rmap,
                                                                                     const __grid_constant__ CUtensorMap smap, int w, int h,
                                                                                     float *__restrict__ wbuf, float *__restrict__ hbuf, int col_ctas,
                                                                                     const unsigned *gate, const FrameParams *__restrict__ params,
                                                                                     unsigned *cert) {
	if (!NORM && gate && *gate == 0) return;             // the batch's normalise-on-load pass was exact
	extern __shared__ unsigned char ct_smem[];
	__shared__ __align__(8) unsigned long long bars[CT_CSTAGES > CT_RSTAGES ? CT_CSTAGES : CT_RSTAGES];
	const unsigned raw = (unsigned) __cvta_generic_to_shared(ct_smem), ring_a = (raw + 1023u) & ~1023u;
	float *ring = reinterpret_cast<float *>(ct_smem + (ring_a - raw));
	const unsigned bar_a = (unsigned) __cvta_generic_to_shared(bars);
	const int f = blockIdx.y, tid = threadIdx.x;
	const bool colcta = (int) blockIdx.x < col_ctas;
	const bool store = NORM && colcta;
	const int stages = colcta ? CT_CSTAGES : CT_RSTAGES;
	const int lead = store ? stages - 2 : stages - 1;    // boxes in flight ahead of the one being summed
	const unsigned box_bytes = colcta ? CT_COLS * CT_CROWS * 4 : CT_RCOLS * CT_ROWS * 4;
	const int x0 = colcta ? blockIdx.x * CT_COLS : 0, y0 = colcta ? 0 : ((int) blockIdx.x - col_ctas) * CT_ROWS;
	const int nit = colcta ? (h + CT_CROWS - 1) / CT_CROWS : (w + CT_RCOLS - 1) / CT_RCOLS;
	float lastmin = 0.0f, span = 1.0f;
	if (NORM) { lastmin = params[f].lastmin; span = params[f].span; }
	if (tid == 0) {
		for (int st = 0; st < stages; st++) mbar_init(bar_a + 8 * st, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	auto issue = [&](int it) {                           // thread 0 only
		if (it >= nit) return;
		const int slot = it % stages;
		const unsigned bar = bar_a + 8 * slot;
		mbar_expect_tx(bar, box_bytes);                  // out-of-bounds fill counts: always the whole box
		if (colcta) tma_box3(ring_a + slot * box_bytes, &cmap, x0, it * CT_CROWS, f, bar);
		else tma_box3(ring_a + slot * box_bytes, &rmap, it * CT_RCOLS, y0, f, bar);
	};
	if (tid == 0) for (int st = 0; st < lead; st++) issue(st);
	float acc = 0.0f;
	unsigned bad = 0;
	// one thread of warp 0 per column / row of the CTA
	const bool owner = tid < CT_COLS && (colcta ? (tid < w - x0) : (tid < h - y0));
	for (int it = 0; it < nit; it++) {
		__syncthreads();                                 // everybody is done with the slot of stage it-1: it may be refilled
		if (tid == 0) {
			if (store) tma_store_wait_read<1>();         // the store of stage it-2 has read the slot about to be refilled
			issue(it + lead);
		}
		const int slot = it % stages;
		mbar_wait(bar_a + 8 * slot, (unsigned) ((it / stages) & 1));
		if (NORM) {
			float *box = ring + slot * (box_bytes / 4);
			if (store) {
				constexpr int K = CT_COLS * CT_CROWS / CT_NTHREADS;
				const int rows = min(CT_CROWS, h - it * CT_CROWS), cols = min(CT_COLS, w - x0);
				float x[K];
				#pragma unroll
				for (int k = 0; k < K; k++) x[k] = box[tid + k * CT_NTHREADS];
				#pragma unroll
				for (int k = 0; k < K; k++) {
					const int e = tid + k * CT_NTHREADS;
					const float v = norm_px(x[k], lastmin, span);
					box[e] = v;
					if (e / CT_COLS < rows && e % CT_COLS < cols) bad |= norm_px_bad(v);      // pixels of the frame only
				}
			} else {                                     // the swizzle permutes a row's chunks: in place it does not matter
				constexpr int K = CT_RCOLS * CT_ROWS / CT_NTHREADS;
				float x[K];
				#pragma unroll
				for (int k = 0; k < K; k++) x[k] = box[tid + k * CT_NTHREADS];
				#pragma unroll
				for (int k = 0; k < K; k++) box[tid + k * CT_NTHREADS] = norm_px(x[k], lastmin, span);
			}
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // the box's generic writes before the bulk copies' access
			__syncthreads();
			if (store && tid == 0) tma_store_box3(&smap, x0, it * CT_CROWS, f, ring_a + slot * box_bytes);   // clipped to the frame
		}
		if (!owner) continue;
		if (colcta) {
			const float *buf = ring + slot * (CT_COLS * CT_CROWS) + tid;
			const int rows = min(CT_CROWS, h - it * CT_CROWS);
			if (rows == CT_CROWS) {
				#pragma unroll
				for (int r = 0; r < CT_CROWS; r++) acc = __fadd_rn(acc, buf[r * CT_COLS]);
			} else for (int r = 0; r < rows; r++) acc = __fadd_rn(acc, buf[r * CT_COLS]);
		} else {
			// row tid is 128 B at tid * 128; its 16-byte chunk c sits at chunk position c ^ (tid & 7) (128-byte swizzle), so the
			// eight lanes of a quarter-warp read eight different chunks: LDS.128 without bank conflicts
			const float4 *row = reinterpret_cast<const float4 *>(ring + slot * (CT_RCOLS * CT_ROWS) + tid * CT_RCOLS);
			const int chunks = min(CT_RCOLS, w - it * CT_RCOLS) >> 2, sw = tid & 7;
			if (chunks == CT_RCOLS / 4) {
				#pragma unroll
				for (int c = 0; c < CT_RCOLS / 4; c++) {
					const float4 q = row[c ^ sw];
					acc = __fadd_rn(acc, q.x); acc = __fadd_rn(acc, q.y); acc = __fadd_rn(acc, q.z); acc = __fadd_rn(acc, q.w);
				}
			} else for (int c = 0; c < chunks; c++) {
				const float4 q = row[c ^ sw];
				acc = __fadd_rn(acc, q.x); acc = __fadd_rn(acc, q.y); acc = __fadd_rn(acc, q.z); acc = __fadd_rn(acc, q.w);
			}
		}
	}
	if (owner) { if (colcta) wbuf[(size_t) f * w + x0 + tid] = acc; else hbuf[(size_t) f * h + y0 + tid] = acc; }
	if (store) {                                         // uniform over the CTA
		if (__syncthreads_or(bad) && tid == 0) atomicOr(cert, 1u);
		if (tid == 0) tma_store_wait_read<0>();          // the ring stays until the last store has read it
	}
}

// Rows at any alignment (odd widths: 1481, 507): every pixel copied with a 4-byte cp.async through a 4-stage ring.
//   column CTA: 128 columns x all rows, stages of 16 rows, thread c owns column c;
//   row CTA:    32 rows x all columns, stages of 64 columns (pitch 65: conflict-free), lane r of warp 0 owns row r.
constexpr int CL_COLS = 128, CL_CROWS = 16, CL_ROWS = 32, CL_RCOLS = 64, CL_STAGES = 4;
constexpr int CL_RPITCH = CL_RCOLS + 1;
constexpr int CL_SMEM_FLOATS = CL_STAGES * (CL_CROWS * CL_COLS > CL_ROWS * CL_RPITCH ? CL_CROWS * CL_COLS : CL_ROWS * CL_RPITCH);
// NORM and `gate` as fs_collapse_tiles: with NORM every thread normalises the pixels it copied once they have landed, in place, and
// in column CTAs also writes them to the low-passed frames `t2` and checks them for the certificate.
template <bool NORM>
__global__ void __launch_bounds__(256) fs_collapse(const float *__restrict__ in, int w, int h, float *__restrict__ wbuf,
                                                   float *__restrict__ hbuf, int col_ctas, const unsigned *gate,
                                                   const FrameParams *__restrict__ params, float *__restrict__ t2, unsigned *cert) {
	if (!NORM && gate && *gate == 0) return;             // the batch's normalise-on-load pass was exact
	__shared__ __align__(16) float ring[CL_SMEM_FLOATS];
	const int f = blockIdx.y, tid = threadIdx.x;
	const float *src = in + (size_t) f * w * h;
	float lastmin = 0.0f, span = 1.0f;
	if (NORM) { lastmin = params[f].lastmin; span = params[f].span; }
	if ((int) blockIdx.x < col_ctas) {
		const int x0 = blockIdx.x * CL_COLS, cols = min(CL_COLS, w - x0);
		const int nit = (h + CL_CROWS - 1) / CL_CROWS;
		auto issue = [&](int it) {
			if (it < nit) {
				float *dst = ring + (it % CL_STAGES) * (CL_CROWS * CL_COLS);
				const int y0 = it * CL_CROWS, rows = min(CL_CROWS, h - y0);
				const float *s0 = src + (size_t) y0 * w + x0;
				for (int idx = tid; idx < rows * CL_COLS; idx += 256) {
					const int r = idx / CL_COLS, c = idx % CL_COLS;
					if (c < cols) __pipeline_memcpy_async(dst + idx, s0 + r * w + c, sizeof(float));
				}
			}
			__pipeline_commit();
		};
		for (int st = 0; st < CL_STAGES - 1; st++) issue(st);
		float acc = 0.0f;
		unsigned bad = 0;
		for (int it = 0; it < nit; it++) {
			__pipeline_wait_prior(CL_STAGES - 2);
			if (NORM) {                                  // this thread's copies of stage `it` have landed
				float *dst = ring + (it % CL_STAGES) * (CL_CROWS * CL_COLS);
				const int y0 = it * CL_CROWS, rows = min(CL_CROWS, h - y0);
				float *t0 = t2 + (size_t) f * w * h + (size_t) y0 * w + x0;
				for (int idx = tid; idx < rows * CL_COLS; idx += 256) {
					const int r = idx / CL_COLS, c = idx % CL_COLS;
					if (c < cols) {
						const float v = norm_px(dst[idx], lastmin, span);
						dst[idx] = v; t0[r * w + c] = v;
						bad |= norm_px_bad(v);
					}
				}
			}
			__syncthreads();                             // stage `it` has landed; the buffer of stage it-1 is free again
			issue(it + CL_STAGES - 1);
			if (tid < cols) {
				const float *buf = ring + (it % CL_STAGES) * (CL_CROWS * CL_COLS) + tid;
				const int rows = min(CL_CROWS, h - it * CL_CROWS);
				if (rows == CL_CROWS) {
					#pragma unroll
					for (int r = 0; r < CL_CROWS; r++) acc = __fadd_rn(acc, buf[r * CL_COLS]);
				} else for (int r = 0; r < rows; r++) acc = __fadd_rn(acc, buf[r * CL_COLS]);
			}
		}
		if (tid < cols) wbuf[(size_t) f * w + x0 + tid] = acc;
		if (NORM && __syncthreads_or(bad) && tid == 0) atomicOr(cert, 1u);
		return;
	}
	const int y0 = ((int) blockIdx.x - col_ctas) * CL_ROWS, rows = min(CL_ROWS, h - y0);
	const int nit = (w + CL_RCOLS - 1) / CL_RCOLS;
	auto issue = [&](int it) {
		if (it < nit) {
			float *dst = ring + (it % CL_STAGES) * (CL_ROWS * CL_RPITCH);
			const int c0 = it * CL_RCOLS, cols = min(CL_RCOLS, w - c0);
			const float *s0 = src + (size_t) y0 * w + c0;
			for (int idx = tid; idx < rows * CL_RCOLS; idx += 256) {
				const int r = idx / CL_RCOLS, c = idx % CL_RCOLS;
				if (c < cols) __pipeline_memcpy_async(dst + r * CL_RPITCH + c, s0 + r * w + c, sizeof(float));
			}
		}
		__pipeline_commit();
	};
	for (int st = 0; st < CL_STAGES - 1; st++) issue(st);
	float acc = 0.0f;
	for (int it = 0; it < nit; it++) {
		__pipeline_wait_prior(CL_STAGES - 2);
		if (NORM) {
			float *dst = ring + (it % CL_STAGES) * (CL_ROWS * CL_RPITCH);
			const int cols = min(CL_RCOLS, w - it * CL_RCOLS);
			for (int idx = tid; idx < rows * CL_RCOLS; idx += 256) {
				const int r = idx / CL_RCOLS, c = idx % CL_RCOLS;
				if (c < cols) dst[r * CL_RPITCH + c] = norm_px(dst[r * CL_RPITCH + c], lastmin, span);
			}
		}
		__syncthreads();
		issue(it + CL_STAGES - 1);
		if (tid < rows) {
			const float *buf = ring + (it % CL_STAGES) * (CL_ROWS * CL_RPITCH) + tid * CL_RPITCH;
			const int cols = min(CL_RCOLS, w - it * CL_RCOLS);
			if (cols == CL_RCOLS) {
				#pragma unroll 16
				for (int c = 0; c < CL_RCOLS; c++) acc = __fadd_rn(acc, buf[c]);
			} else for (int c = 0; c < cols; c++) acc = __fadd_rn(acc, buf[c]);
		}
	}
	if (tid < rows) hbuf[(size_t) f * h + y0 + tid] = acc;
}

// ---------------------------------------------------------------- sync search (syncdetector.c:26-153, gaussian.c)
struct SweetIn { int size, minsize; double lowpass; };

// exact 5-tap circular blur, out of place (gaussian.c:18-79); n < 5 replayed literally by one thread
__device__ void blur_strip(const float *__restrict__ src, float *__restrict__ dst, int n, const float *c) {
	if (n >= 5) {
		for (int j = threadIdx.x; j < n; j += blockDim.x) {
			const int a = (j + n - 2) % n, b = (j + n - 1) % n, d = (j + 1) % n, e = (j + 2) % n;
			float acc = __fmul_rn(src[a], c[0]);
			acc = __fadd_rn(acc, __fmul_rn(src[b], c[1]));
			acc = __fadd_rn(acc, __fmul_rn(src[j], c[2]));
			acc = __fadd_rn(acc, __fmul_rn(src[d], c[3]));
			acc = __fadd_rn(acc, __fmul_rn(src[e], c[4]));
			dst[j] = acc;
		}
	} else if (threadIdx.x == 0) {
		for (int j = 0; j < n; j++) dst[j] = src[j];
		float w0 = dst[0], w1 = dst[1 % n], w2 = dst[2 % n], w3 = dst[3 % n], w4 = dst[4 % n];
		const float k2 = w2, k3 = w3, k4 = w4;
		for (int i = 0; i < n; i++) {
			const int upd = (i < n - 2) ? (i + 2) : (i - (n - 2));
			const int nxt = (i < n - 5) ? (i + 5) : (i - (n - 5));
			float acc = __fmul_rn(w0, c[0]);
			acc = __fadd_rn(acc, __fmul_rn(w1, c[1]));
			acc = __fadd_rn(acc, __fmul_rn(w2, c[2]));
			acc = __fadd_rn(acc, __fmul_rn(w3, c[3]));
			acc = __fadd_rn(acc, __fmul_rn(w4, c[4]));
			dst[upd] = acc;
			w0 = w1; w1 = w2; w2 = w3; w3 = w4;
			if (nxt < 2 || nxt >= 5) w4 = dst[nxt]; else w4 = (nxt == 2) ? k2 : (nxt == 3 ? k3 : k4);
		}
	}
}

// the serial part of findbestfit: window sums for every start position (syncdetector.c:31-49).
// cs[0] = sum of the first `strip` elements; cs[e] = window sum after the e-th slide.  `data` already holds the
// blurred strip widened to double (exact), so the dependent chain is two DADDs per step; the operands of the next
// 8 steps are fetched before the chain needs them (a warp issues in order: without this every step would also
// wait for a shared-memory load).
__device__ void window_sums(const double *__restrict__ data, int size, int strip, double *__restrict__ cs) {
	double cur = 0.0;
	int i = 0;
	for (; i + 8 <= strip; i += 8) {
		double v[8];
		#pragma unroll
		for (int u = 0; u < 8; u++) v[u] = data[i + u];
		#pragma unroll
		for (int u = 0; u < 8; u++) cur = __dadd_rn(cur, v[u]);
	}
	for (; i < strip; i++) cur = __dadd_rn(cur, data[i]);
	cs[0] = cur;
	const int wrap_at = size - strip, last = size - 1;
	i = 0;
	for (; i + 8 <= last; i += 8) {
		double rem[8], add[8];
		#pragma unroll
		for (int u = 0; u < 8; u++) {
			const int k = i + u;
			rem[u] = data[k];
			add[u] = data[(k < wrap_at) ? (k + strip) : (k - wrap_at)];
		}
		#pragma unroll
		for (int u = 0; u < 8; u++) { cur = __dadd_rn(__dsub_rn(cur, rem[u]), add[u]); cs[i + u + 1] = cur; }
	}
	for (; i < last; i++) {
		cur = __dadd_rn(__dsub_rn(cur, data[i]), data[(i < wrap_at) ? (i + strip) : (i - wrap_at)]);
		cs[i + 1] = cur;
	}
}

__device__ double strip_total(const double *__restrict__ data, int size) {       // syncdetector.c:81-82
	double tot = 0.0;
	int i = 0;
	for (; i + 8 <= size; i += 8) {
		double v[8];
		#pragma unroll
		for (int u = 0; u < 8; u++) v[u] = data[i + u];
		#pragma unroll
		for (int u = 0; u < 8; u++) tot = __dadd_rn(tot, v[u]);
	}
	for (; i < size; i++) tot = __dadd_rn(tot, data[i]);
	return tot;
}

__device__ __forceinline__ double fit_score(double total, double cs, double n_out, double n_in) {
	const double contrast = __dsub_rn(__ddiv_rn(__dsub_rn(total, cs), n_out), __ddiv_rn(cs, n_in));
	return __dmul_rn(contrast, contrast);
}

struct Best { double score; int e; };
// first maximum in e-order (the reference updates only on a strict '>')
__device__ __forceinline__ Best best_merge(Best a, Best b) {
	if (b.score > a.score || (b.score == a.score && b.e < a.e)) return b;
	return a;
}

// exact 5-tap circular blur of one strip straight from global memory into a double array (gaussian.c:18-79)
__device__ void blur_to_double(const float *__restrict__ src, double *__restrict__ dst, int n, const float *c, float *tmp) {
	if (n >= 5) {
		for (int j = threadIdx.x; j < n; j += blockDim.x) {
			const int a = (j + n - 2) % n, b = (j + n - 1) % n, d = (j + 1) % n, e = (j + 2) % n;
			float acc = __fmul_rn(__ldg(src + a), c[0]);
			acc = __fadd_rn(acc, __fmul_rn(__ldg(src + b), c[1]));
			acc = __fadd_rn(acc, __fmul_rn(__ldg(src + j), c[2]));
			acc = __fadd_rn(acc, __fmul_rn(__ldg(src + d), c[3]));
			acc = __fadd_rn(acc, __fmul_rn(__ldg(src + e), c[4]));
			dst[j] = (double) acc;
		}
	} else {                          // degenerate strips: literal replay through the float helper
		if (threadIdx.x < n) tmp[threadIdx.x] = src[threadIdx.x];
		__syncthreads();
		blur_strip(tmp, tmp + 8, n, c);
		__syncthreads();
		if (threadIdx.x < n) dst[threadIdx.x] = (double) tmp[8 + threadIdx.x];
	}
}

// ---- exact window sums without the serial chain ------------------------------------------------------------------
// findbestfit's sliding sum cur = (cur - d[i]) + d[i+s] is a serial chain of ~2n dependent double additions per strip
// size.  But the strip holds floats widened to double; when the exponents of its non-zero entries span less than
// 29 - log2(n) binades, EVERY partial sum of up to n entries is an integer multiple of the smallest ulp and smaller than
// 2^53 of them: it is exactly representable, so no addition or subtraction in the chain ever rounds and the chain's
// values equal the exact real-number window sums -- in any association.  Then cs[e] = S[e+s] - S[e] from one exclusive
// prefix scan S (also exact) is bit-identical to the reference's chain, for every strip size at once.  The certificate
// is checked per strip per frame; if it fails (denormals, infinities, > ~2^17 dynamic range) the serial chains run.
struct ExpRange { int lo, hi, bad; };
__device__ __forceinline__ void exp_range_add(ExpRange &r, float v) {
	const unsigned bits = __float_as_uint(v), e = (bits >> 23) & 0xffu, m = bits & 0x7fffffu;
	if (e == 0) { if (m) r.bad = 1; return; }            // zero is harmless, a denormal is not covered
	if (e == 255) { r.bad = 1; return; }
	r.lo = min(r.lo, (int) e); r.hi = max(r.hi, (int) e);
}

// exclusive prefix sums of data[0..n) into S[0..n] IN PLACE over the same storage shifted by one:
// on entry buf[1..n] = data, on exit buf[i] = sum_{j<i} data[j] (buf[0] = 0).  All threads of the CTA take part; buf is in
// shared or global memory.
__device__ void exact_prefix(double *buf, int n, double *warp_tot /* >= 32 */) {
	const int T = blockDim.x, chunk = (n + T - 1) / T;
	const int i0 = min((int) threadIdx.x * chunk, n), i1 = min(i0 + chunk, n);
	double local = 0.0;                                  // every thread owns one contiguous chunk of ceil(n / blockDim.x) entries
	for (int i = i0; i < i1; i++) local += buf[1 + i];
	// exclusive scan of `local` across the CTA
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	double incl = local;
	#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const double up = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += up; }
	if (lane == 31) warp_tot[warp] = incl;
	__syncthreads();                                     // also: every thread has read its chunk
	if (warp == 0) {
		double w = (lane < (T >> 5)) ? warp_tot[lane] : 0.0, wi = w;
		#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const double up = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += up; }
		warp_tot[lane] = wi - w;                         // exclusive
	}
	__syncthreads();
	double run = warp_tot[warp] + (incl - local);
	if (threadIdx.x == 0) buf[0] = 0.0;
	for (int i = i0; i < i1; i++) { run += buf[1 + i]; buf[1 + i] = run; }      // in place: a thread only touches its own chunk
	__syncthreads();
}

__device__ __forceinline__ double window_from_prefix(const double *S, int n, int e, int strip) {
	const int end = e + strip;
	if (end <= n) return S[end] - S[e];
	return (S[n] - S[e]) + S[end - n];
}

// The sync search of a batch is split in two kernels.
//   fs_sync_prep   (one CTA per frame, frames in parallel): everything that does not depend on the previous frame --
//                  blur both strips into double, exactness certificate, exact prefix scans, strip totals -- written as
//                  one record per frame: [x buffer: w+1][y buffer: h+1][ok_x, ok_y, total_x, total_y].  A buffer holds the
//                  prefix sums S[0..n] when its certificate holds, otherwise the blurred strip in [1..n].
//                  Strips too long for shared memory (w + h + 2 > FS_SMEM_STRIPS) are built in the record itself.
//   fs_sync        (one CTA walks the frames in order: the strip size and dx carry from frame to frame): records are
//                  prefetched into shared memory one frame ahead (cp.async) while two fit beside the main stream's CTAs,
//                  the next one at the bottom of the loop while one fits, and read from global memory (L2) when none
//                  does (nbuf = 2 / 1 / 0; the same arithmetic either way), every thread scores a slice of the windows
//                  of every candidate strip size (serial chains first when a certificate failed), first-max reduce,
//                  thread 0 picks the strip size and updates dx/vx and the PLL average.
// Speculation tables.  Which strip sizes frame f tries depends on frame f-1's winner -- but the winner almost always stays where
// it was or moves by one step of 4.  fs_sync_prep therefore scores, for every frame of the batch IN PARALLEL, every strip size
// that can come up while the carried size stays within +-4*FS_SPEC_J of its value at the start of the batch (the sizes
// themselves, their +-4 neighbours, halves and doubles), leaving one (score, first index) pair per size.  fs_sync_walk then
// walks the frames with table look-ups only; the moment a frame asks for a size that is not in its table (a jump by a factor
// of two, a strip that failed the exactness certificate) it stops, and the cluster kernel fs_sync takes over from that frame
// with the literal search.  Same arithmetic, same first-maximum rule: identical integers either way.
constexpr int FS_SPEC_J = 3, FS_SPEC_MAX = 24;            // sizes cur0 + 4j, |j| <= J, and what their candidate lists contain (<= 23)
constexpr int FS_SPEC_AX = 1 + 3 * FS_SPEC_MAX;           // per axis: count, sizes[], scores[], first indices[]
constexpr int FS_PREP_HDR = 4 + 2 * FS_SPEC_AX;
__host__ __device__ __forceinline__ size_t fs_prep_stride(int w, int h) { return (size_t) w + h + 2 + FS_PREP_HDR; }
// whether fs_sync_prep builds a frame's strip buffers in shared memory (then copies them to the record) or directly in the
// global record (strips longer than shared memory holds: w + h up to the reference's 4000 x 4000 pixels)
__host__ __device__ __forceinline__ bool fs_prep_in_smem(int w, int h) { return (size_t) w + h + 2 <= (size_t) FS_SMEM_STRIPS; }

// the strip sizes a frame's search tries, in the reference's order (syncdetector.c:60-69, 73-77, 88-93); vals[t] = -1: skipped.
// `cur` is clamped in place like the reference clamps sweetspot_data_t.curr_stripsize.  vals[0] is always tried, also when the
// clamp leaves 0 (a strip of 1 pixel: half = 0): the reference then scores a zero-length strip, NaN at every start, and keeps index 0.
__device__ __forceinline__ void sweet_candidates(int &cur, int size, int minsize, int vals[5]) {
	if (minsize < 1) minsize = 1;
	const int half = size >> 1;
	if (cur < minsize) cur = minsize; else if (cur > half) cur = half;
	const int tries[5] = {cur, cur - 4, cur + 4, cur >> 1, cur << 1};
	vals[0] = cur;
	for (int t = 1; t < 5; t++) vals[t] = (tries[t] >= minsize && tries[t] < half && tries[t] != cur) ? tries[t] : -1;
}

// GREC: the strip buffers are built in the global record (!fs_prep_in_smem), not in shared memory
template <bool GREC>
__global__ void __launch_bounds__(FS_SYNC_THREADS) fs_sync_prep(const float *__restrict__ wstrips, const float *__restrict__ hstrips,
                                                                int w, int h, float c0, float c1, float c2, float c3, float c4,
                                                                int force_serial, double *__restrict__ prep,
                                                                const SyncState *__restrict__ state, int minsize_x, int minsize_y, int spec_on) {
	extern __shared__ double smem_d[];
	const int f = blockIdx.x;
	double *rec = prep + (size_t) f * fs_prep_stride(w, h);
	double *buf_x = GREC ? rec : smem_d, *buf_y = buf_x + (w + 1);
	__shared__ float tiny[16];
	__shared__ double warp_tot[32];
	__shared__ int range_lo[2], range_hi[2], range_bad[2], exact_ok[2];
	__shared__ float totalf[2];
	const float taps[5] = {c0, c1, c2, c3, c4};
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	if (threadIdx.x < 2) { range_lo[threadIdx.x] = 255; range_hi[threadIdx.x] = 0; range_bad[threadIdx.x] = 0; }
	if (threadIdx.x == 0) { buf_x[0] = 0.0; buf_y[0] = 0.0; }
	blur_to_double(wstrips + (size_t) f * w, buf_x + 1, w, taps, tiny);
	blur_to_double(hstrips + (size_t) f * h, buf_y + 1, h, taps, tiny);
	__syncthreads();
	for (int ax = 0; ax < 2; ax++) {                     // exactness certificate (see above)
		const int n = ax ? h : w; const double *d = (ax ? buf_y : buf_x) + 1;
		ExpRange r; r.lo = 255; r.hi = 0; r.bad = 0;
		for (int i = threadIdx.x; i < n; i += blockDim.x) exp_range_add(r, (float) d[i]);
		for (int o = 16; o > 0; o >>= 1) {
			r.lo = min(r.lo, __shfl_xor_sync(0xffffffffu, r.lo, o)); r.hi = max(r.hi, __shfl_xor_sync(0xffffffffu, r.hi, o));
			r.bad |= __shfl_xor_sync(0xffffffffu, r.bad, o);
		}
		if (lane == 0) { atomicMin(&range_lo[ax], r.lo); atomicMax(&range_hi[ax], r.hi); if (r.bad) atomicOr(&range_bad[ax], 1); }
	}
	__syncthreads();
	if (threadIdx.x < 2) {
		const int ax = threadIdx.x, n = ax ? h : w;
		int lg = 0; while ((1 << lg) < n) lg++;
		const int span = (range_hi[ax] >= range_lo[ax]) ? (range_hi[ax] - range_lo[ax]) : 0;
		exact_ok[ax] = !force_serial && !range_bad[ax] && (span < 29 - lg);
	}
	__syncthreads();
	const bool ok_x = exact_ok[0], ok_y = exact_ok[1];
	if (lane == 0 && warp < 2 && !(warp ? ok_y : ok_x))  // serial total for a strip that failed the certificate (syncdetector.c:81-82)
		totalf[warp] = __double2float_rn(strip_total((warp ? buf_y : buf_x) + 1, warp ? h : w));
	if (ok_x) exact_prefix(buf_x, w, warp_tot);
	if (ok_y) exact_prefix(buf_y, h, warp_tot);
	__syncthreads();
	if (threadIdx.x < 2 && exact_ok[threadIdx.x]) totalf[threadIdx.x] = __double2float_rn(threadIdx.x ? buf_y[h] : buf_x[w]);   // findbestfit takes a float
	__syncthreads();
	const int nbody = w + h + 2;
	if (!GREC) for (int i = threadIdx.x; i < nbody; i += blockDim.x) rec[i] = smem_d[i];
	if (threadIdx.x == 0) {
		rec[nbody + 0] = ok_x ? 1.0 : 0.0; rec[nbody + 1] = ok_y ? 1.0 : 0.0;
		rec[nbody + 2] = (double) totalf[0]; rec[nbody + 3] = (double) totalf[1];
	}
	// ---- speculation tables (see FS_SPEC_*): one warp per (axis, strip size), lanes over the window positions
	__shared__ int spec_n[2], spec_size[2][FS_SPEC_MAX];
	if (threadIdx.x < 2) {
		const int ax = threadIdx.x, size = ax ? h : w, half = size >> 1;
		int minsize = ax ? minsize_y : minsize_x; if (minsize < 1) minsize = 1;
		int n = 0;
		if (spec_on && exact_ok[ax]) {
			int cur0 = ax ? state->y_strip : state->x_strip;
			if (cur0 < minsize) cur0 = minsize; else if (cur0 > half) cur0 = half;
			auto add = [&](int v) { for (int i = 0; i < n; i++) if (spec_size[ax][i] == v) return; if (n < FS_SPEC_MAX) spec_size[ax][n++] = v; };
			for (int j = -FS_SPEC_J; j <= FS_SPEC_J; j++) {
				int c = cur0 + 4 * j;
				if (c < minsize || c > half) continue;           // the carried size always lies in [minsize, half]
				int vals[5];
				sweet_candidates(c, size, minsize, vals);
				for (int t = 0; t < 5; t++) if (vals[t] > 0) add(vals[t]);
			}
		}
		spec_n[ax] = n;
	}
	__syncthreads();
	double *spec = rec + nbody + 4;
	const int items = spec_n[0] + spec_n[1];
	for (int it = warp; it < items; it += (int) (blockDim.x >> 5)) {
		const int ax = it < spec_n[0] ? 0 : 1, idx = ax ? it - spec_n[0] : it;
		const int size = ax ? h : w, strip = spec_size[ax][idx];
		const double *S = ax ? buf_y : buf_x;
		const double tot = (double) totalf[ax], n_out = (double) (size - strip), n_in = (double) strip;
		Best b; b.score = -INFINITY; b.e = 0x7fffffff;
		for (int e = lane; e < size; e += 32) {
			const double sc = fit_score(tot, window_from_prefix(S, size, e, strip), n_out, n_in);
			if (sc > b.score) { b.score = sc; b.e = e; }          // a lane walks upwards: the first of equal scores stays
		}
		for (int o = 16; o > 0; o >>= 1) {
			Best other; other.score = __shfl_xor_sync(0xffffffffu, b.score, o); other.e = __shfl_xor_sync(0xffffffffu, b.e, o);
			b = best_merge(b, other);
		}
		if (lane == 0) {
			if (b.e == 0x7fffffff) { b.score = fit_score(tot, window_from_prefix(S, size, 0, strip), n_out, n_in); b.e = 0; }   // as fs_sync does
			double *a = spec + ax * FS_SPEC_AX;
			a[1 + idx] = (double) strip; a[1 + FS_SPEC_MAX + idx] = b.score; a[1 + 2 * FS_SPEC_MAX + idx] = (double) b.e;
		}
	}
	if (threadIdx.x < 2) spec[threadIdx.x * FS_SPEC_AX] = (double) spec_n[threadIdx.x];
}

__device__ __forceinline__ void fs_prefetch_record(double *dst, const double *__restrict__ src, int count) {
	for (int i = threadIdx.x; i < count; i += blockDim.x) __pipeline_memcpy_async(dst + i, src + i, sizeof(double));
	__pipeline_commit();
}

// What findthesweetspot does once the best window of the winning strip size is known (syncdetector.c:95-118) plus, on the x
// axis, frameratepll's averages (syncdetector.c:134-139): one thread per axis.  Shared by the table walker and the cluster search.
__device__ __forceinline__ void sweet_update(int ax, SyncState &st, Best best, int best_size, int size, tsdrgpu_frame_result_t *r) {
	const double lowpass = ax ? 0.1 : 0.9;          // FRAMERATE_DX_LOWPASS_COEFF_* (syncdetector.c:15-16)
	int &dx = ax ? st.y_dx : st.x_dx; int &vx = ax ? st.y_vx : st.x_vx;
	int &absvx = ax ? st.y_absvx : st.x_absvx; int &cur = ax ? st.y_strip : st.x_strip;
	const int best_start = (best.e == 0) ? 0 : best.e - 1;   // index recorded before the slide
	cur = best_size;
	const int h2 = size / 2;
	int centre = (best_start + best_size / 2) % size;
	const int jump = centre - dx;
	if (jump > h2) dx += size; else if (jump < -h2) centre += size;
	const int before = dx;
	const double mixed = __dadd_rn(__dmul_rn((double) centre, lowpass), __dmul_rn(__dsub_rn(1.0, lowpass), (double) dx));
	dx = (int) (((long long) round(mixed)) % ((long long) size));
	const int moved = dx - before;
	vx = (moved > h2) ? (size - moved) : ((moved < -h2) ? (-size - moved) : moved);
	absvx = (vx >= 0) ? vx : -vx;
	if (ax == 0) {
		// frameratepll bookkeeping (syncdetector.c:134-139); the refreshrate write-back is the host's
		st.avg_speed = __dadd_rn(__dmul_rn(st.avg_speed, 0.99), __dmul_rn(0.01, (double) st.x_vx));
		st.pll_state = (st.avg_speed < 0.5 && st.avg_speed > -0.5) ? 1 : 0;
		r->x_dx = st.x_dx; r->x_vx = st.x_vx; r->x_absvx = st.x_absvx; r->x_stripsize = st.x_strip;
		r->avg_speed = st.avg_speed; r->pll_state = st.pll_state;
		r->autogain_report = 0; r->reserved = 0;
	} else {
		r->y_dx = st.y_dx; r->y_vx = st.y_vx; r->y_absvx = st.y_absvx; r->y_stripsize = st.y_strip;
	}
}

// The table walker (see FS_SPEC_*): one warp per axis walks the frames in order using only fs_sync_prep's per-frame tables.
// Lane i of a warp keeps entry i of its axis' table (size, score, first index) in registers -- the next frame's entries are
// loaded while the current frame is decided -- so a look-up is a ballot and two shuffles; lane 0 then does findthesweetspot's
// scalar update.  *resume receives the first frame that could not be served (nframes when all were): fs_sync continues there.
__global__ void __launch_bounds__(64) fs_sync_walk(const double *__restrict__ prep, int w, int h, int minsize_x, int minsize_y, int nframes,
                                                   SyncState *state, tsdrgpu_frame_result_t *results, int *resume) {
	__shared__ int fail[2];
	__shared__ SyncState st;
	const int rec_len = (int) fs_prep_stride(w, h), nbody = w + h + 2;
	const int ax = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int size = ax ? h : w, minsize = ax ? minsize_y : minsize_x;
	struct Entry { int n, sz, e; double score; };
	auto fetch = [&](int f) {
		const double *a = prep + (size_t) f * rec_len + nbody + 4 + ax * FS_SPEC_AX;
		Entry t;
		t.n = (int) a[0];
		const bool live = lane < FS_SPEC_MAX;                // FS_SPEC_MAX <= 32: one entry per lane
		t.sz = live ? (int) a[1 + lane] : -2;
		t.score = live ? a[1 + FS_SPEC_MAX + lane] : 0.0;
		t.e = live ? (int) a[1 + 2 * FS_SPEC_MAX + lane] : 0;
		if (lane >= t.n) t.sz = -2;                          // entries beyond the count are stale memory
		return t;
	};
	if (threadIdx.x == 0) { st = *state; fail[0] = fail[1] = 0; }
	Entry cur_t = fetch(0);
	__syncthreads();
	int f = 0;
	for (; f < nframes; f++) {
		Entry next_t = cur_t;
		if (f + 1 < nframes) next_t = fetch(f + 1);          // in flight while this frame is decided
		int cur = ax ? st.y_strip : st.x_strip, vals[5];
		sweet_candidates(cur, size, minsize, vals);          // every lane: a handful of integer operations
		Best best; best.score = -1.0; best.e = -1; int best_size = 0;
		bool ok = cur_t.n > 0, first = true;
		#pragma unroll
		for (int t = 0; t < 5; t++) {
			if (vals[t] < 0) continue;
			const unsigned hit = __ballot_sync(0xffffffffu, cur_t.sz == vals[t]);
			if (!hit) { ok = false; continue; }
			const int src = __ffs(hit) - 1;
			Best c; c.score = __shfl_sync(0xffffffffu, cur_t.score, src); c.e = __shfl_sync(0xffffffffu, cur_t.e, src);
			// pick among candidates in the reference's order, strict '>' (syncdetector.c:60-69)
			if (first || c.score > best.score) { best = c; best_size = vals[t]; }
			first = false;
		}
		if (lane == 0 && !ok) fail[ax] = 1;
		__syncthreads();
		if (fail[0] | fail[1]) break;
		if (lane == 0) sweet_update(ax, st, best, best_size, size, results + f);
		__syncthreads();                                     // st is up to date for both warps before the next frame reads it
		cur_t = next_t;
	}
	if (threadIdx.x == 0) {
		state->x_dx = st.x_dx; state->x_vx = st.x_vx; state->x_absvx = st.x_absvx; state->x_strip = st.x_strip;
		state->y_dx = st.y_dx; state->y_vx = st.y_vx; state->y_absvx = st.y_absvx; state->y_strip = st.y_strip;
		state->avg_speed = st.avg_speed; state->pll_state = st.pll_state;
		*resume = f;
	}
}

// fs_sync runs as ONE thread-block cluster of FS_SEL_CLUSTER CTAs (8 SMs).  Scoring a window costs two correctly rounded
// double divisions (~56 FP64 instructions) and a frame has ~9300 windows (5 strip sizes x 2 axes): on one SM that is FP64-
// pipe bound.  The cluster splits the windows in warp-sized units over its 8 SMs; per-CTA maxima travel
// to CTA 0 through distributed shared memory, CTA 0 picks the strip size / updates dx and broadcasts the next frame's
// candidate sizes the same way: two cluster barriers per frame.
constexpr int FS_SEL_THREADS = 512, FS_SEL_CLUSTER = 8, FS_SEL_WARPS = FS_SEL_THREADS / 32;

// GREC: the records are read in global memory (nbuf = 0), not from shared memory
template <bool GREC>
__global__ void __cluster_dims__(FS_SEL_CLUSTER, 1, 1) __launch_bounds__(FS_SEL_THREADS)
fs_sync(const double *__restrict__ prep, int nbuf, int w, int h, int minsize_x, int minsize_y, int nframes,
        SyncState *state, double *__restrict__ chain_scratch, tsdrgpu_frame_result_t *results, const int *__restrict__ resume) {
	const int f_start = resume ? *resume : 0;             // frames before it were served by fs_sync_walk
	if (f_start >= nframes) return;                       // every CTA of the cluster sees the same value: nobody is left at a barrier
	cg::cluster_group cluster = cg::this_cluster();
	const unsigned rank = cluster.block_rank();
	extern __shared__ double smem_d[];
	const int rec_len = (int) fs_prep_stride(w, h), nbody = w + h + 2;
	__shared__ int cand[2][5];                           // strip sizes tried per axis, -1 = skipped (written by CTA 0)
	__shared__ Best warp_best[FS_SEL_WARPS][10];
	__shared__ Best rank_best[FS_SEL_CLUSTER][10];       // CTA 0's copy is the one that is used (written remotely)
	__shared__ Best cand_best[2][5];
	__shared__ SyncState st;                             // CTA 0
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

	// clamp the carried strip size, list the sizes to try (syncdetector.c:73-77, 60-69, 88-93), tell every CTA.  The clamp works on
	// a copy: after a batch's last frame the state keeps the winner itself, as the reference does (where half < minsize, a
	// one-pixel axis, clamping twice is not clamping once: 1 -> 0 -> 1)
	auto list_candidates = [&](int ax) {
		int cur = ax ? st.y_strip : st.x_strip;
		int vals[5];
		sweet_candidates(cur, ax ? h : w, ax ? minsize_y : minsize_x, vals);
		for (unsigned r = 0; r < FS_SEL_CLUSTER; r++) {
			int *rc = cluster.map_shared_rank(&cand[0][0], r);
			for (int t = 0; t < 5; t++) rc[ax * 5 + t] = vals[t];
		}
	};
	if (rank == 0) {
		if (threadIdx.x == 0) st = *state;
		__syncthreads();
		if (threadIdx.x == 0 || threadIdx.x == 32) list_candidates(threadIdx.x >> 5);
	}
	if (!GREC) fs_prefetch_record(smem_d + (size_t) (nbuf == 2 ? (f_start & 1) : 0) * rec_len, prep + (size_t) f_start * rec_len, rec_len);
	cluster.sync();
	const size_t chain_len = (size_t) max(w, h);         // one window sum per start position of the longer strip (fs_reserve)

	const int units_x = (w + 31) >> 5, units_y = (h + 31) >> 5, units = 5 * (units_x + units_y);
	for (int f = f_start; f < nframes; f++) {
		// nbuf = 0: records longer than shared memory holds are read where fs_sync_prep left them (global memory, mostly from L2)
		const double *rec = GREC ? prep + (size_t) f * rec_len : smem_d + (size_t) (nbuf == 2 ? (f & 1) : 0) * rec_len;
		__pipeline_wait_prior(0);
		__syncthreads();                                 // record f is in shared memory; the other buffer is no longer read
		if (!GREC && nbuf == 2 && f + 1 < nframes) fs_prefetch_record(smem_d + (size_t) ((f + 1) & 1) * rec_len, prep + (size_t) (f + 1) * rec_len, rec_len);
		const double *buf_x = rec, *buf_y = rec + (w + 1);     // prefix sums S[0..n], or the blurred strip in [1..n]
		const bool ok_x = rec[nbody + 0] != 0.0, ok_y = rec[nbody + 1] != 0.0;
		const float tot_x = (float) rec[nbody + 2], tot_y = (float) rec[nbody + 3];
		// serial chains for strips that failed the certificate: chain ci on CTA ci % 8, window sums to the global scratch
		if (!ok_x || !ok_y) {
			if (lane == 0) {
				const int ci = (int) rank + FS_SEL_CLUSTER * warp;
				if (ci < 10) {
					const int ax = ci / 5, strip = cand[ax][ci % 5];
					if (strip >= 0 && !(ax ? ok_y : ok_x)) window_sums((ax ? buf_y : buf_x) + 1, ax ? h : w, strip, chain_scratch + (size_t) ci * chain_len);
				}
			}
			cluster.sync();
		}
		// score every window of every candidate: warp-sized units dealt round-robin over the cluster's warps
		if (lane < 10) { Best z; z.score = -INFINITY; z.e = 0x7fffffff; warp_best[warp][lane] = z; }
		__syncwarp();
		for (int u = (int) rank * FS_SEL_WARPS + warp; u < units; u += FS_SEL_CLUSTER * FS_SEL_WARPS) {
			int ci, blk;
			if (u < 5 * units_x) { ci = u / units_x; blk = u - ci * units_x; }
			else { const int u2 = u - 5 * units_x; ci = u2 / units_y; blk = u2 - ci * units_y; ci += 5; }
			const int ax = ci / 5, strip = cand[ax][ci % 5];
			if (strip < 0) continue;
			const int size = ax ? h : w, e = (blk << 5) + lane;
			Best b; b.score = -INFINITY; b.e = 0x7fffffff;
			if (e < size) {
				const bool ok = ax ? ok_y : ok_x;
				const double c = ok ? window_from_prefix(ax ? buf_y : buf_x, size, e, strip) : chain_scratch[(size_t) ci * chain_len + e];
				const double sc = fit_score((double) (ax ? tot_y : tot_x), c, (double) (size - strip), (double) strip);
				if (sc > b.score) { b.score = sc; b.e = e; }
			}
			for (int o = 16; o > 0; o >>= 1) {
				Best other; other.score = __shfl_xor_sync(0xffffffffu, b.score, o); other.e = __shfl_xor_sync(0xffffffffu, b.e, o);
				b = best_merge(b, other);
			}
			if (lane == 0) warp_best[warp][ci] = best_merge(warp_best[warp][ci], b);
		}
		__syncthreads();
		if (threadIdx.x < 10) {
			Best r = warp_best[0][threadIdx.x];
			for (int k = 1; k < FS_SEL_WARPS; k++) r = best_merge(r, warp_best[k][threadIdx.x]);
			Best *dst = cluster.map_shared_rank(&rank_best[0][0], 0);
			dst[rank * 10 + threadIdx.x] = r;
		}
		cluster.sync();
		if (rank == 0) {
			if (threadIdx.x < 10) {
				const int ci = threadIdx.x, ax = ci / 5, t = ci % 5;
				const int strip = cand[ax][t];
				Best r; r.score = -1.0; r.e = -1;
				if (strip >= 0) {
					const int size = ax ? h : w;
					r = rank_best[0][ci];
					for (int k = 1; k < FS_SEL_CLUSTER; k++) r = best_merge(r, rank_best[k][ci]);
					// e = 0 is the starting value of the reference's running maximum even when it is NaN
					// (with the certificate every score is a finite square, so this only matters on the serial-chain path)
					const bool ok = ax ? ok_y : ok_x;
					if (!ok || r.e == 0x7fffffff) {
						const double c0s = ok ? window_from_prefix(ax ? buf_y : buf_x, size, 0, strip) : chain_scratch[(size_t) ci * chain_len];
						const double s0 = fit_score((double) (ax ? tot_y : tot_x), c0s, (double) (size - strip), (double) strip);
						if (!(s0 == s0) || r.e == 0x7fffffff) { r.score = s0; r.e = 0; }
					}
				}
				cand_best[ax][t] = r;
			}
			__syncthreads();
			if (threadIdx.x == 0 || threadIdx.x == 32) {         // one thread per axis
				const int ax = threadIdx.x >> 5;
				// pick among candidates in the reference's order, strict '>' (syncdetector.c:60-69)
				Best best = cand_best[ax][0];
				int best_size = cand[ax][0];
				for (int t = 1; t < 5; t++) {
					if (cand[ax][t] < 0) continue;
					if (cand_best[ax][t].score > best.score) { best = cand_best[ax][t]; best_size = cand[ax][t]; }
				}
				sweet_update(ax, st, best, best_size, ax ? h : w, results + f);   // the auto-gain fields of the record belong to fs_results_autogain
				list_candidates(ax);                              // for the next frame
			}
		}
		cluster.sync();
		if (!GREC && nbuf == 1 && f + 1 < nframes) fs_prefetch_record(smem_d, prep + (size_t) (f + 1) * rec_len, rec_len);
	}
	if (rank == 0 && threadIdx.x == 0) {
		// auto-gain fields of the state are owned by the auto-gain epilogue: write back the sync part only
		state->x_dx = st.x_dx; state->x_vx = st.x_vx; state->x_absvx = st.x_absvx; state->x_strip = st.x_strip;
		state->y_dx = st.y_dx; state->y_vx = st.y_vx; state->y_absvx = st.y_absvx; state->y_strip = st.y_strip;
		state->avg_speed = st.avg_speed; state->pll_state = st.pll_state;
	}
}

// refresh the auto-gain fields of already written results (auto-gain-after-processing order)
__global__ void fs_results_autogain(int nframes, const FrameParams *__restrict__ params, const SyncState *__restrict__ state,
                                    tsdrgpu_frame_result_t *results, unsigned *clear = NULL) {
	if (clear && threadIdx.x == 0) *clear = 0;           // the certificate word of the batch about to be collapsed
	for (int f = threadIdx.x; f < nframes; f += blockDim.x) {
		if (params) { results[f].lastmax = params[f].lastmax; results[f].lastmin = params[f].lastmin; results[f].snr = params[f].snr; }
		else { results[f].lastmax = state->lastmax; results[f].lastmin = state->lastmin; results[f].snr = state->snr; }
	}
}

// ---------------------------------------------------------------- circular 2-D re-centre (syncdetector.c:187-207)
// 16-byte rows (w % 4 == 0, aligned in / out): a CTA copies a band of `band` destination rows of one frame, viewed as one run of
// band * w/4 float4s, four of them in flight per thread.  Destination float4 j of a row takes pixels (4j + dx .. 4j + dx + 3) mod w of
// its source row: with a = dx & 3 these are the last 4 - a of aligned source float4 s and the first a of the next one (the
// row's first float4 after the last), so every load and store is 16 bytes and the second load of a lane is mostly its
// neighbour's first, from L1.
__global__ void __launch_bounds__(256) fs_shift4(const float *__restrict__ in, float *__restrict__ out, int w, int h, int band,
                                                 const tsdrgpu_frame_result_t *__restrict__ results) {
	const int f = blockIdx.y;
	const int dx = results[f].x_dx, dy = results[f].y_dx;
	const int w4 = w >> 2, a = dx & 3, s0 = dx >> 2;
	const int y0 = blockIdx.x * band, rows = min(band, h - y0);
	const size_t n = (size_t) w * h;
	const float4 *src = reinterpret_cast<const float4 *>(in + f * n);
	float4 *dst = reinterpret_cast<float4 *>(out + f * n + (size_t) y0 * w);
	const int items = rows * w4;
	for (int i0 = threadIdx.x; i0 < items; i0 += 4 * 256) {
		float4 v[4];
		#pragma unroll
		for (int u = 0; u < 4; u++) {
			const int i = i0 + u * 256;
			if (i < items) {
				const int r = i / w4, j = i - r * w4;
				int sy = y0 + r + dy; if (sy >= h) sy -= h;
				const float4 *srow = src + (size_t) sy * w4;
				int s = j + s0; if (s >= w4) s -= w4;
				const float4 lo = __ldg(srow + s);
				if (a == 0) v[u] = lo;
				else {
					const float4 hi = __ldg(srow + (s + 1 == w4 ? 0 : s + 1));
					v[u] = (a == 1) ? make_float4(lo.y, lo.z, lo.w, hi.x) : (a == 2) ? make_float4(lo.z, lo.w, hi.x, hi.y)
					                                                                 : make_float4(lo.w, hi.x, hi.y, hi.z);
				}
			}
		}
		#pragma unroll
		for (int u = 0; u < 4; u++) if (i0 + u * 256 < items) dst[i0 + u * 256] = v[u];
	}
}

// rows at any alignment (odd widths): one destination row per CTA iteration
__global__ void __launch_bounds__(256) fs_shift(const float *__restrict__ in, float *__restrict__ out, int w, int h,
                                                const tsdrgpu_frame_result_t *__restrict__ results) {
	// no division per pixel, the wrap is a compare; up to 4 loads in flight per thread
	const int f = blockIdx.y;
	const int dx = results[f].x_dx, dy = results[f].y_dx;
	const size_t n = (size_t) w * h;
	const float *src = in + (size_t) f * n;
	float *dst = out + (size_t) f * n;
	for (int y = blockIdx.x; y < h; y += gridDim.x) {
		int sy = y + dy; if (sy >= h) sy -= h;
		const float *srow = src + (size_t) sy * w;
		float *drow = dst + (size_t) y * w;
		for (int x0 = threadIdx.x; x0 < w; x0 += 4 * 256) {
			float v[4];
			#pragma unroll
			for (int u = 0; u < 4; u++) {
				const int x = x0 + u * 256;
				int sx = x + dx; if (sx >= w) sx -= w;
				if (x < w) v[u] = __ldg(srow + sx);
			}
			#pragma unroll
			for (int u = 0; u < 4; u++) { const int x = x0 + u * 256; if (x < w) drow[x] = v[u]; }
		}
	}
}

// green marker lines (syncdetector.c:121-131, 209-220): copy (if out != in) then draw
__global__ void __launch_bounds__(256) fs_copy(const float *__restrict__ in, float *__restrict__ out, size_t total) {
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t) gridDim.x * blockDim.x) out[i] = in[i];
}
__global__ void __launch_bounds__(256) fs_greenlines(float *frames, int w, int h, const tsdrgpu_frame_result_t *__restrict__ results) {
	const int f = blockIdx.y;
	float *d = frames + (size_t) f * w * h;
	const int dx = results[f].x_dx, dy = results[f].y_dx;
	// vertical line first, then the horizontal one (its pixels win at the crossing; both are 512.0 anyway)
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < h + w; i += gridDim.x * blockDim.x) {
		if (i < h) d[dx + (size_t) w * i] = 512.0f; else d[(i - h) + (size_t) w * dy] = 512.0f;
	}
}

__global__ void __launch_bounds__(256) fs_argb(const float *__restrict__ frame, int n, int inverted, int *__restrict__ argb) {
	const int white = 255 | (255 << 8) | (255 << 16);
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float v = frame[i];
		int px;
		if (v > 0.0f && v <= 1.0f) {
			int g = (int) __fmul_rn(v, 255.0f);
			if (inverted) g = 255 - g;
			px = g | (g << 8) | (g << 16);
		} else if (v <= 0.0f) px = inverted ? white : 0;
		else if (v == 256.0f) px = 255 << 16;
		else if (v == 512.0f) px = 255 << 8;
		else if (v == 1024.0f) px = 255;
		else if (v == 2048.0f) continue;                 // transparent: slot left untouched
		else px = inverted ? 0 : white;
		argb[i] = px;
	}
}

// The same rule over a batch of frames, in place (a float frame becomes its int32 pixels), with the host's persistent pixel
// buffer (`last`) carried from frame to frame: a transparent sample (2048.0f) shows what that pixel showed before.
__global__ void __launch_bounds__(256) fs_argb_batch(float *frames, size_t n, int nframes, int inverted, int *__restrict__ last) {
	const int white = 255 | (255 << 8) | (255 << 16);
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) {
		int prev = last[i];
		for (int f = 0; f < nframes; f++) {
			float *slot = frames + (size_t) f * n + i;
			const float v = *slot;
			int px;
			if (v > 0.0f && v <= 1.0f) {
				int g = (int) __fmul_rn(v, 255.0f);
				if (inverted) g = 255 - g;
				px = g | (g << 8) | (g << 16);
			} else if (v <= 0.0f) px = inverted ? white : 0;
			else if (v == 256.0f) px = 255 << 16;
			else if (v == 512.0f) px = 255 << 8;
			else if (v == 1024.0f) px = 255;
			else if (v == 2048.0f) px = prev;
			else px = inverted ? 0 : white;
			*reinterpret_cast<int *>(slot) = px;
			prev = px;
		}
		last[i] = prev;
	}
}

// in shared memory, or (scratch != NULL: strips too long for it) from a copy in `scratch` straight back into `data`
__global__ void fs_blur_kernel(float *data, float *scratch, int n, float c0, float c1, float c2, float c3, float c4) {
	extern __shared__ float smem[];
	float *src = scratch ? scratch : smem, *dst = scratch ? data : smem + n;
	const float taps[5] = {c0, c1, c2, c3, c4};
	for (int i = threadIdx.x; i < n; i += blockDim.x) src[i] = data[i];
	__syncthreads();
	blur_strip(src, dst, n, taps);
	__syncthreads();
	if (!scratch) for (int i = threadIdx.x; i < n; i += blockDim.x) data[i] = dst[i];
}

inline unsigned grid_for(size_t n, int sm_count, int per_sm = 8) {
	const size_t want = (n + 255) / 256;
	const size_t cap = (size_t) sm_count * per_sm;
	return (unsigned) (want < cap ? (want ? want : 1) : cap);
}

// fs_collapse_tiles' two tensor maps over a batch of frames (w % 4 == 0 and a 16-byte aligned base: row and frame strides are
// multiples of 16 bytes, as the TMA unit requires).  cuTensorMapEncodeTiled comes from the driver through the runtime's
// entry-point query, so the library does not link libcuda.
struct CollapseMaps {
	const void *ptr; int w, h, nframes;
	CUtensorMap col, row;
};

int encode_collapse_maps(tsdrgpu_ctx_t *ctx, const float *ptr, int w, int h, int nframes, CollapseMaps *m) {
	static PFN_cuTensorMapEncodeTiled_v12000 encode = NULL;
	if (!encode) {
		void *fn = NULL;
		cudaDriverEntryPointQueryResult q;
		CU_TRY(ctx, cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q));
		if (q != cudaDriverEntryPointSuccess || !fn)
			return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "cuTensorMapEncodeTiled not found in the driver", cudaSuccess, __FILE__, __LINE__);
		encode = (PFN_cuTensorMapEncodeTiled_v12000) fn;
	}
	const cuuint64_t dims[3] = {(cuuint64_t) w, (cuuint64_t) h, (cuuint64_t) nframes};
	const cuuint64_t strides[2] = {(cuuint64_t) w * 4, (cuuint64_t) w * h * 4};
	const cuuint32_t cbox[3] = {CT_COLS, CT_CROWS, 1}, rbox[3] = {CT_RCOLS, CT_ROWS, 1}, unit[3] = {1, 1, 1};
	CUresult r = encode(&m->col, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *) ptr, dims, strides, cbox, unit, CU_TENSOR_MAP_INTERLEAVE_NONE,
	                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r == CUDA_SUCCESS)
		r = encode(&m->row, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void *) ptr, dims, strides, rbox, unit, CU_TENSOR_MAP_INTERLEAVE_NONE,
		           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "cuTensorMapEncodeTiled (collapse)", cudaSuccess, __FILE__, __LINE__);
	m->ptr = ptr; m->w = w; m->h = h; m->nframes = nframes;
	return TSDRGPU_OK;
}

// the collapse that normalises the raw frames on load (fs_collapse_tiles<true> / fs_collapse<true>)
struct NormOnLoad {
	const FrameParams *params;                   // (lastmin, span) per frame
	float *out;                                  // the normalised frames (aligned: a tensor map over it on the tiles path)
	unsigned *cert;                              // certificate word, set when the batch has to be redone
};

// row and column sums of `nframes` frames: the tensor-map kernel on 16-byte rows, the cp.async kernel otherwise.
// `name` labels the launch in the profile; with `gate`, the kernel returns at once unless *gate is set; with `norm`, src holds the
// raw frames and the collapse normalises them on load.
int launch_collapse(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *src, int w, int h, int nframes, float *wbuf, float *hbuf,
                    CollapseMaps *cache, int ncache, const char *name = "fs_collapse", const unsigned *gate = NULL,
                    const NormOnLoad *norm = NULL) {
	if ((w % 4 == 0) && ((reinterpret_cast<unsigned long long>(src) & 15ull) == 0)) {
		auto maps = [&](const float *ptr, CollapseMaps *out) -> int {      // the maps over `ptr`, from the cache or encoded into it
			for (int i = 0; i < ncache; i++)
				if (cache[i].ptr == ptr && cache[i].w == w && cache[i].h == h && cache[i].nframes == nframes) { *out = cache[i]; return TSDRGPU_OK; }
			int rc = encode_collapse_maps(ctx, ptr, w, h, nframes, out);
			if (rc) return rc;
			if (ncache) {                                // the frame stage collapses a handful of buffers: evict the oldest
				for (int i = ncache - 1; i > 0; i--) cache[i] = cache[i - 1];
				cache[0] = *out;
			}
			return TSDRGPU_OK;
		};
		CollapseMaps m, mo;
		int rc;
		if ((rc = maps(src, &m))) return rc;
		if (norm && (rc = maps(norm->out, &mo))) return rc;
		const int col_ctas = (w + CT_COLS - 1) / CT_COLS, row_ctas = (h + CT_ROWS - 1) / CT_ROWS;
		const dim3 grid(col_ctas + row_ctas, nframes);
		if (norm) {
			CU_TRY(ctx, cudaFuncSetAttribute(fs_collapse_tiles<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM));
			KL(ctx, name, stream, fs_collapse_tiles<true><<<grid, CT_NTHREADS, CT_SMEM, stream>>>(m.col, m.row, mo.col, w, h, wbuf, hbuf, col_ctas, NULL,
			                                                                                        norm->params, norm->cert));
		} else {
			CU_TRY(ctx, cudaFuncSetAttribute(fs_collapse_tiles<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM));
			KL(ctx, name, stream, fs_collapse_tiles<false><<<grid, CT_THREADS, CT_SMEM, stream>>>(m.col, m.row, m.col, w, h, wbuf, hbuf, col_ctas, gate, NULL, NULL));
		}
	} else {
		const int col_ctas = (w + CL_COLS - 1) / CL_COLS, row_ctas = (h + CL_ROWS - 1) / CL_ROWS;
		const dim3 grid(col_ctas + row_ctas, nframes);
		if (norm) KL(ctx, name, stream, fs_collapse<true><<<grid, 256, 0, stream>>>(src, w, h, wbuf, hbuf, col_ctas, NULL, norm->params, norm->out, norm->cert));
		else KL(ctx, name, stream, fs_collapse<false><<<grid, 256, 0, stream>>>(src, w, h, wbuf, hbuf, col_ctas, gate, NULL, NULL, NULL));
	}
	return TSDRGPU_OK;
}

}  // namespace

int fs_copy_async(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *in, float *out, size_t total) {
	KL(ctx, "fs_copy", stream, fs_copy<<<grid_for(total, ctx->sm_count), 256, 0, stream>>>(in, out, total));
	return TSDRGPU_OK;
}

// -----------------------------------------------------------------------------------------------------------------
struct tsdrgpu_framestage {
	tsdrgpu_ctx_t *ctx;
	DeviceBuf<float> d_screen;                   // dsp_postprocess_t.screenbuffer / bufsize
	int w, h; size_t n;                          // current geometry (pp->width/height/sizetopoll)
	int lp_before_sync;                          // pp->lowpass_before_sync
	int runs;                                    // pp->runs
	DeviceBuf<SyncState> d_state;
	// batch temporaries.  The sync search + re-centre of batch k may run on the side stream while the main stream
	// already produces batch k+1, so everything they read is double-buffered ("phase" = batch parity).
	DeviceBuf<float> d_t1, d_t2[2];
	DeviceBuf<float> d_wstrips[2], d_hstrips[2];
	DeviceBuf<float> d_pmin, d_pmax; DeviceBuf<double> d_psum, d_psq, d_plin; DeviceBuf<FrameParams> d_params;
	int batch_cap;                               // frames every per-batch buffer holds (0 until all of them are allocated)
	int ag_mode, ag_ppm;                         // tsdrgpu_framestage_set_autogain (kept across reset)
	DeviceBuf<unsigned> d_sel_hist; DeviceBuf<SelState> d_sel; DeviceBuf<float2> d_levels;     // clip-mode selection, batch_cap frames
	EnhanceState enh;                            // tsdrgpu_framestage_set_contrast / _set_denoise / _set_stack / _set_deblur (kept across reset)
	tsdrgpu_stack_record_t *h_stack_next;        // framestage_stack_next: where the next run's stack records go
	DeviceBuf<tsdrgpu_frame_result_t> d_results[2];
	DeviceBuf<double> d_chain;
	DeviceBuf<int> d_resume;                     // first frame of the batch fs_sync_walk could not serve from the tables
	float taps[5];
	int overlap, phase, side_pending;
	DeviceBuf<double> d_prep;                    // fs_sync_prep's per-frame records (consumed by fs_sync on the same stream)
	cudaStream_t s_side;
	cudaEvent_t ev_ready[2];                     // main: collapse of this phase done -> side may start
	cudaEvent_t ev_done[2];                      // side: sync + emit of this phase done -> buffers of the phase are free
	CollapseMaps collapse_maps[6];               // fs_collapse_tiles' tensor maps of the buffers collapsed last (d_t2[0/1], d_t1, inputs)
	DeviceBuf<unsigned> d_cert;                  // the batch's normalise-on-load certificate (fs_collapse_tiles<true>), cleared per batch
};

// hands a's buffer to b and b's to a (DeviceBuf can be neither copied nor moved)
static void fs_exchange(DeviceBuf<float> &a, DeviceBuf<float> &b) { std::swap(a.ptr, b.ptr); std::swap(a.cap, b.cap); }

// every buffer of a group at exactly n elements, all of them reallocated when one is short (a failed reallocation leaves that one
// empty, so the next call tries again); the side stream may still be reading them
template <class T, size_t K> static int fs_assign_group(tsdrgpu_ctx_t *ctx, DeviceBuf<T> *const (&bufs)[K], size_t n) {
	bool grow = false;
	for (DeviceBuf<T> *b : bufs) grow |= b->cap < n;
	if (!grow) return TSDRGPU_OK;
	CU_TRY(ctx, cudaDeviceSynchronize());
	for (DeviceBuf<T> *b : bufs) CU_TRY(ctx, b->assign(n));
	return TSDRGPU_OK;
}

static int fs_reserve(tsdrgpu_framestage *fs, int nframes, size_t n, int w, int h) {
	tsdrgpu_ctx_t *ctx = fs->ctx;
	int rc;
	DeviceBuf<float> *const frames[] = {&fs->d_t1, &fs->d_t2[0], &fs->d_t2[1]};
	if ((rc = fs_assign_group(ctx, frames, (size_t) nframes * n))) return rc;
	DeviceBuf<float> *const strips[] = {&fs->d_wstrips[0], &fs->d_wstrips[1], &fs->d_hstrips[0], &fs->d_hstrips[1]};
	if ((rc = fs_assign_group(ctx, strips, (size_t) nframes * (size_t) (w > h ? w : h)))) return rc;
	DeviceBuf<double> *const prep[] = {&fs->d_prep};
	if ((rc = fs_assign_group(ctx, prep, (size_t) nframes * fs_prep_stride(w, h)))) return rc;
	DeviceBuf<double> *const chain[] = {&fs->d_chain};       // fs_sync's serial chains: 10 candidates x the longer strip
	if ((rc = fs_assign_group(ctx, chain, (size_t) 10 * (size_t) (w > h ? w : h)))) return rc;
	if (fs->batch_cap < nframes) {
		CU_TRY(ctx, cudaDeviceSynchronize());
		fs->batch_cap = 0;
		const size_t pc = (size_t) nframes * FS_MM_CHUNKS;
		CU_TRY(ctx, fs->d_pmin.assign(pc));
		CU_TRY(ctx, fs->d_pmax.assign(pc));
		CU_TRY(ctx, fs->d_psum.assign(pc));
		CU_TRY(ctx, fs->d_psq.assign(pc));
		CU_TRY(ctx, fs->d_plin.assign(pc));
		CU_TRY(ctx, fs->d_params.assign(nframes));
		CU_TRY(ctx, fs->d_sel_hist.assign((size_t) 2 * SEL_BINS * nframes));
		CU_TRY(ctx, cudaMemset(fs->d_sel_hist.ptr, 0, sizeof(unsigned) * 2 * SEL_BINS * nframes));     // each scan re-zeroes what it read
		CU_TRY(ctx, fs->d_sel.assign(nframes));
		CU_TRY(ctx, fs->d_levels.assign(nframes));
		for (int i = 0; i < 2; i++) {
			CU_TRY(ctx, fs->d_results[i].assign(nframes));
			CU_TRY(ctx, cudaMemset(fs->d_results[i].ptr, 0, sizeof(tsdrgpu_frame_result_t) * nframes));
		}
		// the memsets run on the legacy default stream, which does not order work on non-blocking streams (the pipeline's):
		// the selection's first histogram round must see the zeroed counts
		CU_TRY(ctx, cudaDeviceSynchronize());
		fs->batch_cap = nframes;
	}
	return enhance_reserve(ctx, &fs->enh, nframes, w, h);
}

// clip mode's levels of a batch into d_levels (and, with snr, the per-chunk sums into d_psum): three radix-select rounds
static int fs_select_batch(tsdrgpu_framestage *fs, cudaStream_t stream, const float *in, int nframes, size_t n, int ppm, int chunks,
                           bool snr) {
	tsdrgpu_ctx_t *ctx = fs->ctx;
	const dim3 grid(chunks, nframes);
	if (snr) KL(ctx, "fs_select_hist", stream, (fs_select_hist<1, true><<<grid, 256, 0, stream>>>(in, n, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_psum.ptr)));
	else KL(ctx, "fs_select_hist", stream, (fs_select_hist<1, false><<<grid, 256, 0, stream>>>(in, n, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_psum.ptr)));
	KL(ctx, "fs_select_scan", stream, fs_select_scan<1><<<nframes, 256, 0, stream>>>(in, n, ppm, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_levels.ptr));
	KL(ctx, "fs_select_hist", stream, (fs_select_hist<2, false><<<grid, 256, 0, stream>>>(in, n, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_psum.ptr)));
	KL(ctx, "fs_select_scan", stream, fs_select_scan<2><<<nframes, 256, 0, stream>>>(in, n, ppm, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_levels.ptr));
	KL(ctx, "fs_select_hist", stream, (fs_select_hist<3, false><<<grid, 256, 0, stream>>>(in, n, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_psum.ptr)));
	KL(ctx, "fs_select_scan", stream, fs_select_scan<3><<<nframes, 256, 0, stream>>>(in, n, ppm, fs->d_sel.ptr, fs->d_sel_hist.ptr, fs->d_levels.ptr));
	return TSDRGPU_OK;
}

static int fs_chunks(size_t n) { return (int) ((n + 4095) / 4096 < FS_MM_CHUNKS ? (n + 4095) / 4096 : FS_MM_CHUNKS); }

// auto-gain of a batch: in -> out, state updated, params[f] filled
static int fs_autogain_batch(tsdrgpu_framestage *fs, cudaStream_t stream, const float *in, float *out, int nframes, size_t n,
                             float norm, bool snr) {
	tsdrgpu_ctx_t *ctx = fs->ctx;
	const int chunks = fs_chunks(n);
	dim3 grid(chunks, nframes);
	const bool clip = fs->ag_mode == TSDRGPU_AG_CLIP;
	int rc;
	if (clip) { if ((rc = fs_select_batch(fs, stream, in, nframes, n, fs->ag_ppm, chunks, snr))) return rc; }
	else if (snr) KL(ctx, "fs_minmax", stream, fs_minmax<true><<<grid, 256, 0, stream>>>(in, n, fs->d_pmin.ptr, fs->d_pmax.ptr, fs->d_psum.ptr));
	else KL(ctx, "fs_minmax", stream, fs_minmax<false><<<grid, 256, 0, stream>>>(in, n, fs->d_pmin.ptr, fs->d_pmax.ptr, fs->d_psum.ptr));
	KL(ctx, "fs_autogain_iir", stream, fs_autogain_iir<<<1, 256, 0, stream>>>(in, n, nframes, chunks, fs->d_pmin.ptr, fs->d_pmax.ptr, fs->d_psum.ptr, snr, norm, fs->d_state.ptr, fs->d_params.ptr,
	                                                                         clip ? fs->d_levels.ptr : NULL));
	if (!out) return TSDRGPU_OK;                     // statistics only: the caller fuses the normalisation elsewhere
	const unsigned gx = grid_for(n, ctx->sm_count, 4);
	dim3 grid2(snr ? (gx < (unsigned) FS_MM_CHUNKS ? gx : FS_MM_CHUNKS) : gx, nframes);
	if (snr) KL(ctx, "fs_normalise", stream, fs_normalise<true><<<grid2, 256, 0, stream>>>(in, out, n, fs->d_params.ptr, fs->d_psq.ptr, fs->d_plin.ptr));
	else KL(ctx, "fs_normalise", stream, fs_normalise<false><<<grid2, 256, 0, stream>>>(in, out, n, fs->d_params.ptr, fs->d_psq.ptr, fs->d_plin.ptr));
	if (snr) KL(ctx, "fs_snr_finish", stream, fs_snr_finish<<<1, 256, 0, stream>>>(nframes, (int) grid2.x, n, fs->d_psq.ptr, fs->d_plin.ptr, fs->d_params.ptr, fs->d_state.ptr));
	return TSDRGPU_OK;
}

extern "C" {

// a frame stage whole or half built: its stream and events (null ones are skipped), then the object; its buffers go with it
static void release(tsdrgpu_framestage *fs) {
	if (fs->s_side) cudaStreamDestroy(fs->s_side);
	for (cudaEvent_t e : {fs->ev_ready[0], fs->ev_ready[1], fs->ev_done[0], fs->ev_done[1]}) if (e) cudaEventDestroy(e);
	delete fs;
}

static int create_handles(tsdrgpu_framestage *fs) {
	tsdrgpu_ctx_t *ctx = fs->ctx;
	CU_TRY(ctx, fs->d_state.assign(1));
	CU_TRY(ctx, fs->d_resume.assign(64));
	CU_TRY(ctx, cudaMemset(fs->d_resume.ptr, 0, 256));
	CU_TRY(ctx, fs->d_cert.assign(1));
	{   // highest priority: its single CTA should be placed as soon as an SM has room, ahead of the main stream's queued CTAs
		int lo = 0, hi = 0;
		CU_TRY(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
		CU_TRY(ctx, cudaStreamCreateWithPriority(&fs->s_side, cudaStreamNonBlocking, hi));
	}
	for (int i = 0; i < 2; i++) {
		CU_TRY(ctx, cudaEventCreateWithFlags(&fs->ev_ready[i], cudaEventDisableTiming));
		CU_TRY(ctx, cudaEventCreateWithFlags(&fs->ev_done[i], cudaEventDisableTiming));
	}
	return tsdrgpu_framestage_reset(fs, NULL);
}

int tsdrgpu_framestage_create(tsdrgpu_ctx_t *ctx, tsdrgpu_framestage_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_framestage *fs = new tsdrgpu_framestage();      // value-initialised: every field not set here starts at zero
	fs->ctx = ctx;
	tsdrgpu_gauss_taps(fs->taps);
	const int rc = create_handles(fs);
	if (rc) { release(fs); return rc; }
	*out = fs;
	return TSDRGPU_OK;
}

void tsdrgpu_framestage_destroy(tsdrgpu_framestage_t *fs) {
	if (!fs) return;
	cudaSetDevice(fs->ctx->device);
	cudaDeviceSynchronize();
	release(fs);
}

int tsdrgpu_framestage_reset(tsdrgpu_framestage_t *fs, void *stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	BIND(fs->ctx);
	CU_TRY(fs->ctx, cudaStreamSynchronize(fs->s_side));
	SyncState s; memset(&s, 0, sizeof s);
	s.snr = 1.0f;                                        // dsp_autogain_init (dsp.c:35-39)
	CU_TRY(fs->ctx, cudaMemcpyAsync(fs->d_state.ptr, &s, sizeof s, cudaMemcpyHostToDevice, (cudaStream_t) stream));
	CU_TRY(fs->ctx, cudaStreamSynchronize((cudaStream_t) stream));
	{   // the screen buffer goes with `old` (DeviceBuf frees only in its destructor); the next run allocates and zeroes one of its
		// geometry.  Like every free in a destructor, an error of this one is not reported: nothing is left to recover.
		DeviceBuf<float> old;
		fs_exchange(old, fs->d_screen);
	}
	fs->w = 0; fs->h = 0; fs->n = 0; fs->lp_before_sync = 0; fs->runs = 0; fs->side_pending = 0;
	fs->enh.stack.m = 0;                                 // the stack restarts; its mode stays
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_autogain(tsdrgpu_framestage_t *fs, int mode, int ppm) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	ARG_TRY(fs->ctx, autogain_ok(mode, ppm));
	fs->ag_mode = mode; fs->ag_ppm = ppm;
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_contrast(tsdrgpu_framestage_t *fs, int mode, int clip_centi, int tx, int ty) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	ARG_TRY(fs->ctx, contrast_ok(mode, clip_centi, tx, ty));
	fs->enh.contrast = mode;
	if (mode == TSDRGPU_CONTRAST_CLAHE) { fs->enh.clip_centi = clip_centi; fs->enh.tx = tx; fs->enh.ty = ty; }
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_denoise(tsdrgpu_framestage_t *fs, int mode, int h_milli, int r, int p) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	ARG_TRY(fs->ctx, denoise_ok(mode, h_milli, r, p));
	fs->enh.denoise = mode;
	if (mode == TSDRGPU_DENOISE_NLM) { fs->enh.h_milli = h_milli; fs->enh.r = r; fs->enh.p = p; }
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_deblur(tsdrgpu_framestage_t *fs, int mode, int sigma_centi, int iterations) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	ARG_TRY(fs->ctx, deblur_ok(mode, sigma_centi, iterations));
	fs->enh.deblur = mode;
	if (mode == TSDRGPU_DEBLUR_RL) { fs->enh.sigma_centi = sigma_centi; fs->enh.iters = iterations; }
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_stack(tsdrgpu_framestage_t *fs, int mode, int depth, int rx, int ry) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	ARG_TRY(fs->ctx, stack_ok(mode, depth, rx, ry));
	return stack_set(&fs->enh.stack, mode, depth, rx, ry);
}

int tsdrgpu_framestage_stack_records(tsdrgpu_framestage_t *fs, tsdrgpu_stack_record_t *h_records, int nframes) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	BIND(fs->ctx);
	const StackState &st = fs->enh.stack;
	ARG_TRY(fs->ctx, h_records != NULL && nframes >= 0 && nframes <= st.last_frames && st.d_rec.ptr != NULL);
	CU_TRY(fs->ctx, cudaDeviceSynchronize());
	CU_TRY(fs->ctx, cudaMemcpy(h_records, st.d_rec.ptr, sizeof(tsdrgpu_stack_record_t) * nframes, cudaMemcpyDeviceToHost));
	return TSDRGPU_OK;
}

int framestage_stack_next(tsdrgpu_framestage_t *fs, int restart, tsdrgpu_stack_record_t *h_records_pinned) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	if (restart) fs->enh.stack.m = 0;
	fs->h_stack_next = h_records_pinned;
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_set_overlap(tsdrgpu_framestage_t *fs, int on) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	fs->overlap = on != 0;
	return TSDRGPU_OK;
}

// make `stream` wait for everything this object has queued on its side stream
int tsdrgpu_framestage_join(tsdrgpu_framestage_t *fs, void *stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	BIND(fs->ctx);
	// side_pending stays set once the side stream has been used: every consumer stream that joins (the pipeline's output
	// stream after each batch, the caller's main stream when it leaves the overlapped order) must get its own wait, and a
	// wait on an event that completed long ago costs nothing on the device
	if (fs->side_pending) {
		CU_TRY(fs->ctx, cudaStreamWaitEvent((cudaStream_t) stream, fs->ev_done[0], 0));
		CU_TRY(fs->ctx, cudaStreamWaitEvent((cudaStream_t) stream, fs->ev_done[1], 0));
	}
	return TSDRGPU_OK;
}

static int framestage_run_impl(tsdrgpu_framestage_t *fs, void *stream_, const float *d_in, int nframes, int w, int h,
                               float motionblur, float lowpasscoeff, unsigned flags, float *d_out, tsdrgpu_frame_result_t *h_results,
                               bool synchronise, int32_t *h_report) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, fs != NULL);
	tsdrgpu_ctx_t *ctx = fs->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, nframes > 0 && w > 0 && h > 0 && d_in != NULL && d_out != NULL && d_in != d_out);
	const size_t n = (size_t) w * h;
	const bool autoshift = flags & TSDRGPU_FS_AUTOSHIFT, lpbs = flags & TSDRGPU_FS_LOWPASS_BEFORE_SYNC;
	const bool aap = flags & TSDRGPU_FS_AUTOGAIN_AFTER_PROC, superres = flags & TSDRGPU_FS_SUPERRESOLUTION;
	const bool snr = flags & TSDRGPU_FS_COMPUTE_SNR;
	// the side stream is used for the default order only (low-pass before sync, auto-gain first); anything else is serial
	const bool overlapped = fs->overlap && lpbs && !aap && !(h_results && synchronise);
	int rc;
	if (!overlapped && (rc = tsdrgpu_framestage_join(fs, stream))) return rc;

	// buffer (re)sizing exactly as dsp.c:152-186
	if (h != fs->h || w != fs->w) {
		if ((rc = tsdrgpu_framestage_join(fs, stream))) return rc;
		if (n > fs->d_screen.cap) {
			CU_TRY(ctx, cudaStreamSynchronize(stream));
			{   // the new buffer first, then the old one goes with `nb`: a failed allocation leaves the old buffer and the geometry it
				// was made for in place, so the next call either keeps using both or tries the new geometry again
				DeviceBuf<float> nb;
				CU_TRY(ctx, nb.assign(n));
				fs_exchange(nb, fs->d_screen);
			}
			CU_TRY(ctx, cudaMemsetAsync(fs->d_screen.ptr, 0, sizeof(float) * n, stream));
		}
		fs->h = h; fs->w = w; fs->n = n;
	}
	if (fs->lp_before_sync != (int) lpbs) {
		if ((rc = tsdrgpu_framestage_join(fs, stream))) return rc;
		fs->lp_before_sync = lpbs;
		CU_TRY(ctx, cudaMemsetAsync(fs->d_screen.ptr, 0, sizeof(float) * n, stream));
	}
	const size_t tneed = (size_t) nframes * n;          // fs_reserve reallocates the group of d_t1 and d_t2 when any of them is short
	if (fs->d_t1.cap < tneed || fs->d_t2[0].cap < tneed || fs->d_t2[1].cap < tneed || fs->batch_cap < nframes) {
		if ((rc = tsdrgpu_framestage_join(fs, stream))) return rc;
	}
	if ((rc = fs_reserve(fs, nframes, n, w, h))) return rc;

	const int ph = fs->phase; fs->phase ^= 1;
	float *T2 = fs->d_t2[ph].ptr;
	tsdrgpu_frame_result_t *d_results = fs->d_results[ph].ptr;
	const double fresh = 1.0 - (double) motionblur;      // dsp.c:29
	const int minsize_x = (int) (w * 0.05f), minsize_y = (int) (h * 0.01f);   // syncdetector.c:178-179
	const size_t prep_smem = fs_prep_in_smem(w, h) ? sizeof(double) * ((size_t) w + h + 2) : 0;
	const size_t rec_bytes = sizeof(double) * fs_prep_stride(w, h);
	const size_t rec_smem_max = sizeof(double) * (FS_SMEM_STRIPS + FS_PREP_HDR);
	// prefetch one frame ahead while two records fit beside the main stream's CTAs, else one record at a time while one fits in
	// shared memory, else read them in global memory
	const int sync_nbuf = (2 * rec_bytes <= 96 * 1024) ? 2 : (rec_bytes <= rec_smem_max ? 1 : 0);
	const size_t sync_smem = rec_bytes * sync_nbuf;
	CU_TRY(ctx, cudaFuncSetAttribute(fs_sync_prep<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) (sizeof(double) * FS_SMEM_STRIPS)));
	CU_TRY(ctx, cudaFuncSetAttribute(fs_sync<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) rec_smem_max));
	const int force_serial = getenv("TSDRGPU_SYNC_SERIAL") ? 1 : 0;      // test hook: always take the serial-chain path
	const unsigned gx = grid_for(n, ctx->sm_count, 4);
	const size_t total = (size_t) nframes * n;

	// collapse on `stream`, then sync search on `s2` (== stream unless overlapped)
	auto collapse_sync = [&](const float *src, cudaStream_t s2, const char *name, const unsigned *gate) -> int {
		if ((rc = launch_collapse(ctx, stream, src, w, h, nframes, fs->d_wstrips[ph].ptr, fs->d_hstrips[ph].ptr, fs->collapse_maps, 6, name, gate))) return rc;
		if (s2 != stream) {
			CU_TRY(ctx, cudaEventRecord(fs->ev_ready[ph], stream));
			CU_TRY(ctx, cudaStreamWaitEvent(s2, fs->ev_ready[ph], 0));
		}
		static const bool no_spec = getenv("TSDRGPU_SYNC_NO_SPEC") != NULL;      // test hook: always the literal cluster search
		auto prep_kernel = fs_prep_in_smem(w, h) ? fs_sync_prep<false> : fs_sync_prep<true>;
		KL(ctx, "fs_sync_prep", s2, prep_kernel<<<nframes, FS_SYNC_THREADS, prep_smem, s2>>>(fs->d_wstrips[ph].ptr, fs->d_hstrips[ph].ptr, w, h,
			fs->taps[0], fs->taps[1], fs->taps[2], fs->taps[3], fs->taps[4], force_serial, fs->d_prep.ptr, fs->d_state.ptr, minsize_x, minsize_y, no_spec ? 0 : 1));
		KL(ctx, "fs_sync_walk", s2, fs_sync_walk<<<1, 64, 0, s2>>>(fs->d_prep.ptr, w, h, minsize_x, minsize_y, nframes, fs->d_state.ptr, d_results, fs->d_resume.ptr));
		if (sync_nbuf) KL(ctx, "fs_sync", s2, fs_sync<false><<<FS_SEL_CLUSTER, FS_SEL_THREADS, sync_smem, s2>>>(fs->d_prep.ptr, sync_nbuf, w, h, minsize_x, minsize_y, nframes,
			fs->d_state.ptr, fs->d_chain.ptr, d_results, fs->d_resume.ptr));
		else KL(ctx, "fs_sync", s2, fs_sync<true><<<FS_SEL_CLUSTER, FS_SEL_THREADS, 0, s2>>>(fs->d_prep.ptr, 0, w, h, minsize_x, minsize_y, nframes,
			fs->d_state.ptr, fs->d_chain.ptr, d_results, fs->d_resume.ptr));
		return TSDRGPU_OK;
	};
	// syncdetector_run's output stage: src -> dst (dst != src), or in place on src when allowed
	auto emit = [&](float *src, float *dst, bool greenlines, bool may_modify, float **result, cudaStream_t s2) -> int {
		if (autoshift) {
			if ((w % 4 == 0) && (((reinterpret_cast<unsigned long long>(src) | reinterpret_cast<unsigned long long>(dst)) & 15ull) == 0)) {
				// bands of rows, about one wave of 8 CTAs per SM over the batch
				const int want = (int) ((ctx->sm_count * 8 + nframes - 1) / nframes);
				const int band = (h + (want < h ? want : h) - 1) / (want < h ? want : h), bands = (h + band - 1) / band;
				KL(ctx, "fs_shift", s2, fs_shift4<<<dim3((unsigned) bands, nframes), 256, 0, s2>>>(src, dst, w, h, band, d_results));
			} else KL(ctx, "fs_shift", s2, fs_shift<<<dim3((unsigned) h, nframes), 256, 0, s2>>>(src, dst, w, h, d_results));
			*result = dst;
		} else if (greenlines && may_modify) {
			KL(ctx, "fs_greenlines", s2, fs_greenlines<<<dim3(8, nframes), 256, 0, s2>>>(src, w, h, d_results));
			*result = src;
		} else if (greenlines) {
			if ((rc = fs_copy_async(ctx, s2, src, dst, total))) return rc;
			KL(ctx, "fs_greenlines", s2, fs_greenlines<<<dim3(8, nframes), 256, 0, s2>>>(dst, w, h, d_results));
			*result = dst;
		} else *result = src;
		return TSDRGPU_OK;
	};
	float *res = NULL;
	cudaStream_t tail = stream;                          // the stream the results / output become valid on
	if (lpbs) {                                          // dsp.c:201-212
		const float *lp_in = d_in;
		if (overlapped) CU_TRY(ctx, cudaStreamWaitEvent(stream, fs->ev_done[ph], 0));      // this phase's buffers are free again
		static const bool no_fuse = getenv("TSDRGPU_NO_FUSE") != NULL;
		const bool fuse = !aap && !snr && nframes <= 4096 && !no_fuse;
		if (!aap) {
			if ((rc = fs_autogain_batch(fs, stream, d_in, fuse ? NULL : fs->d_t1.ptr, nframes, n, lowpasscoeff, snr))) return rc;
			lp_in = fs->d_t1.ptr;
			KL(ctx, "fs_results_autogain", stream, fs_results_autogain<<<1, 256, 0, stream>>>(nframes, fs->d_params.ptr, fs->d_state.ptr, d_results,
			                                                                                   fuse ? fs->d_cert.ptr : NULL));
		}
		// motion blur 0: the collapse normalises on load and writes T2 (fs_collapse_tiles<true>); then, gated by the batch's
		// certificate, the literal low-pass from the start-of-batch screen (or, when clear, the screen's update from T2) and the
		// literal collapse of T2
		const bool norm_on_load = fuse && motionblur == 0.0f;
		if (fuse) {
			// one thread per four pixels on the 16-byte path, one per pixel otherwise (odd frame sizes, unaligned input)
			const bool vec = ((n & 3) == 0) && (((reinterpret_cast<unsigned long long>(d_in) | reinterpret_cast<unsigned long long>(T2) | reinterpret_cast<unsigned long long>(fs->d_screen.ptr)) & 15ull) == 0);
			const size_t threads = vec ? n / 4 : n;
			const unsigned grid = (unsigned) ((threads + 255) / 256 ? (threads + 255) / 256 : 1);
			const char *name = norm_on_load ? "fs_redo_lowpass" : "fs_norm_lowpass";
			if (norm_on_load) {
				const NormOnLoad norm = {fs->d_params.ptr, T2, fs->d_cert.ptr};
				if ((rc = launch_collapse(ctx, stream, d_in, w, h, nframes, fs->d_wstrips[ph].ptr, fs->d_hstrips[ph].ptr, fs->collapse_maps, 6,
				                          "fs_collapse", NULL, &norm))) return rc;
				if (vec) KL(ctx, name, stream, (fs_norm_lowpass<true, true><<<grid, 256, sizeof(float2) * nframes, stream>>>(d_in, T2, fs->d_screen.ptr, n, nframes, fs->d_params.ptr, motionblur, fresh, fs->d_cert.ptr)));
				else KL(ctx, name, stream, (fs_norm_lowpass<false, true><<<grid, 256, sizeof(float2) * nframes, stream>>>(d_in, T2, fs->d_screen.ptr, n, nframes, fs->d_params.ptr, motionblur, fresh, fs->d_cert.ptr)));
			} else if (vec) KL(ctx, name, stream, (fs_norm_lowpass<true, false><<<grid, 256, sizeof(float2) * nframes, stream>>>(d_in, T2, fs->d_screen.ptr, n, nframes, fs->d_params.ptr, motionblur, fresh, NULL)));
			else KL(ctx, name, stream, (fs_norm_lowpass<false, false><<<grid, 256, sizeof(float2) * nframes, stream>>>(d_in, T2, fs->d_screen.ptr, n, nframes, fs->d_params.ptr, motionblur, fresh, NULL)));
		}
		else KL(ctx, "fs_timelowpass", stream, fs_timelowpass<<<gx, 256, 0, stream>>>(lp_in, T2, fs->d_screen.ptr, n, nframes, motionblur, fresh));
		if (overlapped) tail = fs->s_side;
		if ((rc = collapse_sync(T2, tail, norm_on_load ? "fs_redo_collapse" : "fs_collapse", norm_on_load ? fs->d_cert.ptr : NULL))) return rc;
		float *dst = aap ? fs->d_t1.ptr : d_out;
		if ((rc = emit(T2, dst, !superres, false, &res, tail))) return rc;
		if (aap) {
			if ((rc = fs_autogain_batch(fs, stream, res, d_out, nframes, n, lowpasscoeff, snr))) return rc;
			KL(ctx, "fs_results_autogain", stream, fs_results_autogain<<<1, 256, 0, stream>>>(nframes, fs->d_params.ptr, fs->d_state.ptr, d_results));
		} else if (res != d_out && (rc = fs_copy_async(ctx, tail, res, d_out, total))) return rc;
	} else {                                             // dsp.c:214-226
		float *work = fs->d_t1.ptr;
		if (!aap) {
			if ((rc = fs_autogain_batch(fs, stream, d_in, fs->d_t1.ptr, nframes, n, lowpasscoeff, snr))) return rc;
			KL(ctx, "fs_results_autogain", stream, fs_results_autogain<<<1, 256, 0, stream>>>(nframes, fs->d_params.ptr, fs->d_state.ptr, d_results));
		} else if ((rc = fs_copy_async(ctx, stream, d_in, fs->d_t1.ptr, total))) return rc;
		if ((rc = collapse_sync(work, stream, "fs_collapse", NULL))) return rc;
		if ((rc = emit(work, T2, (motionblur == 0.0f) && !superres, true, &res, stream))) return rc;
		float *lp_out = aap ? ((res == fs->d_t1.ptr) ? T2 : fs->d_t1.ptr) : d_out;
		KL(ctx, "fs_timelowpass", stream, fs_timelowpass<<<gx, 256, 0, stream>>>(res, lp_out, fs->d_screen.ptr, n, nframes, motionblur, fresh));
		if (aap) {
			if ((rc = fs_autogain_batch(fs, stream, lp_out, d_out, nframes, n, lowpasscoeff, snr))) return rc;
			KL(ctx, "fs_results_autogain", stream, fs_results_autogain<<<1, 256, 0, stream>>>(nframes, fs->d_params.ptr, fs->d_state.ptr, d_results));
		}
	}
	// the stack, deblur, NLM, then CLAHE, on the frames as delivered, after every branch's last step; nothing either does feeds back
	if ((rc = enhance_run(ctx, &fs->enh, tail, d_out, nframes, w, h))) return rc;
	if (fs->h_stack_next && fs->enh.stack.mode != TSDRGPU_STACK_OFF)
		CU_TRY(ctx, cudaMemcpyAsync(fs->h_stack_next, fs->enh.stack.d_rec.ptr, sizeof(tsdrgpu_stack_record_t) * nframes, cudaMemcpyDeviceToHost, tail));
	fs->h_stack_next = NULL;
	if (h_results) CU_TRY(ctx, cudaMemcpyAsync(h_results, d_results, sizeof(tsdrgpu_frame_result_t) * nframes, cudaMemcpyDeviceToHost, tail));
	if (overlapped) {
		CU_TRY(ctx, cudaEventRecord(fs->ev_done[ph], fs->s_side));
		fs->side_pending = 1;
	}
	if (h_results && synchronise) CU_TRY(ctx, cudaStreamSynchronize(tail));
	for (int f = 0; f < nframes; f++) {
		int report = 0;
		if (fs->runs++ > 5) { fs->runs = 0; report = 1; }                              // dsp.c:231-235
		if (h_report) h_report[f] = report;
		if (h_results && synchronise) h_results[f].autogain_report = report;
	}
	return TSDRGPU_OK;
}

int tsdrgpu_framestage_run(tsdrgpu_framestage_t *fs, void *stream, const float *d_in, int nframes, int w, int h,
                           float motionblur, float lowpasscoeff, unsigned flags, float *d_out, tsdrgpu_frame_result_t *h_results) {
	return framestage_run_impl(fs, stream, d_in, nframes, w, h, motionblur, lowpasscoeff, flags, d_out, h_results, true, NULL);
}

int tsdrgpu_framestage_run_async(tsdrgpu_framestage_t *fs, void *stream, const float *d_in, int nframes, int w, int h,
                                 float motionblur, float lowpasscoeff, unsigned flags, float *d_out,
                                 tsdrgpu_frame_result_t *h_results_pinned, int32_t *h_autogain_report) {
	return framestage_run_impl(fs, stream, d_in, nframes, w, h, motionblur, lowpasscoeff, flags, d_out, h_results_pinned, false, h_autogain_report);
}

// ---- stage-level entry points -------------------------------------------------------------------------------
int tsdrgpu_autogain(tsdrgpu_ctx_t *ctx, void *stream_, float *h_lastmax, float *h_lastmin, float *h_snr,
                     int n, const float *d_in, float *d_out, float norm) {
	BIND(ctx);
	ARG_TRY(ctx, n > 0 && d_in && d_out && h_lastmax && h_lastmin);
	cudaStream_t stream = (cudaStream_t) stream_;
	tsdrgpu_framestage_t *fs;
	int rc = tsdrgpu_framestage_create(ctx, &fs);
	if (rc) return rc;
	SyncState s; memset(&s, 0, sizeof s);
	s.lastmax = *h_lastmax; s.lastmin = *h_lastmin; s.snr = h_snr ? *h_snr : 1.0f;
	CU_TRY(ctx, cudaMemcpy(fs->d_state.ptr, &s, sizeof s, cudaMemcpyHostToDevice));
	if ((rc = fs_reserve(fs, 1, 1, 1, 1))) { tsdrgpu_framestage_destroy(fs); return rc; }
	rc = fs_autogain_batch(fs, stream, d_in, d_out, 1, (size_t) n, norm, h_snr != NULL);
	if (rc == TSDRGPU_OK) {
		CU_TRY(ctx, cudaStreamSynchronize(stream));
		CU_TRY(ctx, cudaMemcpy(&s, fs->d_state.ptr, sizeof s, cudaMemcpyDeviceToHost));
		*h_lastmax = s.lastmax; *h_lastmin = s.lastmin; if (h_snr) *h_snr = s.snr;
	}
	tsdrgpu_framestage_destroy(fs);
	return rc;
}

int tsdrgpu_frame_levels(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_frames, uint64_t n, int nframes, int ppm,
                         float *h_lo, float *h_hi, uint64_t *h_valid) {
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_frames && h_lo && h_hi && n > 0 && n <= TSDRGPU_MAX_FRAME_PIXELS && nframes > 0 && nframes <= 65535);
	ARG_TRY(ctx, autogain_ok(TSDRGPU_AG_CLIP, ppm) && (((uintptr_t) d_frames) & 3) == 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	tsdrgpu_framestage_t *fs;
	int rc = tsdrgpu_framestage_create(ctx, &fs);
	if (rc) return rc;
	if (!(rc = fs_reserve(fs, nframes, 1, 1, 1)) && !(rc = fs_select_batch(fs, stream, d_frames, nframes, (size_t) n, ppm, fs_chunks((size_t) n), false))) {
		std::vector<float2> lv(nframes);
		std::vector<SelState> st(nframes);
		cudaError_t e = cudaMemcpyAsync(lv.data(), fs->d_levels.ptr, sizeof(float2) * nframes, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaMemcpyAsync(st.data(), fs->d_sel.ptr, sizeof(SelState) * nframes, cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
		if (e == cudaSuccess) {
			for (int f = 0; f < nframes; f++) { h_lo[f] = lv[f].x; h_hi[f] = lv[f].y; if (h_valid) h_valid[f] = st[f].nvalid; }
		} else rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "tsdrgpu_frame_levels", e, __FILE__, __LINE__);
	}
	tsdrgpu_framestage_destroy(fs);
	return rc;
}

int tsdrgpu_timelowpass(tsdrgpu_ctx_t *ctx, void *stream, float coeff, int n, const float *d_in, float *d_screen) {
	BIND(ctx);
	ARG_TRY(ctx, n > 0 && d_in && d_screen);
	// single frame: the per-frame output IS the screen buffer
	KL(ctx, "fs_timelowpass", (cudaStream_t) stream, fs_timelowpass<<<grid_for((size_t) n, ctx->sm_count, 4), 256, 0, (cudaStream_t) stream>>>(d_in, d_screen, d_screen, (size_t) n, 1, coeff, 1.0 - (double) coeff));
	return TSDRGPU_OK;
}

int tsdrgpu_average_v_h(tsdrgpu_ctx_t *ctx, void *stream, int w, int h, const float *d_in, float *d_wbuf, float *d_hbuf) {
	BIND(ctx);
	ARG_TRY(ctx, w > 0 && h > 0 && d_in && d_wbuf && d_hbuf);
	return launch_collapse(ctx, (cudaStream_t) stream, d_in, w, h, 1, d_wbuf, d_hbuf, NULL, 0);
}

int tsdrgpu_gaussianblur(tsdrgpu_ctx_t *ctx, void *stream, float *d_data, int n) {
	BIND(ctx);
	ARG_TRY(ctx, n > 0 && d_data);
	float t[5];
	tsdrgpu_gauss_taps(t);
	constexpr int smem_n = 2 * 8192;                     // strips kept in shared memory (source and result: 128 KB)
	const int smem_max = (int) (sizeof(float) * 2 * smem_n);
	const bool in_smem = n <= smem_n;
	CU_TRY(ctx, cudaFuncSetAttribute(fs_blur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
	float *scratch = NULL;                               // longer strips: a copy on the stream, allocated and freed in stream order
	if (!in_smem) CU_TRY(ctx, cudaMallocAsync((void **) &scratch, sizeof(float) * (size_t) n, (cudaStream_t) stream));
	fs_blur_kernel<<<1, 256, in_smem ? sizeof(float) * 2 * n : 0, (cudaStream_t) stream>>>(d_data, scratch, n, t[0], t[1], t[2], t[3], t[4]);
	const cudaError_t launched = cudaGetLastError();
	if (scratch) CU_TRY(ctx, cudaFreeAsync(scratch, (cudaStream_t) stream));
	if (launched != cudaSuccess) return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "kernel launch", launched, __FILE__, __LINE__);
	ctx->launches++;
	return TSDRGPU_OK;
}

int tsdrgpu_pixels_argb(tsdrgpu_ctx_t *ctx, void *stream, const float *d_frame, int n, int inverted, int32_t *d_argb) {
	BIND(ctx);
	ARG_TRY(ctx, n > 0 && d_frame && d_argb);
	fs_argb<<<grid_for((size_t) n, ctx->sm_count), 256, 0, (cudaStream_t) stream>>>(d_frame, n, inverted, d_argb);
	LAUNCH_CHECK(ctx);
	return TSDRGPU_OK;
}

int tsdrgpu_pixels_argb_batch(tsdrgpu_ctx_t *ctx, void *stream, float *d_frames_inout, uint64_t n, int nframes, int inverted, int32_t *d_last) {
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, n > 0 && nframes > 0 && d_frames_inout && d_last);
	KL(ctx, "fs_argb_batch", (cudaStream_t) stream, fs_argb_batch<<<grid_for((size_t) n, ctx->sm_count), 256, 0, (cudaStream_t) stream>>>(d_frames_inout, (size_t) n, nframes, inverted, d_last));
	return TSDRGPU_OK;
}

}  // extern "C"
