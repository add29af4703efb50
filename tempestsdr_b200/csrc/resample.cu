// resample.cu -- a2 + a6: AM demodulation fused with the reference's area-weighted box resampler.
//
// Replaces am_demod (TSDRLibrary.c:244-262) and dsp_resample_process (dsp.c:256-307), bit-exact.
//
// How a serial loop becomes a data-parallel kernel
// ------------------------------------------------
// The reference walks samples k = 0..size-1 keeping `pid`, the next pixel to complete.  Sample k covers
//     lo_k = fl(fl(k*r) + phase),  hi_k = fl(lo_k + r),  c_k = fl(hi_k - 1)           (dsp.c:282-284)
// on the pixel axis.  After sample k, pid == P(k) := max(0, ceil(c_k)) -- a closed form, because c_k is
// monotone in k.  So sample k emits pixels P(k-1) .. P(k)-1:
//     the first one is an "A" pixel,  float(bank + v_k*((1-lo_k)+p)),   iff p < lo_k && p < c_k  (dsp.c:288-292)
//     all others are "B" pixels,      v_k                                                    (dsp.c:294-297)
// and then banks t_k = (P(k) < hi_k && P(k) > lo_k) ? (hi_k-P(k))*v_k : r*v_k               (dsp.c:299-302).
// `bank` before sample k is the left-to-right double sum of t_j since the last A pixel (where it is zeroed):
// for r > 1 that is just t_{k-1}; the general case walks back until it meets an A sample.  Everything except
// the sample values is data-independent, and all double operations are issued as separate IEEE
// round-to-nearest instructions (no FMA contraction), so every pixel is bit-identical to gcc's x86-64 result.
//
// Only one pixel per decimator block cannot be produced locally: the first A pixel, whose bank reaches back
// into the previous block (or into the carried `contrib` state).  A small second kernel (rs_fixup) resolves
// those, fills slots the reference leaves stale, and writes the new `contrib`.
//
// Memory plan: 8 B read per IQ pair (ld.global.nc, L1 no-allocate), magnitudes staged once in shared memory,
// pixels assembled in shared memory and written back as full contiguous runs.  Algorithmic traffic:
// 8 B + 4*r B per sample (~16 B at r ~ 2).  Bound: HBM.
#include "common.cuh"
#include "host_plan.h"

namespace {

constexpr int RS_TILE = 2048;        // samples per CTA tile
constexpr int RS_THREADS = 256;
constexpr int RS_HALO = 8;           // samples before the tile kept in smem for short bank chains
constexpr int RS_OUT_CAP = 3 * RS_TILE + 16;   // pixels staged per tile (r <= 3); larger ratios store directly

struct RsBlock { unsigned long long in_start, out_start; unsigned size, n_out; double r, phase; };
static_assert(sizeof(RsBlock) == sizeof(tsdrgpu_rs_block_t), "device/host block layout");

struct Geo { double lo, hi, c; };

__device__ __forceinline__ Geo rs_geo(unsigned k, double r, double phase) {
	Geo g;
	g.lo = __dadd_rn(__dmul_rn((double) k, r), phase);
	g.hi = __dadd_rn(g.lo, r);
	g.c = __dadd_rn(g.hi, -1.0);
	return g;
}
// pid after a sample whose c is `c`, as a double holding an exact non-negative integer
__device__ __forceinline__ double rs_P(double c) { return fmax(0.0, ceil(c)); }

template <bool IQ>
__device__ __forceinline__ float rs_load(const float *in, unsigned long long idx) {
	if (IQ) { const float2 v = ldg_stream_f2(reinterpret_cast<const float2 *>(in) + idx); return mag_exact(v.x, v.y); }
	return ldg_stream_f1(in + idx);
}

// what sample k leaves in the bank (dsp.c:299-302)
__device__ __forceinline__ double rs_t(const Geo &g, double Pk, double r, double v) {
	if (Pk < g.hi && Pk > g.lo) return __dmul_rn(__dsub_rn(g.hi, Pk), v);
	return __dmul_rn(r, v);
}
__device__ __forceinline__ void sts_f32_if(unsigned addr, float v, bool p) {
	asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %2, 0;\n\t@q st.shared.f32 [%0], %1;\n\t}" :: "r"(addr), "f"(v), "r"((int) p) : "memory");
}
__device__ __forceinline__ void sts_f32(unsigned addr, float v) { asm volatile("st.shared.f32 [%0], %1;" :: "r"(addr), "f"(v) : "memory"); }
// does sample k emit an A pixel?  (dsp.c:288)
__device__ __forceinline__ bool rs_isA(const Geo &g, double Pkm1) { return Pkm1 < g.lo && Pkm1 < g.c; }

// -------------------------------------------------------------------------------------------------------------
template <bool IQ>
__global__ void __launch_bounds__(RS_THREADS) rs_main(const float *__restrict__ in, float *__restrict__ out,
                                                      const RsBlock *__restrict__ blocks,
                                                      const uint2 *__restrict__ tile_info /* {block, first sample} per tile */,
                                                      float *__restrict__ mag_out /* optional: |x| of every input sample, same indexing as `in` */) {
	__shared__ float s_mag[RS_HALO + RS_TILE];
	__shared__ __align__(16) float s_out[RS_OUT_CAP + 8];

	const uint2 ti = tile_info[blockIdx.x];
	const RsBlock B = blocks[ti.x];
	const unsigned s0 = ti.y;
	const unsigned s1 = min(s0 + (unsigned) RS_TILE, B.size);
	const unsigned halo = min((unsigned) RS_HALO, s0);
	const double r = B.r, phase = B.phase;

	// stage magnitudes (demod fused): s_mag[RS_HALO + (k - s0)] = |x_k|.  Loads are issued 8 deep per thread.
	{
		const unsigned n_load = (s1 - s0) + halo;
		const unsigned long long first = B.in_start + s0 - halo;
		float *dst = s_mag + (RS_HALO - halo);
		#pragma unroll 8
		for (unsigned i = threadIdx.x; i < n_load; i += RS_THREADS) {
			const float m = rs_load<IQ>(in, first + i);
			dst[i] = m;
			if (IQ && mag_out != NULL && i >= halo) mag_out[first + i] = m;      // the demodulated stream, for the frame-rate detector
		}
	}
	const double pbase_d = (s0 == 0) ? 0.0 : rs_P(rs_geo(s0 - 1, r, phase).c);
	const double pend_d = rs_P(rs_geo(s1 - 1, r, phase).c);
	const unsigned pbase = (unsigned) pbase_d;
	const unsigned pend = (unsigned) pend_d;
	const bool staged = (pend - pbase) <= (unsigned) RS_OUT_CAP;
	float *gout = out + B.out_start;
	// staging index = (p - pbase) + aoff, chosen so that shared and global addresses are congruent modulo 16 bytes
	const unsigned aoff = (unsigned) ((reinterpret_cast<unsigned long long>(gout + pbase) >> 2) & 3ull);
	float *sq = s_out + aoff;
	const unsigned sq_addr = (unsigned) __cvta_generic_to_shared(s_out) + (aoff << 2);      // array base folds to a constant
	__syncthreads();

	// One warp owns 256 CONSECUTIVE samples, 32 per round: what sample k needs from sample k-1 (its pid, whether it emitted
	// an A pixel, what it banked) arrives by warp shuffle, or from the previous round's lane 31.
	const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const unsigned wbase = s0 + warp * (RS_TILE / (RS_THREADS / 32));
	if (wbase < s1) {
		// "the sample before" lives in lane 31's old* registers: in round 0 it is sample wbase-1, later the previous round's
		// lane 31.  One rotate-by-one shuffle per quantity then serves every lane (lane 31 contributes its OLD value, which
		// nobody else needs this round; lane 0 receives it).
		double oldP = 0.0, oldT = 0.0; int oldA = 0;
		if (wbase > 0) {                                         // the sample just before this warp's range (once per warp)
			const unsigned kp = wbase - 1;
			const Geo gp = rs_geo(kp, r, phase);
			oldP = rs_P(gp.c);
			const double Ppm1 = (kp == 0) ? 0.0 : rs_P(rs_geo(kp - 1, r, phase).c);
			oldA = rs_isA(gp, Ppm1);
			const float vp = (kp + RS_HALO >= s0) ? s_mag[RS_HALO + kp - s0] : rs_load<IQ>(in, B.in_start + kp);
			oldT = rs_t(gp, oldP, r, (double) vp);
		}
		const unsigned wend = min(wbase + (unsigned) (RS_TILE / (RS_THREADS / 32)), s1);
		const unsigned from = (lane + 31u) & 31u;
		const bool is_last = lane == 31u;
		double kd = (double) (wbase + lane);                     // exact; advanced by 32.0 per round instead of converted
		const float *sm = s_mag + RS_HALO + (wbase - s0) + lane;
		for (unsigned base = wbase; base < wend; base += 32, kd = __dadd_rn(kd, 32.0), sm += 32) {
			const unsigned k = base + lane;
			Geo g;
			g.lo = __dadd_rn(__dmul_rn(kd, r), phase);
			g.hi = __dadd_rn(g.lo, r);
			g.c = __dadd_rn(g.hi, -1.0);
			double Pk = ceil(g.c);                               // == rs_P: fmax(0, ceil(c))
			if (!(g.c > 0.0)) Pk = 0.0;
			const float vf = *sm;                                // lanes past the tile's end read a valid slot; their results are unused
			const double v = (double) vf;
			const double tk = __dmul_rn((Pk < g.hi && Pk > g.lo) ? __dsub_rn(g.hi, Pk) : r, v);     // == rs_t
			const double Pkm1 = __shfl_sync(0xffffffffu, is_last ? oldP : Pk, from);
			const bool isA = rs_isA(g, Pkm1);
			const int prevA = __shfl_sync(0xffffffffu, is_last ? oldA : (int) isA, from);
			const double prevT = __shfl_sync(0xffffffffu, is_last ? oldT : tk, from);
			oldP = Pk; oldA = (int) isA; oldT = tk;
			if (k >= s1) continue;
			const unsigned p0 = (unsigned) Pkm1, cnt = (unsigned) Pk - p0;
			float first = vf;
			bool write_first = true;
			if (isA) {
				double bank = 0.0;
				bool have = false;
				if (k > 0 && prevA) { bank = __dadd_rn(0.0, prevT); have = true; }      // the common case for r > 1
				else if (k > 0) {
					// general case: bank = t_L + ... + t_{k-1}, L = latest earlier sample that emitted an A pixel
					long long L = (long long) k - 2;
					while (L >= 0) {
						const Geo gl = rs_geo((unsigned) L, r, phase);
						const double Plm1 = (L == 0) ? 0.0 : rs_P(rs_geo((unsigned) L - 1, r, phase).c);
						if (rs_isA(gl, Plm1)) break;
						L--;
					}
					if (L >= 0) {
						for (unsigned j = (unsigned) L; j < k; j++) {
							const Geo gj = rs_geo(j, r, phase);
							const float vj = (j + RS_HALO >= s0) ? s_mag[RS_HALO + j - s0] : rs_load<IQ>(in, B.in_start + j);
							bank = __dadd_rn(bank, rs_t(gj, rs_P(gj.c), r, (double) vj));
						}
						have = true;
					}
				}
				if (have) {
					const double w = __dadd_rn(__dsub_rn(1.0, g.lo), Pkm1);
					first = __double2float_rn(__dadd_rn(bank, __dmul_rn(v, w)));
				} else write_first = false;      // the bank reaches past the block start -> rs_fixup writes this pixel
			}
			if (staged) {
				const unsigned d = sq_addr + ((p0 - pbase) << 2);   // 32-bit shared address: one add per store
				if (cnt > 0 && write_first) sts_f32(d, first);
				if (cnt > 1) sts_f32(d + 4, vf);
				if (cnt > 2) sts_f32(d + 8, vf);
				for (unsigned c = 3; c < cnt; c++) sts_f32(d + 4 * c, vf);
			} else {
				for (unsigned c = 0; c < cnt; c++) {
					const unsigned p = p0 + c;
					if (p < B.n_out && (c > 0 || write_first)) gout[p] = c ? vf : first;
				}
			}
		}
	}
	if (!staged) return;
	__syncthreads();
	// write the assembled run of pixels: scalar head to a 16-byte boundary, float4 body, scalar tail
	const unsigned pe = min(pend, B.n_out);
	if (pe <= pbase) return;
	const unsigned count = pe - pbase;
	float *gdst = gout + pbase;
	const unsigned head = min((4u - aoff) & 3u, count);
	if (threadIdx.x < head) gdst[threadIdx.x] = sq[threadIdx.x];
	const unsigned body4 = (count - head) >> 2;
	const float4 *s4 = reinterpret_cast<const float4 *>(sq + head);
	float4 *g4 = reinterpret_cast<float4 *>(gdst + head);
	for (unsigned q = threadIdx.x; q < body4; q += RS_THREADS) g4[q] = s4[q];
	const unsigned done = head + (body4 << 2);
	if (threadIdx.x < count - done) gdst[done + threadIdx.x] = sq[done + threadIdx.x];
}

// -------------------------------------------------------------------------------------------------------------
// rs_main4: the same function as rs_main, laid out for fewer instructions per sample (rs_main: 156 per sample, issue-slot bound
// well below the HBM roofline).  A thread owns FOUR consecutive samples:
//   * it loads them itself with two 16-byte loads (IQ) / one (magnitudes) straight from global memory -- groups are aligned on
//     the ADDRESS, so a tile may start up to three samples early; those samples only serve as "the sample before" -- and writes
//     their magnitudes back with one 16-byte store where the address allows: no staging of the input in shared memory at all;
//   * what sample k needs from sample k-1 (its pid, whether it emitted an A pixel, what it banked) is in the thread's own
//     registers for three samples out of four; the fourth comes from the lane below with one shuffle per quantity, lane 0 works
//     it out for itself (once per 128 samples);
//   * everything else -- closed-form pid, exact double operations, pixel assembly in shared memory, 16-byte stores of the
//     finished run -- is rs_main's.  Bit-identical output (same tests, and TSDRGPU_RS_V1=1 switches back to rs_main).
// The rare sample whose bank is not simply what the previous sample left (r <= 1, or a landing within one ulp of a pixel edge)
// goes through rs_bank_walk, out of line.
template <bool IQ>
__device__ __noinline__ bool rs_bank_walk(const float *__restrict__ in, unsigned long long in_start, double r, double phase, unsigned k, double *bank_out) {
	long long L = (long long) k - 2;
	while (L >= 0) {
		const Geo gl = rs_geo((unsigned) L, r, phase);
		const double Plm1 = (L == 0) ? 0.0 : rs_P(rs_geo((unsigned) L - 1, r, phase).c);
		if (rs_isA(gl, Plm1)) break;
		L--;
	}
	if (L < 0) return false;                             // the bank reaches past the block start -> rs_fixup writes this pixel
	double bank = 0.0;
	for (unsigned j = (unsigned) L; j < k; j++) {
		const Geo gj = rs_geo(j, r, phase);
		bank = __dadd_rn(bank, rs_t(gj, rs_P(gj.c), r, (double) rs_load<IQ>(in, in_start + j)));
	}
	*bank_out = bank;
	return true;
}

template <bool IQ, int MINB>
__global__ void __launch_bounds__(RS_THREADS, MINB) rs_main4(const float *__restrict__ in, float *__restrict__ out,
                                                       const RsBlock *__restrict__ blocks, const uint2 *__restrict__ tile_info,
                                                       float *__restrict__ mag_out) {
	__shared__ __align__(16) float s_out[RS_OUT_CAP + 8];
	const uint2 ti = tile_info[blockIdx.x];
	const RsBlock B = blocks[ti.x];
	// Tiles are windows of RS_TILE samples aligned on the input ADDRESS (16 bytes; the host cuts a block's first tile short by
	// `shift` samples so that every later tile starts aligned): the window starts `shift` samples before s0, and the samples
	// in front of s0 only serve as "the sample before".  Two rounds of 128 samples per warp cover the window exactly.
	const unsigned s0 = ti.y;
	const float *tile_in = in + (IQ ? 2ull : 1ull) * (B.in_start + s0);
	const int shift = IQ ? (int) ((reinterpret_cast<unsigned long long>(tile_in) >> 3) & 1ull) : (int) ((reinterpret_cast<unsigned long long>(tile_in) >> 2) & 3ull);
	const unsigned s1 = min(s0 - (unsigned) shift + (unsigned) RS_TILE, B.size);
	const double r = B.r, phase = B.phase;
	const unsigned long long in_start = B.in_start;
	const double pbase_d = (s0 == 0) ? 0.0 : rs_P(rs_geo(s0 - 1, r, phase).c);
	const unsigned pbase = (unsigned) pbase_d, pend = (unsigned) rs_P(rs_geo(s1 - 1, r, phase).c);
	float *gout = out + B.out_start;
	const unsigned aoff = (unsigned) ((reinterpret_cast<unsigned long long>(gout + pbase) >> 2) & 3ull);
	float *sq = s_out + aoff;
	const unsigned sq_addr = (unsigned) __cvta_generic_to_shared(s_out) + (aoff << 2);
	const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const int size = (int) B.size;
	constexpr int ROUNDS = RS_TILE / (RS_THREADS * 4);       // 2
	// ---- all loads of the tile first (four 16-byte loads in flight per thread), then the magnitudes
	float vf[ROUNDS][4];
	{
		float4 raw[ROUNDS][IQ ? 2 : 1];
		bool fast[ROUNDS];
		#pragma unroll
		for (int rd = 0; rd < ROUNDS; rd++) {
			const int k0 = (int) s0 - shift + rd * (RS_THREADS * 4) + (int) warp * 128 + 4 * (int) lane;
			fast[rd] = k0 >= 0 && k0 + 3 < size;
			if (fast[rd]) {
				if (IQ) {
					const float4 *p4 = reinterpret_cast<const float4 *>(in + 2ull * (in_start + (unsigned) k0));
					raw[rd][0] = ldg_stream_f4(p4); raw[rd][IQ ? 1 : 0] = ldg_stream_f4(p4 + 1);
				} else raw[rd][0] = ldg_stream_f4(reinterpret_cast<const float4 *>(in + in_start + (unsigned) k0));
			}
		}
		#pragma unroll
		for (int rd = 0; rd < ROUNDS; rd++) {
			const int k0 = (int) s0 - shift + rd * (RS_THREADS * 4) + (int) warp * 128 + 4 * (int) lane;
			if (fast[rd]) {
				if (IQ) {
					const float4 a = raw[rd][0], b = raw[rd][IQ ? 1 : 0];
					vf[rd][0] = mag_exact(a.x, a.y); vf[rd][1] = mag_exact(a.z, a.w); vf[rd][2] = mag_exact(b.x, b.y); vf[rd][3] = mag_exact(b.z, b.w);
				} else { const float4 a = raw[rd][0]; vf[rd][0] = a.x; vf[rd][1] = a.y; vf[rd][2] = a.z; vf[rd][3] = a.w; }
			} else {
				#pragma unroll
				for (int j = 0; j < 4; j++) vf[rd][j] = (k0 + j >= 0 && k0 + j < size) ? rs_load<IQ>(in, in_start + (unsigned) (k0 + j)) : 0.0f;
			}
		}
	}
	#pragma unroll
	for (int rd = 0; rd < ROUNDS; rd++) {
		const int k0 = (int) s0 - shift + rd * (RS_THREADS * 4) + (int) warp * 128 + 4 * (int) lane;
		if (k0 - 4 * (int) lane >= (int) s1) break;           // the whole warp is past the tile's end (uniform per warp)
		const float *v4 = vf[rd];
		if (IQ && mag_out != NULL) {                          // the demodulated stream, for the frame-rate detector: owned samples only
			float *m = mag_out + ((long long) in_start + k0);   // (k0 may be negative: the pointer is only dereferenced under the masks below)
			const bool all_owned = k0 >= (int) s0 && k0 + 3 < (int) s1;
			const unsigned ma = (unsigned) ((reinterpret_cast<unsigned long long>(m) >> 2) & 3ull);
			if (all_owned && ma == 0) *reinterpret_cast<float4 *>(m) = make_float4(v4[0], v4[1], v4[2], v4[3]);
			else if (all_owned && ma == 2) { *reinterpret_cast<float2 *>(m) = make_float2(v4[0], v4[1]); *reinterpret_cast<float2 *>(m + 2) = make_float2(v4[2], v4[3]); }
			else {
				#pragma unroll
				for (int j = 0; j < 4; j++) if (k0 + j >= (int) s0 && k0 + j < (int) s1) m[j] = v4[j];
			}
		}
		// ---- geometry of the four samples (dsp.c:282-284), all exact single IEEE operations
		const double kd0 = (double) k0;
		double lo[4], hi[4], cc[4], P[4], T[4];
		#pragma unroll
		for (int j = 0; j < 4; j++) {
			const double kd = (j == 0) ? kd0 : __dadd_rn(kd0, (double) j);      // exact
			lo[j] = __dadd_rn(__dmul_rn(kd, r), phase);
			hi[j] = __dadd_rn(lo[j], r);
			cc[j] = __dadd_rn(hi[j], -1.0);
			double pk = ceil(cc[j]);
			if (!(cc[j] > 0.0)) pk = 0.0;                     // == rs_P
			P[j] = pk;
			T[j] = __dmul_rn((pk < hi[j] && pk > lo[j]) ? __dsub_rn(hi[j], pk) : r, (double) v4[j]);      // == rs_t
		}
		// ---- the sample before this thread's first one: from the lane below, lane 0 works it out itself
		const int a3 = (P[2] < lo[3] && P[2] < cc[3]) ? 1 : 0;            // does this thread's last sample emit an A pixel?  (dsp.c:288)
		double Pm = __shfl_up_sync(0xffffffffu, P[3], 1), Tm = __shfl_up_sync(0xffffffffu, T[3], 1);
		int Am = __shfl_up_sync(0xffffffffu, a3, 1);
		if (lane == 0) {
			Pm = 0.0; Tm = 0.0; Am = 0;
			if (k0 > 0) {
				const unsigned kp = (unsigned) k0 - 1;
				const Geo gp = rs_geo(kp, r, phase);
				Pm = rs_P(gp.c);
				Am = rs_isA(gp, kp == 0 ? 0.0 : rs_P(rs_geo(kp - 1, r, phase).c)) ? 1 : 0;
				Tm = rs_t(gp, Pm, r, (double) rs_load<IQ>(in, in_start + kp));
			}
		}
		const double Pprev[4] = {Pm, P[0], P[1], P[2]}, Tprev[4] = {Tm, T[0], T[1], T[2]};
		bool A[4];
		#pragma unroll
		for (int j = 0; j < 4; j++) A[j] = Pprev[j] < lo[j] && Pprev[j] < cc[j];
		const bool Aprev[4] = {Am != 0, A[0], A[1], A[2]};
		// ---- emit: sample k owns pixels P(k-1) .. P(k)-1 (see the header of this file).  Straight-line code: the A value is
		// computed for every sample and selected, the stores are predicated instructions (r <= 2: at most three pixels per
		// sample); the only branch left is the rare bank walk.
		#pragma unroll
		for (int j = 0; j < 4; j++) {
			const int k = k0 + j;
			const double Pkm1 = Pprev[j];
			const bool own = k >= (int) s0 && k < (int) s1;   // not owned: alignment lead-in, or past the tile's end
			const unsigned p0 = (unsigned) Pkm1, cnt = (unsigned) P[j] - p0;
			double bank = __dadd_rn(0.0, Tprev[j]);           // the common case for r > 1: what the previous sample left
			bool have = k > 0 && Aprev[j];
			if (A[j] && !Aprev[j] && k > 0 && own) have = rs_bank_walk<IQ>(in, in_start, r, phase, (unsigned) k, &bank);   // rare
			const float aval = __double2float_rn(__dadd_rn(bank, __dmul_rn((double) v4[j], __dadd_rn(__dsub_rn(1.0, lo[j]), Pkm1))));
			const float first = A[j] ? aval : v4[j];
			// an A pixel whose bank reaches past the block start is left to rs_fixup (have == false)
			const unsigned d = sq_addr + ((p0 - pbase) << 2);
			sts_f32_if(d, first, own && cnt > 0 && (!A[j] || have));
			sts_f32_if(d + 4, v4[j], own && cnt > 1);
			sts_f32_if(d + 8, v4[j], own && cnt > 2);
		}
	}
	__syncthreads();
	// write the assembled run of pixels: scalar head to a 16-byte boundary, float4 body, scalar tail
	const unsigned pe = min(pend, B.n_out);
	if (pe <= pbase) return;
	const unsigned count = pe - pbase;
	float *gdst = gout + pbase;
	const unsigned head = min((4u - aoff) & 3u, count);
	if (threadIdx.x < head) gdst[threadIdx.x] = sq[threadIdx.x];
	const unsigned body4 = (count - head) >> 2;
	const float4 *s4 = reinterpret_cast<const float4 *>(sq + head);
	float4 *g4 = reinterpret_cast<float4 *>(gdst + head);
	for (unsigned q = threadIdx.x; q < body4; q += RS_THREADS) g4[q] = s4[q];
	const unsigned done = head + (body4 << 2);
	if (threadIdx.x < count - done) gdst[done + threadIdx.x] = sq[done + threadIdx.x];
}

// -------------------------------------------------------------------------------------------------------------
// One CTA.  Resolves the per-block quantities that cross block boundaries (see header comment).
template <bool IQ>
__global__ void __launch_bounds__(256) rs_fixup(const float *__restrict__ in, float *__restrict__ out,
                                                const RsBlock *__restrict__ blocks, unsigned nblocks,
                                                double *__restrict__ bank_in /* nblocks+1 */, int *__restrict__ has_a,
                                                double *contrib_state) {
	// 1. per block: bank left at the end of the block, if the block contains an A sample
	for (unsigned b = threadIdx.x; b < nblocks; b += blockDim.x) {
		const RsBlock B = blocks[b];
		long long L = (long long) B.size - 1;
		while (L >= 0) {
			const Geo gl = rs_geo((unsigned) L, B.r, B.phase);
			const double Plm1 = (L == 0) ? 0.0 : rs_P(rs_geo((unsigned) L - 1, B.r, B.phase).c);
			if (rs_isA(gl, Plm1)) break;
			L--;
		}
		if (L >= 0) {
			double bank = 0.0;
			for (unsigned j = (unsigned) L; j < B.size; j++) {
				const Geo gj = rs_geo(j, B.r, B.phase);
				bank = __dadd_rn(bank, rs_t(gj, rs_P(gj.c), B.r, (double) rs_load<IQ>(in, B.in_start + j)));
			}
			bank_in[b + 1] = bank;
			has_a[b] = 1;
		} else has_a[b] = 0;
	}
	if (threadIdx.x == 0) bank_in[0] = *contrib_state;
	int missing = 0;
	for (unsigned b = threadIdx.x; b < nblocks; b += blockDim.x) missing |= !has_a[b];      // own writes
	missing = __syncthreads_or(missing);
	// 2. blocks without any A sample pass the incoming bank through (serial, practically never taken)
	if (threadIdx.x == 0 && !missing) *contrib_state = bank_in[nblocks];
	if (threadIdx.x == 0 && missing) {
		for (unsigned b = 0; b < nblocks; b++) {
			if (has_a[b]) continue;
			const RsBlock B = blocks[b];
			double bank = bank_in[b];
			for (unsigned j = 0; j < B.size; j++) {
				const Geo gj = rs_geo(j, B.r, B.phase);
				bank = __dadd_rn(bank, rs_t(gj, rs_P(gj.c), B.r, (double) rs_load<IQ>(in, B.in_start + j)));
			}
			bank_in[b + 1] = bank;
		}
		*contrib_state = bank_in[nblocks];
	}
	__syncthreads();
	// 3. first A pixel of every block, and slots the reference's loop never writes
	for (unsigned b = threadIdx.x; b < nblocks; b += blockDim.x) {
		const RsBlock B = blocks[b];
		double bank = bank_in[b];
		for (unsigned k = 0; k < B.size; k++) {
			const Geo g = rs_geo(k, B.r, B.phase);
			const double Pkm1 = (k == 0) ? 0.0 : rs_P(rs_geo(k - 1, B.r, B.phase).c);
			const double v = (double) rs_load<IQ>(in, B.in_start + k);
			if (rs_isA(g, Pkm1)) {
				const double w = __dadd_rn(__dsub_rn(1.0, g.lo), Pkm1);
				const unsigned p = (unsigned) Pkm1;
				if (p < B.n_out) out[B.out_start + p] = __double2float_rn(__dadd_rn(bank, __dmul_rn(v, w)));
				break;
			}
			bank = __dadd_rn(bank, rs_t(g, rs_P(g.c), B.r, v));
		}
		const unsigned emitted = (unsigned) rs_P(rs_geo(B.size - 1, B.r, B.phase).c);
		for (unsigned p = emitted; p < B.n_out; p++) out[B.out_start + p] = 0.0f;   // stale in the reference
	}
}

// nearest-neighbour mode (dsp.c:274-276): out[p] = x[(size*p)/output_samples]
template <bool IQ>
__global__ void __launch_bounds__(256) rs_nearest(const float *__restrict__ in, float *__restrict__ out,
                                                  const RsBlock *__restrict__ blocks) {
	const RsBlock B = blocks[blockIdx.y];
	for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < B.n_out; p += gridDim.x * blockDim.x) {
		const unsigned long long src = ((unsigned long long) B.size * p) / B.n_out;
		out[B.out_start + p] = rs_load<IQ>(in, B.in_start + src);
	}
}

// -------------------------------------------------------------------------------------------------------------
// Windowed-sinc mode (definition, delay and history in tsdrgpu.h).  A CTA computes a tile of up to `pt` consecutive pixels
// of one block.  It stages the magnitudes its taps need in shared memory (IQ demodulated on load) and reads the taps
// through L1: the 16 KB table is shared by every CTA on an SM, so staging it per CTA would cost more L2 traffic than the
// tile's own IQ.  The warp's 32 consecutive pixels touch few phase rows (at r ~ 2 two clusters of rows ~L/2 apart, each a
// row or two wide), so a tap load is one or two distinct lines, broadcast to the lanes.
//
// Magnitude output: the newest tap of pixel p is K(p) = k0(p) + T/2, non-decreasing in p.  The tile [p_lo, p_hi) owns
// samples [K(p_lo), K(p_hi)) (clamped at 0; the block's first tile from 0, its last to `size`), so the tiles of a block
// partition its samples and every magnitude is written exactly once.
constexpr int SINC_T = TSDRGPU_SINC_TAPS, SINC_L = TSDRGPU_SINC_PHASES, SINC_D = TSDRGPU_SINC_DELAY, SINC_H = TSDRGPU_SINC_HISTORY;
constexpr int SINC_THREADS = 256;
constexpr int SINC_SCAP = 4096 + 64;          // staged samples per CTA
constexpr int SINC_PT_MAX = 4096;             // pixels per CTA
static_assert(SINC_T == 16, "rs_sinc loads a phase row as four float4");

// pixels per tile at ratio r: the staged span is at most (pt + 1.5)/r + T + 8 samples (tile edges, the rounding of k0, and the
// last tile's samples past its last pixel's newest tap), which must fit SINC_SCAP
static unsigned sinc_pixels_per_tile(double r) {
	const double pt = floor((double) (SINC_SCAP - SINC_T - 16) * r - 2.0);
	return pt >= (double) SINC_PT_MAX ? (unsigned) SINC_PT_MAX : (unsigned) pt;
}

__device__ __forceinline__ long long sinc_pos(unsigned p, double phase, double rinv, int *j_out) {
	const double q = __dsub_rn(__dmul_rn(__dsub_rn(__dadd_rn((double) p, 0.5), phase), rinv), 0.5 + (double) SINC_D);
	double k0 = floor(q);
	int j = (int) __dadd_rn(__dmul_rn(__dsub_rn(q, k0), (double) SINC_L), 0.5);
	if (j == SINC_L) { j = 0; k0 = __dadd_rn(k0, 1.0); }
	*j_out = j;
	return (long long) k0;
}

template <bool IQ>
__global__ void __launch_bounds__(SINC_THREADS) rs_sinc(const float *__restrict__ in, float *__restrict__ out,
                                                        const RsBlock *__restrict__ blocks, const uint2 *__restrict__ tile_info /* {block, first pixel} */,
                                                        unsigned pt, const float4 *__restrict__ taps /* [L][T/4] */,
                                                        const float *__restrict__ hist_in, float *__restrict__ hist_out,
                                                        unsigned long long run_samples, float *__restrict__ mag_out) {
	__shared__ float s_x[SINC_SCAP];
	const uint2 ti = tile_info[blockIdx.x];
	const RsBlock B = blocks[ti.x];
	const double rinv = __drcp_rn(B.r), phase = B.phase;
	const unsigned p_lo = ti.y, p_hi = min(p_lo + pt, B.n_out);
	int jj;
	const long long first_lo = sinc_pos(p_lo, phase, rinv, &jj) - (SINC_T / 2 - 1);                 // oldest tap of the first pixel
	const long long newest_hi = sinc_pos(p_hi - 1, phase, rinv, &jj) + SINC_T / 2;                  // newest tap of the last pixel
	const long long own_lo = (p_lo == 0) ? 0 : max(0ll, first_lo + (SINC_T - 1));
	const long long own_hi = (p_hi == B.n_out) ? (long long) B.size : max(0ll, sinc_pos(p_hi, phase, rinv, &jj) + SINC_T / 2);
	const long long st_lo = min(own_lo, first_lo), st_hi = max(own_hi, newest_hi + 1);
	const int n_st = (int) (st_hi - st_lo);
	const long long base = (long long) B.in_start + st_lo;                                          // >= -H (r >= TSDRGPU_SINC_MIN_RATIO)
	#pragma unroll 4
	for (int i = threadIdx.x; i < n_st; i += SINC_THREADS) {
		const long long g = base + i;
		float v;
		if (g < 0) v = hist_in[SINC_H + g];
		else {
			v = rs_load<IQ>(in, (unsigned long long) g);
			const long long k = st_lo + i;
			if (IQ && mag_out != NULL && k >= own_lo && k < own_hi) mag_out[g] = v;
		}
		s_x[i] = v;
	}
	// the history the next run reads: the last H magnitudes of everything seen so far
	if (blockIdx.x == 0 && threadIdx.x < SINC_H) {
		const long long g = (long long) run_samples - SINC_H + threadIdx.x;
		hist_out[threadIdx.x] = g < 0 ? hist_in[SINC_H + g] : rs_load<IQ>(in, (unsigned long long) g);
	}
	__syncthreads();
	float *gout = out + B.out_start;
	for (unsigned p = p_lo + threadIdx.x; p < p_hi; p += SINC_THREADS) {
		int j;
		const long long k0 = sinc_pos(p, phase, rinv, &j);
		const float *x = s_x + (int) (k0 - (SINC_T / 2 - 1) - st_lo);
		const float4 *h = taps + j * (SINC_T / 4);
		float hv[SINC_T];
		#pragma unroll
		for (int q = 0; q < SINC_T / 4; q++) { const float4 v = __ldg(h + q); hv[4 * q] = v.x; hv[4 * q + 1] = v.y; hv[4 * q + 2] = v.z; hv[4 * q + 3] = v.w; }
		float y = __fmul_rn(x[0], hv[0]);
		#pragma unroll
		for (int t = 1; t < SINC_T; t++) y = __fadd_rn(y, __fmul_rn(x[t], hv[t]));
		gout[p] = y;
	}
}

__global__ void __launch_bounds__(256) demod_kernel(const float2 *__restrict__ iq, float *__restrict__ out, unsigned long long pairs) {
	const unsigned long long stride = (unsigned long long) gridDim.x * blockDim.x;
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += stride) {
		const float2 v = ldg_stream_f2(iq + i);
		out[i] = mag_exact(v.x, v.y);
	}
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
struct tsdrgpu_resampler {
	tsdrgpu_ctx_t *ctx;
	double offset;             // host: data-independent phase state (dsp_resample_t.offset)
	DeviceBuf<double> d_contrib;                        // device: dsp_resample_t.contrib
	// descriptor staging: pinned ring + device copies (bytes), one slot per in-flight run
	static constexpr int SLOTS = 4;
	PinnedBuf<unsigned char> h_desc[SLOTS]; DeviceBuf<unsigned char> d_desc[SLOTS]; cudaEvent_t ev[SLOTS]; int next;
	DeviceBuf<double> d_bank; DeviceBuf<int> d_has_a;
	float *d_mag_next;         // one-shot: the next IQ run also writes the magnitudes here (tsdrgpu_resampler_set_mag_out)
	// windowed-sinc mode (tsdrgpu_resampler_set_kernel)
	int kernel;                // TSDRGPU_RS_BOX / TSDRGPU_RS_SINC
	DeviceBuf<float> d_hist[2]; int hist_cur; int hist_zero;      // last H magnitudes: runs read d_hist[hist_cur], write the other; zero before the next run
	DeviceBuf<float> d_taps; double taps_fc;            // tap table on the device, built for min(1, r) == taps_fc (0: none yet)
};

extern "C" {

int tsdrgpu_am_demod(tsdrgpu_ctx_t *ctx, void *stream, const float *d_iq, uint64_t pairs, float *d_out) {
	BIND(ctx);
	if (pairs == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_iq != NULL && d_out != NULL);
	const unsigned long long want = (pairs + 255) / 256;
	const unsigned grid = (unsigned) (want < (unsigned long long) ctx->sm_count * 16 ? want : (unsigned long long) ctx->sm_count * 16);
	KL(ctx, "demod_kernel", (cudaStream_t) stream, demod_kernel<<<grid, 256, 0, (cudaStream_t) stream>>>(reinterpret_cast<const float2 *>(d_iq), d_out, pairs));
	return TSDRGPU_OK;
}

// a resampler whole or half built: its events (null ones are skipped), then the object; its buffers go with it
static void release(tsdrgpu_resampler *r) {
	for (cudaEvent_t e : r->ev) if (e) cudaEventDestroy(e);
	delete r;
}

static int create_handles(tsdrgpu_resampler *r) {
	tsdrgpu_ctx_t *ctx = r->ctx;
	CU_TRY(ctx, r->d_contrib.assign(1));
	CU_TRY(ctx, cudaMemset(r->d_contrib.ptr, 0, sizeof(double)));
	for (cudaEvent_t &e : r->ev) CU_TRY(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
	for (DeviceBuf<float> &h : r->d_hist) {
		CU_TRY(ctx, h.assign(SINC_H));
		CU_TRY(ctx, cudaMemset(h.ptr, 0, sizeof(float) * SINC_H));
	}
	CU_TRY(ctx, r->d_taps.assign(SINC_T * SINC_L));
	return TSDRGPU_OK;
}

uint32_t tsdrgpu_sinc_tile_pixels(double r) {
	return r >= TSDRGPU_SINC_MIN_RATIO ? sinc_pixels_per_tile(r) : 0;
}

int tsdrgpu_resampler_create(tsdrgpu_ctx_t *ctx, tsdrgpu_resampler_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_resampler *r = new tsdrgpu_resampler();      // value-initialised: every field not set here starts at zero
	r->ctx = ctx;
	const int rc = create_handles(r);
	if (rc) { release(r); return rc; }
	*out = r;
	return TSDRGPU_OK;
}

void tsdrgpu_resampler_destroy(tsdrgpu_resampler_t *r) {
	if (!r) return;
	cudaSetDevice(r->ctx->device);
	cudaDeviceSynchronize();
	release(r);
}

int tsdrgpu_resampler_set_kernel(tsdrgpu_resampler_t *r, int kernel) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	ARG_TRY(r->ctx, kernel == TSDRGPU_RS_BOX || kernel == TSDRGPU_RS_SINC);
	if (kernel == TSDRGPU_RS_SINC && r->kernel != TSDRGPU_RS_SINC) r->hist_zero = 1;      // a fresh start, not a box run's leftovers
	r->kernel = kernel;
	return TSDRGPU_OK;
}

int tsdrgpu_resampler_set_mag_out(tsdrgpu_resampler_t *r, float *d_mag) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	r->d_mag_next = d_mag;
	return TSDRGPU_OK;
}

int tsdrgpu_resampler_reset(tsdrgpu_resampler_t *r, void *stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	BIND(r->ctx);
	r->offset = 0.0;
	CU_TRY(r->ctx, cudaMemsetAsync(r->d_contrib.ptr, 0, sizeof(double), (cudaStream_t) stream));
	CU_TRY(r->ctx, cudaMemsetAsync(r->d_hist[r->hist_cur].ptr, 0, sizeof(float) * SINC_H, (cudaStream_t) stream));
	r->hist_zero = 0;
	return TSDRGPU_OK;
}

int tsdrgpu_resampler_get_state(tsdrgpu_resampler_t *r, void *stream, double *contrib, double *offset) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	BIND(r->ctx);
	if (contrib) {
		CU_TRY(r->ctx, cudaMemcpyAsync(contrib, r->d_contrib.ptr, sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t) stream));
		CU_TRY(r->ctx, cudaStreamSynchronize((cudaStream_t) stream));
	}
	if (offset) *offset = r->offset;
	return TSDRGPU_OK;
}

int tsdrgpu_resampler_set_state(tsdrgpu_resampler_t *r, void *stream, double contrib, double offset) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	BIND(r->ctx);
	r->offset = offset;
	CU_TRY(r->ctx, cudaMemcpyAsync(r->d_contrib.ptr, &contrib, sizeof(double), cudaMemcpyHostToDevice, (cudaStream_t) stream));
	CU_TRY(r->ctx, cudaStreamSynchronize((cudaStream_t) stream));
	return TSDRGPU_OK;
}

uint64_t tsdrgpu_resampler_plan(tsdrgpu_resampler_t *r, const uint32_t *block_sizes, uint32_t uniform_block,
                                uint32_t nblocks, double upsample_by, double downsample_by) {
	if (!r) return 0;
	double off = r->offset;
	const uint64_t n = tsdrgpu_plan_resample(&off, block_sizes, uniform_block, nblocks, upsample_by, downsample_by, NULL);
	return n == UINT64_MAX ? 0 : n;
}

int tsdrgpu_resampler_run(tsdrgpu_resampler_t *r, void *stream_, const float *d_in, int in_is_iq,
                          const uint32_t *block_sizes, uint32_t uniform_block, uint32_t nblocks,
                          double upsample_by, double downsample_by, int nearest,
                          float *d_out, uint64_t out_capacity, uint64_t *h_n_out) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, r != NULL);
	tsdrgpu_ctx_t *ctx = r->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	if (h_n_out) *h_n_out = 0;
	if (nblocks == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in != NULL && d_out != NULL);
	ARG_TRY(ctx, upsample_by > 0 && downsample_by > 0);
	ARG_TRY(ctx, nblocks <= 65535u);

	const double ratio = upsample_by / downsample_by;
	const bool sinc = r->kernel == TSDRGPU_RS_SINC && !nearest;
	if (sinc && !(ratio >= TSDRGPU_SINC_MIN_RATIO))
		return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "the sinc resampler needs upsample_by/downsample_by >= 1/16", cudaSuccess, __FILE__, __LINE__);
	// A refused call changes nothing: not the state, not the descriptor ring, not the armed magnitude output.
	if (r->d_mag_next && (!in_is_iq || nearest)) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "magnitude output needs IQ input and the box resampler", cudaSuccess, __FILE__, __LINE__);
	const unsigned sinc_pt = sinc ? sinc_pixels_per_tile(ratio) : 0;
	// descriptor slot: [RsBlock x nblocks][{block, first sample (box) / first pixel (sinc)} x tiles]
	size_t max_tiles = 0;
	for (uint32_t b = 0; b < nblocks; b++) {
		const size_t size = block_sizes ? block_sizes[b] : uniform_block;
		max_tiles += sinc ? (size_t) ((double) size * ratio + 2.0) / sinc_pt + 2 : (size + RS_TILE - 1) / RS_TILE + 1;
	}
	const size_t need = sizeof(tsdrgpu_rs_block_t) * nblocks + sizeof(uint2) * (max_tiles + 1);
	const int slot = r->next;
	CU_TRY(ctx, cudaEventSynchronize(r->ev[slot]));
	if (r->h_desc[slot].cap < need || r->d_desc[slot].cap < need) {
		const int rc = r->h_desc[slot].assign(ctx, need * 2);
		if (rc) return rc;
		CU_TRY(ctx, r->d_desc[slot].assign(need * 2));
	}
	tsdrgpu_rs_block_t *hb = (tsdrgpu_rs_block_t *) r->h_desc[slot].ptr;
	uint2 *hp = (uint2 *) (hb + nblocks);

	double off = r->offset;
	const uint64_t total = tsdrgpu_plan_resample(&off, block_sizes, uniform_block, nblocks, upsample_by, downsample_by, hb);
	if (total == UINT64_MAX)
		return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "a block would produce no pixel (the reference asserts here, extbuffer.c:48)", cudaSuccess, __FILE__, __LINE__);
	if (total > out_capacity)
		return tsdrgpu_fail(ctx, TSDRGPU_ECAPACITY, "resampler output buffer too small", cudaSuccess, __FILE__, __LINE__);
	r->next = (slot + 1) % tsdrgpu_resampler::SLOTS;
	unsigned tiles = 0, max_out = 0;
	// rs_main4 (four samples per thread) stages every tile's pixels in shared memory: ratios up to 3; beyond that, and on
	// request (TSDRGPU_RS_V1=1, the cross-check of the tests), the one-sample-per-thread kernel (every geometry the reference
	// can produce has r = (int)(2x)/x <= 2, TSDRLibrary.c:540-550).  rs_main4's tiles are windows
	// aligned on the input address: a block's first tile is cut short by the samples its start lies past a 16-byte boundary.
	const bool v1 = getenv("TSDRGPU_RS_V1") != NULL || !(ratio <= 2.0) || nearest;      // r <= 2: a sample emits at most 3 pixels
	for (uint32_t b = 0; b < nblocks; b++) {
		if (sinc) {                                       // rs_sinc tiles the block's pixels
			for (unsigned p0 = 0; p0 < hb[b].n_out; p0 += sinc_pt) hp[tiles++] = make_uint2(b, p0);
			continue;
		}
		unsigned lead = 0;
		if (!v1) {
			const unsigned long long addr = reinterpret_cast<unsigned long long>(d_in) + (in_is_iq ? 8ull : 4ull) * hb[b].in_start;
			lead = in_is_iq ? (unsigned) ((addr >> 3) & 1ull) : (unsigned) ((addr >> 2) & 3ull);
		}
		for (unsigned s0 = 0; s0 < hb[b].size; s0 = (s0 == 0) ? RS_TILE - lead : s0 + RS_TILE) hp[tiles++] = make_uint2(b, s0);
		if (hb[b].n_out > max_out) max_out = hb[b].n_out;
	}
	CU_TRY(ctx, cudaMemcpyAsync(r->d_desc[slot].ptr, r->h_desc[slot].ptr, need, cudaMemcpyHostToDevice, stream));
	CU_TRY(ctx, cudaEventRecord(r->ev[slot], stream));
	const RsBlock *db = (const RsBlock *) r->d_desc[slot].ptr;
	const uint2 *dp = (const uint2 *) (db + nblocks);

	float *mag = r->d_mag_next; r->d_mag_next = NULL;
	if (sinc) {
		const double fc = ratio < 1.0 ? ratio : 1.0;
		if (r->taps_fc != fc) {                           // pageable source: the copy is staged before the call returns
			static thread_local float h_taps[SINC_T * SINC_L];
			tsdrgpu_sinc_taps(ratio, h_taps, NULL, NULL);
			CU_TRY(ctx, cudaMemcpyAsync(r->d_taps.ptr, h_taps, sizeof h_taps, cudaMemcpyHostToDevice, stream));
			r->taps_fc = fc;
		}
		if (r->hist_zero) { CU_TRY(ctx, cudaMemsetAsync(r->d_hist[r->hist_cur].ptr, 0, sizeof(float) * SINC_H, stream)); r->hist_zero = 0; }
		uint64_t run_samples = 0;
		for (uint32_t b = 0; b < nblocks; b++) run_samples += hb[b].size;
		const float *hin = r->d_hist[r->hist_cur].ptr;
		float *hout = r->d_hist[r->hist_cur ^ 1].ptr;
		const float4 *taps = reinterpret_cast<const float4 *>(r->d_taps.ptr);
		if (in_is_iq) KL(ctx, "rs_sinc", stream, rs_sinc<true><<<tiles, SINC_THREADS, 0, stream>>>(d_in, d_out, db, dp, sinc_pt, taps, hin, hout, run_samples, mag));
		else KL(ctx, "rs_sinc", stream, rs_sinc<false><<<tiles, SINC_THREADS, 0, stream>>>(d_in, d_out, db, dp, sinc_pt, taps, hin, hout, run_samples, (float *) NULL));
		r->hist_cur ^= 1;
	} else if (nearest) {
		dim3 grid((max_out + 1023) / 1024, nblocks);
		if (in_is_iq) KL(ctx, "rs_nearest", stream, rs_nearest<true><<<grid, 256, 0, stream>>>(d_in, d_out, db));
		else KL(ctx, "rs_nearest", stream, rs_nearest<false><<<grid, 256, 0, stream>>>(d_in, d_out, db));
	} else {
		if (r->d_bank.cap < (size_t) nblocks + 1 || r->d_has_a.cap < (size_t) nblocks + 1) {
			if (r->d_bank.ptr || r->d_has_a.ptr) CU_TRY(ctx, cudaStreamSynchronize(stream));
			CU_TRY(ctx, r->d_bank.assign((size_t) nblocks * 2 + 2));
			CU_TRY(ctx, r->d_has_a.assign((size_t) nblocks * 2 + 2));
		}
		if (v1) {
			if (in_is_iq) KL(ctx, "rs_main", stream, rs_main<true><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, mag));
			else KL(ctx, "rs_main", stream, rs_main<false><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, (float *) NULL));
		} else {
			// Resident CTAs per SM the register allocation aims at.  Whole device-resident bench step (bench.py, BENCH_QUICK, cfg2) on
			// an H100 SXM at a 400 W power limit, two alternating runs each: 18.8 GS/s at 3 CTAs (80 registers), 19.0-19.2 at 4 (64),
			// 18.6 at 5 (48, with spills), 17.8 at 6 (40).  TSDRGPU_RS_MINB overrides for experiments.
			static const int minb = getenv("TSDRGPU_RS_MINB") ? atoi(getenv("TSDRGPU_RS_MINB")) : 4;
			if (in_is_iq) {
				if (minb >= 6) KL(ctx, "rs_main", stream, rs_main4<true, 6><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, mag));
				else if (minb == 5) KL(ctx, "rs_main", stream, rs_main4<true, 5><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, mag));
				else if (minb == 4) KL(ctx, "rs_main", stream, rs_main4<true, 4><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, mag));
				else KL(ctx, "rs_main", stream, rs_main4<true, 3><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, mag));
			} else KL(ctx, "rs_main", stream, rs_main4<false, 5><<<tiles, RS_THREADS, 0, stream>>>(d_in, d_out, db, dp, (float *) NULL));
		}
		if (in_is_iq) KL(ctx, "rs_fixup", stream, rs_fixup<true><<<1, 256, 0, stream>>>(d_in, d_out, db, nblocks, r->d_bank.ptr, r->d_has_a.ptr, r->d_contrib.ptr));
		else KL(ctx, "rs_fixup", stream, rs_fixup<false><<<1, 256, 0, stream>>>(d_in, d_out, db, nblocks, r->d_bank.ptr, r->d_has_a.ptr, r->d_contrib.ptr));
	}
	r->offset = off;
	if (h_n_out) *h_n_out = total;
	return TSDRGPU_OK;
}

}  // extern "C"
