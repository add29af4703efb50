// fft.cu -- a18..a20, a22: FFT, "autocorrelation", cross-correlation, the frame-rate detector's running means and
// the superbandwidth stitch.
//
// Replaces fft_perform / fft_autocorrelation / fft_crosscorrelation (fft.c:49-176), accummulate and
// frameratedetector_runontodata (frameratedetector.c:34-126), complex_to_abs_diff / superb_bestfit /
// superb_ondataready (superbandwidth.c:67-152).
//
// FFT design (no tensor cores: nothing here is a dense contraction; the bound is HBM bandwidth and issue slots):
//   N = 2^m is factored into 1, 2 or 3 line lengths (Cooley-Tukey index maps; 2 passes up to 2^20, 3 above).  One CTA
//   transforms a BUNDLE of C adjacent lines (4096 points, 512 threads): radix-8 Stockham stages written as their radix-2
//   layers, the first fed from global memory, the last storing to global memory through the epilogue (inter-pass twiddle,
//   scale, |.|), the ones between through XOR-swizzled shared memory.  Bundling makes every global access a run of >= C
//   consecutive complex values even on the strided passes, so each pass is one coalesced read + one coalesced write of
//   the array: 16 N bytes per pass.  The transposing last pass writes to the other buffer, so no copy pass exists.
//   Real->complex widening and |X|/N are fused into the first / last pass of the autocorrelation's forward transform (the
//   N-point path; on the default half-size path the forward finish is fused into the inverse's first pass, see RSPLIT).
// Numerics: float32 data.  Layer twiddles come from host-built double-precision tables that carry the REFERENCE'S stage
// angles (its half-angle recurrence, fft.c:161, is off by up to 5e-5 relative at the largest stages: see
// tsdrgpu_fft_reference_eps), inter-pass twiddles from sincospif of an exactly reduced argument times a host-built step
// table.  The reference keeps float32 storage between its radix-2 stages too (fft.c:150-155); results agree to <= 1e-6 of
// the spectrum's peak up to 2^22 (not bit-exact).
#include "common.cuh"
#include <math.h>
#include <stdlib.h>
#include <vector>

namespace {

constexpr int FFT_MAX_LOG2L = 11;            // longest line transformed inside one CTA: 2048
constexpr int FFT_TABLE = 1 << FFT_MAX_LOG2L;
constexpr int FFT_MAX_ELEMS = 4096;          // complex elements per CTA bundle: 512 threads x 8 (35 KB of shared memory, >= 3 CTAs/SM)

struct FftPass {
	int log2L, C, log2C, c_fast_in, c_fast_out;
	long long in_bs, out_bs;                            // batch strides (blockIdx.y), in elements of the in / out type
	unsigned G_lo;
	long long in_hi, in_lo, in_cs, in_js;
	long long out_hi, out_lo, out_cs, out_ks;
	unsigned long long tw_M; long long tw_lo, tw_cs;    // column index = g_lo*tw_lo + c*tw_cs ; tw_M == 0: none
	float scale;
	int in_real, out_abs;                               // in_real: 1 = real input widened to (x, 0); 2 = complex input given as PAIRS OF FLOATS that are only 4-byte aligned (in_bs then counts floats); 3 = see rs_* below
	const float2 *tw_step;                              // host-built W_M^(col (L/8) j), [col][8]; NULL: compute every twiddle
	int exact0;                                         // the first three layers of this pass have eps = 0: plain DFT-8
	int conj_in, conj_out;                              // inverse transforms: conjugate on load (first pass) / on store (last pass)
	int dbg;                                            // timing experiments only (TSDRGPU_FFT_DBG): 1 = no global loads, 2 = no global stores; results are garbage
	// in_real = 3 (first pass, fft_pass_kernel<..., RSPLIT = true>): `in` is the unscaled half-size forward spectrum Z of a real
	// sequence (rs_half points per transform) and the input is formed on load as z'[n] = (R[2n], R[2n+1]), R = |X| * rs_scale
	// from the real split with the last-stage table rs_last (see real_split_rn)
	const float2 *rs_last; unsigned rs_half; float rs_scale;
	const float *win;                                   // first pass, in_real = 2: each pair times win[n] (__fmul_rn), n = its index in the transform
	// fft_acc_kernel (a last pass): |X|^2 of the transforms blockIdx.y, blockIdx.y + gridDim.y, ... < nseg (in_bs apart) summed in
	// double into row blockIdx.y of acc (acc_bs doubles apart, bins in natural order); rows < acc_keep add to what they hold
	double *acc; long long acc_bs; unsigned nseg, acc_keep;
};

// The coherence (tsdrgpu_coherence_*), beside an FftPass whose layout (and so the Welch kernels' code) it leaves alone.  Its first
// pass reads the complex window w+ from FftPass.win as float2.  fft_acc2_kernel: transforms 2j and 2j + 1 are U+ and U- of segment
// j, which starts at pair (seg0 + j) hop of the report; row blockIdx.y of FftPass.acc holds four planes of `plane` doubles:
// Re C, Im C, P+, P-.
struct CohPass { double alpha, fs; unsigned long long seg0, hop; long long plane; };

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// ---- in-register small DFTs (natural order in, natural order out) -------------------------------------------------
// Explicitly rounded single precision (__f*_rn never contracts), so the rounding sequence of every butterfly is fixed by the
// source and not by the compiler: a complex multiply by a twiddle kept in both forms (c, s) and (-s, c) is one rounded
// product and one fused multiply-add per component.
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
// x * w with w given as (c, s) and its quarter turn (-s, c):  (x.x c - x.y s, x.x s + x.y c)
__device__ __forceinline__ float2 cmulp(float2 x, float4 w) {
	return make_float2(__fmaf_rn(x.x, w.x, __fmul_rn(x.y, w.z)), __fmaf_rn(x.x, w.y, __fmul_rn(x.y, w.w)));
}
__device__ __forceinline__ float4 twform(float2 w) { return make_float4(w.x, w.y, -w.y, w.x); }
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s)); }
// multiply by -i (forward) or +i (inverse)
__device__ __forceinline__ float2 rot90(float2 a, bool inverse) { return inverse ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x); }

__device__ __forceinline__ void dft2(float2 &a, float2 &b) { const float2 t = a; a = cadd(t, b); b = csub(t, b); }
__device__ __forceinline__ void dft4(float2 &v0, float2 &v1, float2 &v2, float2 &v3, bool inverse) {
	const float2 a0 = cadd(v0, v2), a1 = csub(v0, v2), a2 = cadd(v1, v3), a3 = rot90(csub(v1, v3), inverse);
	v0 = cadd(a0, a2); v1 = cadd(a1, a3); v2 = csub(a0, a2); v3 = csub(a1, a3);
}
__device__ __forceinline__ void dft8(float2 (&v)[8], bool inverse) {
	// even / odd halves as two 4-point DFTs, then the W8^k twiddles
	dft4(v[0], v[2], v[4], v[6], inverse);
	dft4(v[1], v[3], v[5], v[7], inverse);
	const float h = 0.70710678118654752440f;
	const float2 o0 = v[1];
	const float2 t1 = v[3];            // * W8^1 = (1 -+ i)/sqrt2
	const float2 o1 = inverse ? make_float2(h * (t1.x - t1.y), h * (t1.x + t1.y)) : make_float2(h * (t1.x + t1.y), h * (t1.y - t1.x));
	const float2 o2 = rot90(v[5], inverse);
	const float2 t3 = v[7];            // * W8^3 = (-1 -+ i)/sqrt2
	const float2 o3 = inverse ? make_float2(-h * (t3.x + t3.y), h * (t3.x - t3.y)) : make_float2(h * (t3.y - t3.x), -h * (t3.x + t3.y));
	const float2 e0 = v[0], e1 = v[2], e2 = v[4], e3 = v[6];
	v[0] = cadd(e0, o0); v[1] = cadd(e1, o1); v[2] = cadd(e2, o2); v[3] = cadd(e3, o3);
	v[4] = csub(e0, o0); v[5] = csub(e1, o1); v[6] = csub(e2, o2); v[7] = csub(e3, o3);
}

// transforms of 2 or 4 points (whole transforms only: passes of longer ones have lines of >= 64): one thread each, exact
// twiddles (the reference's first two stages have no angle error), the same load / store conventions as the pass kernel
template <int LOG2L>
__global__ void __launch_bounds__(32) fft_tiny_kernel(const float2 *in, float2 *out, FftPass P) {
	if (threadIdx.x != 0) return;
	constexpr int L = 1 << LOG2L;
	const long long ib = (long long) blockIdx.y * P.in_bs, ob = (long long) blockIdx.y * P.out_bs;
	float2 v[L];
	#pragma unroll
	for (int j = 0; j < L; j++) {
		if (P.in_real == 2) { const float *pr = reinterpret_cast<const float *>(in) + ib + 2 * j; v[j] = make_float2(pr[0], pr[1]); }
		else v[j] = P.in_real ? make_float2(reinterpret_cast<const float *>(in)[ib + j], 0.0f) : in[ib + j];
		if (P.conj_in) v[j].y = -v[j].y;
	}
	if (L == 2) dft2(v[0], v[1]); else dft4(v[0], v[1], v[2], v[3], false);
	#pragma unroll
	for (int k = 0; k < L; k++) {
		float2 r = make_float2(v[k].x * P.scale, v[k].y * (P.conj_out ? -P.scale : P.scale));
		if (P.out_abs) r = make_float2(__fsqrt_rn(__fadd_rn(__fmul_rn(r.x, r.x), __fmul_rn(r.y, r.y))), 0.0f);
		out[ob + k] = r;
	}
}

// ---- the pass kernel for lines of length L >= 8 --------------------------------------------------------------------
// Each thread owns 8 points per stage.  The first radix-8 butterfly is fed straight from global memory and the last
// butterfly (radix 8, 4 or 2) stores straight to global memory (through the inter-pass twiddle / scale / |.| epilogue),
// so a 1024-point line makes 3 trips through shared memory instead of 5 + load + store, with one barrier each
// (ping-pong buffers).  Thread -> (line, butterfly) maps are chosen per pass so that the global accesses of a warp are
// runs of consecutive complex values: line-fastest on strided passes, butterfly-fastest on contiguous lines.
//
// Butterflies are written as their radix-2 layers (a radix-8 Stockham step with block size p = layers with blocks p, 2p,
// 4p): layer t multiplies the upper input by T_t[K], K = k + p q0 (+ 2p q1).  The layer twiddles come from a per-pass
// table built on the host in double precision, T_s[K] = exp(-i pi K / 2^s (1 + eps_s)), stored layer after layer
// (layer s at offset 2^s - 1), so the seven twiddles of a radix-8 butterfly are table[k + j p - 1], j = 1..7.
// eps_s is the relative angle error of the reference's stage l_base + s (tsdrgpu_fft_reference_eps; fft.c:161 derives
// its twiddles by a half-angle recurrence that loses accuracy for small angles) or 0 for the mathematically exact DFT:
// same kernel, same operation count (12 complex multiplications + 24 additions per 8 points) either way.
//
// Shared memory is unpadded; a line's point q lives at slot (q ^ swz(q)) ^ xc(line): swz permutes inside aligned groups
// of 16 so that the stride-8 stores of stage 0 and the stride-p stores of the p = 8 stage hit 16 distinct bank pairs per
// half-warp, and xc (a per-line constant < 16) does the same for the line-fastest thread maps of strided passes.
// swz is linear over GF(2): swz(a ^ b) = swz(a) ^ swz(b).  Every index the kernel forms is a sum of two terms with
// disjoint bits (i + m L/8, 8 i + m, j + m p), so slot = swz(thread part) ^ swz(m part) and the m part is a compile-time
// constant: one XOR and one add per access on 32-bit shared addresses.
__host__ __device__ constexpr int swz(int q) { return q ^ ((q >> 4) & 7) ^ (((q >> 6) & 1) << 3); }
__device__ __forceinline__ unsigned smem_addr(const void *p) { return (unsigned) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void sts2(unsigned addr, float2 v) { asm volatile("st.shared.v2.f32 [%0], {%1, %2};" :: "r"(addr), "f"(v.x), "f"(v.y) : "memory"); }
__device__ __forceinline__ float2 lds2(unsigned addr) { float2 v; asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory"); return v; }

// Butterflies exist in the FORWARD direction only.  An inverse transform is the conjugate of the forward transform of the
// conjugated input -- conj(x conj(w)) = conj(x) w, and IEEE arithmetic is sign-symmetric -- so an inverse pass conjugates what it
// loads from global memory in its first pass and what it stores in its last one (FftPass.conj_in / conj_out) and is otherwise
// the same code.  Layer twiddles are loaded as (c, s) and turned into cmulp's (c, s, -s, c) in registers: 16-byte table entries
// were measured slower (twice the L1 wavefronts on a kernel whose first stall reason is the memory-instruction queue).
__device__ __forceinline__ void bf8(float2 *v, const float2 *__restrict__ tw /* = table + k - 1 */, int p) {
	float2 a[4][2], b[2][2][2];
	const float4 TA = twform(__ldg(tw + p)), TB0 = twform(__ldg(tw + 2 * p)), TB1 = twform(__ldg(tw + 3 * p));
	const float4 TC00 = twform(__ldg(tw + 4 * p)), TC10 = twform(__ldg(tw + 5 * p)), TC01 = twform(__ldg(tw + 6 * p)), TC11 = twform(__ldg(tw + 7 * p));
	#pragma unroll
	for (int r = 0; r < 4; r++) { const float2 hi = cmulp(v[r + 4], TA); a[r][0] = cadd(v[r], hi); a[r][1] = csub(v[r], hi); }
	#pragma unroll
	for (int q0 = 0; q0 < 2; q0++) {
		const float4 TB = q0 ? TB1 : TB0;
		#pragma unroll
		for (int m0 = 0; m0 < 2; m0++) { const float2 hi = cmulp(a[m0 + 2][q0], TB); b[m0][q0][0] = cadd(a[m0][q0], hi); b[m0][q0][1] = csub(a[m0][q0], hi); }
	}
	#pragma unroll
	for (int q0 = 0; q0 < 2; q0++) {
		#pragma unroll
		for (int q1 = 0; q1 < 2; q1++) {
			const float4 TC = q1 ? (q0 ? TC11 : TC01) : (q0 ? TC10 : TC00);
			const float2 hi = cmulp(b[1][q0][q1], TC);
			v[q0 + 2 * q1] = cadd(b[0][q0][q1], hi); v[q0 + 2 * q1 + 4] = csub(b[0][q0][q1], hi);
		}
	}
}
__device__ __forceinline__ void bf4(float2 *v, const float2 *__restrict__ tw, int p) {
	float2 a[2][2];
	const float4 TA = twform(__ldg(tw + p)), TB0 = twform(__ldg(tw + 2 * p)), TB1 = twform(__ldg(tw + 3 * p));
	#pragma unroll
	for (int r = 0; r < 2; r++) { const float2 hi = cmulp(v[r + 2], TA); a[r][0] = cadd(v[r], hi); a[r][1] = csub(v[r], hi); }
	#pragma unroll
	for (int q0 = 0; q0 < 2; q0++) {
		const float2 hi = cmulp(a[1][q0], q0 ? TB1 : TB0);
		v[q0] = cadd(a[0][q0], hi); v[q0 + 2] = csub(a[0][q0], hi);
	}
}
__device__ __forceinline__ void bf2(float2 *v, const float2 *__restrict__ tw, int p) {
	const float2 hi = cmulp(v[1], twform(__ldg(tw + p)));
	const float2 lo = v[0];
	v[0] = cadd(lo, hi); v[1] = csub(lo, hi);
}

// ---- TMA: a pass whose lines are contiguous in memory (the second pass of a two-pass plan, the third of a three-pass plan,
// a single-pass transform) gets its whole bundle with bulk copies (cp.async.bulk.shared::cluster.global, SASS UBLKCP) issued
// by one thread and counted in bytes on an mbarrier: C copies of one line each -- or ONE copy of C L complex values when the
// lines of the bundle are adjacent, as in two-pass plans -- land linearly in the half of the ping-pong buffer the first
// butterfly does not write; the threads wait on the barrier and read their eight inputs from shared memory (consecutive
// lanes read consecutive values: conflict-free without a swizzle).  The eight dependent global loads per thread, their address
// arithmetic and their scoreboard stalls are gone from the instruction stream.
__device__ __forceinline__ void fft_mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void fft_mbar_expect_tx(unsigned bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void fft_mbar_wait(unsigned bar, unsigned parity) {
	asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
	             :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void fft_bulk_g2s(unsigned dst_smem, const void *src, unsigned bytes, unsigned bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
	             :: "r"(dst_smem), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// ---- real-input transforms at half size (see autocorrelation_batch_half) -------------------------------------------------
// z[j] = x[2j] + i x[2j+1] has been transformed (N/2 points, unscaled) into Z.  With E, O the transforms of the even and odd
// samples, E = (Z[k] + conj Z[-k]) / 2, O = (Z[k] - conj Z[-k]) / 2i, and the reference's LAST radix-2 stage (its perturbed
// angle: last[k] = exp(-i pi k / (N/2) (1 + eps_{m-1})), host-built) gives X[k] = E + w O, X[k + N/2] = E - w O with w = last[k]
// (forward) or conj(last[k]) (inverse).  Explicitly rounded, so that the result does not depend on where it is inlined: the
// halving is one product on the O side and fused into the final sums on the E side, t = w O is one product and one fused
// multiply-add per component.
__device__ __forceinline__ void real_split_rn(float2 zk, float2 zm, float2 w, float2 &x0, float2 &x1) {
	const float sx = __fadd_rn(zk.x, zm.x), dy = __fsub_rn(zk.y, zm.y);
	const float ox = __fmul_rn(__fadd_rn(zk.y, zm.y), 0.5f), oy = __fmul_rn(__fsub_rn(zk.x, zm.x), -0.5f);
	const float tx = __fmaf_rn(w.x, ox, -__fmul_rn(w.y, oy)), ty = __fmaf_rn(w.x, oy, __fmul_rn(w.y, ox));
	x0 = make_float2(__fmaf_rn(sx, 0.5f, tx), __fmaf_rn(dy, 0.5f, ty));
	x1 = make_float2(__fmaf_rn(sx, 0.5f, -tx), __fmaf_rn(dy, 0.5f, -ty));
}

// The pass over transform `by` of the batch (fft_pass_kernel: by = blockIdx.y).  RSPLIT: the first pass of the inverse half-size
// transform (FftPass.in_real = 3) -- the forward finish happens on load.  WIN = 1: pairs of floats (in_real = 2) are multiplied by
// P.win on load; WIN = 2: by the complex window w+ in P.win (by even) or its conjugate (by odd), transform `by` reading segment
// by / 2.  ACC = 1 (fft_acc_kernel): nothing is stored; |X|^2 of every output is added to the thread's sums acc[8], which the CTA's
// last transform (`last`) adds to its row of P.acc.  ACC = 2 (fft_acc2_kernel): by even keeps U+ in stash[8]; by odd adds
// U+ conj(U-) e^{i theta} (ph = (cos, sin) theta), |U+|^2 and |U-|^2 to acc[32] (four per output), written like ACC = 1 into the
// `plane`-apart planes of the row.
template <int LOG2L, bool TMA, bool RSPLIT, int ACC, int WIN>
__device__ __forceinline__ void fft_pass_body(const float2 *in, float2 *out, const FftPass &P, const float2 *__restrict__ stw, unsigned by,
                                              double *acc, bool last, float2 *stash = nullptr, double2 ph = double2(), long long plane = 0) {
	extern __shared__ __align__(128) float2 s[];
	constexpr int L = 1 << LOG2L, NST8 = LOG2L / 3, RL = LOG2L % 3;
	constexpr int RLAST = (RL == 0) ? 8 : ((RL == 1) ? 2 : 4);
	constexpr int NSTAGES = NST8 + (RL ? 1 : 0);
	constexpr int NMID = NSTAGES - 2;                    // radix-8 stages between the first and the last one
	constexpr int L8 = L / 8, LOG2L8 = LOG2L - 3;
	const int C = P.C, log2C = P.log2C;
	const int tid = threadIdx.x;
	const unsigned g = blockIdx.x, g_hi = g / P.G_lo, g_lo = g - g_hi * P.G_lo;
	const long long in_base = (long long) g_hi * P.in_hi + (long long) g_lo * P.in_lo + (P.in_real == 2 ? 0ll : (long long) by * P.in_bs);
	const long long out_base = (long long) g_hi * P.out_hi + (long long) g_lo * P.out_lo;
	float2 *gout = ACC ? nullptr : out + (out_base + (long long) by * P.out_bs);
	const bool active = tid < C * L8;                    // tiny bundles leave part of the last warp idle
	// per-line slot constants (see above): xa for the buffer stage 0 writes, xb for the buffer the last stage reads
	const int sha = (log2C >= 4) ? 0 : 3 - log2C, shb = (NSTAGES == 2 || log2C >= 4) ? sha : 4 - log2C;
	const unsigned sbase = smem_addr(s);
	float2 v[8];
	// Inter-pass twiddles W_M^(col k): a thread's eight outputs are k = i0 + (L/8) j, j = 0..7, of ONE column, so
	// W^(col k) = W^(col i0) * W^(col (L/8) j): one sincospif per thread for the first factor (exactly reduced argument),
	// the second from a host-built table of 8 values per column (double precision; P.tw_step[col * 8 + j]).
	const bool tw_fast = P.tw_step != NULL && P.c_fast_out && (int) blockDim.x == C * L8;

	// ---- stage 0: radix 8, p = 1, inputs x[i + m L/8] from global memory (or, TMA, from the bundle the bulk copies landed)
	{
		int c, i;
		if (P.c_fast_in) { c = tid & (C - 1); i = tid >> log2C; } else { i = tid & (L8 - 1); c = tid >> LOG2L8; }
		if (P.dbg & 1) {
			#pragma unroll
			for (int m = 0; m < 8; m++) v[m] = make_float2((float) tid, (float) m);
		} else if (TMA) {
			__shared__ __align__(8) unsigned long long bar_mem;
			const unsigned bar = smem_addr(&bar_mem);
			const unsigned landing = sbase + ((NSTAGES > 1) ? (unsigned) (C * L) * 8u : 0u);      // the half stage 0 does not write
			if (tid == 0) { fft_mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
			__syncthreads();
			if (tid == 0) {
				const unsigned line_bytes = (unsigned) L * 8u;
				fft_mbar_expect_tx(bar, (unsigned) C * line_bytes);
				const float2 *g0 = in + in_base;
				if ((int) P.in_cs == L) fft_bulk_g2s(landing, g0, (unsigned) C * line_bytes, bar);          // adjacent lines: one copy
				else for (int cc = 0; cc < C; cc++) fft_bulk_g2s(landing + (unsigned) cc * line_bytes, g0 + (long long) cc * P.in_cs, line_bytes, bar);
			}
			fft_mbar_wait(bar, 0);
			if (active) {
				const unsigned lr = landing + (unsigned) (c * L + i) * 8u;
				#pragma unroll
				for (int m = 0; m < 8; m++) v[m] = lds2(lr + (unsigned) (m * L8) * 8u);
				if (P.conj_in) {
					#pragma unroll
					for (int m = 0; m < 8; m++) v[m].y = -v[m].y;
				}
			}
		} else if (active) {
			const int off = c * (int) P.in_cs + i * (int) P.in_js, step = L8 * (int) P.in_js;
			if (RSPLIT) {
				// v[m] = z'[n] and v[m + 4] = z'[n + M/2] (n = n0 + m step, 4 step = M/2 in every plan) come from the same two splits,
				// at K = 2n and 2n + 1: R[K] = |x0| and R[K + M] = |x1|.  Z[2n], Z[2n+1] and last[2n], last[2n+1] are one 16-byte
				// load each; the mirrors Z[M - 2n], Z[M - 2n - 1] of adjacent columns are a contiguous run read backwards.
				const unsigned M = P.rs_half;
				const float2 *z = in + (long long) by * P.in_bs;
				const unsigned n0 = (unsigned) (in_base - (long long) by * P.in_bs) + (unsigned) off;
				#pragma unroll
				for (int m = 0; m < 4; m++) {
					const unsigned K = 2u * (n0 + (unsigned) (m * step));
					const float4 zk = __ldg(reinterpret_cast<const float4 *>(z + K)), w = __ldg(reinterpret_cast<const float4 *>(P.rs_last + K));
					const float2 zm0 = __ldg(z + ((M - K) & (M - 1))), zm1 = __ldg(z + (M - K - 1));
					float2 a0, a1, b0, b1;
					real_split_rn(make_float2(zk.x, zk.y), zm0, make_float2(w.x, w.y), a0, a1);
					real_split_rn(make_float2(zk.z, zk.w), zm1, make_float2(w.z, w.w), b0, b1);
					const float s = P.rs_scale;
					v[m] = make_float2(mag_exact(__fmul_rn(a0.x, s), __fmul_rn(a0.y, s)), mag_exact(__fmul_rn(b0.x, s), __fmul_rn(b0.y, s)));
					v[m + 4] = make_float2(mag_exact(__fmul_rn(a1.x, s), __fmul_rn(a1.y, s)), mag_exact(__fmul_rn(b1.x, s), __fmul_rn(b1.y, s)));
				}
				if (P.conj_in) {
					#pragma unroll
					for (int m = 0; m < 8; m++) v[m].y = -v[m].y;
				}
			} else if (P.in_real == 2) {                             // pairs of floats, 4-byte aligned (a capture that starts on an odd sample)
				const float *gr = reinterpret_cast<const float *>(in) + (long long) (WIN == 2 ? by >> 1 : by) * P.in_bs + 2 * (in_base + off);
				#pragma unroll
				for (int m = 0; m < 8; m++) v[m] = make_float2(__ldg(gr + 2 * m * step), __ldg(gr + 2 * m * step + 1));
				if (WIN == 1) {                                      // the window of the spectrum (tsdrgpu_spectrum_*)
					const float *wr = P.win + in_base + off;
					#pragma unroll
					for (int m = 0; m < 8; m++) { const float wv = __ldg(wr + m * step); v[m] = make_float2(__fmul_rn(v[m].x, wv), __fmul_rn(v[m].y, wv)); }
				} else if (WIN == 2) {                               // the coherence's w+ or w- = conj(w+) (tsdrgpu_coherence_*)
					const float2 *wr = reinterpret_cast<const float2 *>(P.win) + in_base + off;
					const bool minus = by & 1;
					#pragma unroll
					for (int m = 0; m < 8; m++) {
						const float2 wc = __ldg(wr + m * step);
						const float wy = minus ? -wc.y : wc.y;
						v[m] = make_float2(__fsub_rn(__fmul_rn(v[m].x, wc.x), __fmul_rn(v[m].y, wy)), __fadd_rn(__fmul_rn(v[m].x, wy), __fmul_rn(v[m].y, wc.x)));
					}
				}
				if (P.conj_in) {
					#pragma unroll
					for (int m = 0; m < 8; m++) v[m].y = -v[m].y;
				}
			} else if (P.in_real) {
				const float *gr = reinterpret_cast<const float *>(in) + in_base + off;
				#pragma unroll
				for (int m = 0; m < 8; m++) v[m] = make_float2(__ldg(gr + m * step), 0.0f);
			} else {
				const float2 *gc = in + in_base + off;
				#pragma unroll
				for (int m = 0; m < 8; m++) v[m] = __ldg(gc + m * step);
				if (P.conj_in) {
					#pragma unroll
					for (int m = 0; m < 8; m++) v[m].y = -v[m].y;
				}
			}
		}
		if (active) {
			if (P.exact0) { float2 (&u)[8] = *reinterpret_cast<float2 (*)[8]>(&v[0]); dft8(u, false); }     // layers with eps = 0: plain DFT-8
			else bf8(v, stw - 1, 1);
		}
		if (NSTAGES > 1) {
			if (active) {
				const unsigned la = sbase + (unsigned) (c * L) * 8u, rb = (unsigned) (swz(8 * i) ^ ((c << sha) & 15)) * 8u;
				#pragma unroll
				for (int m = 0; m < 8; m++) sts2(la + (rb ^ (unsigned) (m * 8)), v[m]);
			}
			__syncthreads();
		}
	}
	unsigned src = sbase, dst = sbase + (unsigned) (C * L) * 8u;
	// ---- middle radix-8 stages (shared -> shared, ping-pong)
	#pragma unroll
	for (int st = 0; st < (NMID > 0 ? NMID : 0); st++) {
		const int p = 8 << (3 * st);
		const int i = tid & (L8 - 1), c = tid >> LOG2L8;
		if (active) {
			const int xa = (c << sha) & 15, xw = (st == NMID - 1) ? ((c << shb) & 15) : xa;
			const unsigned lr = src + (unsigned) (c * L) * 8u, rb = (unsigned) (swz(i) ^ xa) * 8u;
			#pragma unroll
			for (int m = 0; m < 8; m++) v[m] = lds2(lr + (rb ^ (unsigned) (swz(m * L8) * 8)));
			const int k = i & (p - 1);
			bf8(v, stw + k - 1, p);
			const int j = ((i - k) << 3) + k;
			const unsigned lw = dst + (unsigned) (c * L) * 8u, wb = (unsigned) (swz(j) ^ xw) * 8u;
			#pragma unroll
			for (int m = 0; m < 8; m++) sts2(lw + (wb ^ (unsigned) (swz(m * p) * 8)), v[m]);
		}
		__syncthreads();
		const unsigned t = src; src = dst; dst = t;
	}
	// ---- last stage: radix RLAST with p = L / RLAST, results X[i + m p] go to global memory
	constexpr int NB = 8 / RLAST, PL = L / RLAST, LOG2PL = LOG2L - (RLAST == 8 ? 3 : (RLAST == 4 ? 2 : 1));
	const int T = blockDim.x;
	const unsigned twmask = (unsigned) (P.tw_M - 1);
	const float inv_M = P.tw_M ? 1.0f / (float) P.tw_M : 0.0f;       // a power of two: exact
	float4 tw_base4 = make_float4(1.0f, 0.0f, -0.0f, 1.0f);
	#pragma unroll
	for (int it = 0; it < NB; it++) {
		const int widx = tid + it * T;
		if (widx >= C * PL) continue;
		int c, i;
		if (P.c_fast_out) { c = widx & (C - 1); i = widx >> log2C; } else { i = widx & (PL - 1); c = widx >> LOG2PL; }
		float2 *w = v + it * RLAST;
		if (NSTAGES > 1) {
			const unsigned lr = src + (unsigned) (c * L) * 8u, rb = (unsigned) (swz(i) ^ ((c << shb) & 15)) * 8u;
			#pragma unroll
			for (int m = 0; m < RLAST; m++) w[m] = lds2(lr + (rb ^ (unsigned) (swz(m * PL) * 8)));
			if (RLAST == 8) bf8(w, stw + i - 1, PL);
			else if (RLAST == 4) bf4(w, stw + i - 1, PL);
			else bf2(w, stw + i - 1, PL);
		}
		float2 *o = gout + c * (int) P.out_cs;
		const int ks = (int) P.out_ks;
		if (P.tw_M) {
			// inter-pass twiddle W_M^(col k): the argument is reduced exactly in integers, sincospif sees an exact float
			const unsigned col = (unsigned) ((int) g_lo * (int) P.tw_lo + c * (int) P.tw_cs);
			if (tw_fast) {
				if (it == 0) {
					const unsigned e = (col * (unsigned) i) & twmask;            // i == i0 in the first round
					float sn, cs;
					sincospif(-2.0f * ((float) e * inv_M), &sn, &cs);
					tw_base4 = make_float4(cs, sn, -sn, cs);
				}
				#pragma unroll
				for (int m = 0; m < RLAST; m++) {
					const float2 st = __ldg(P.tw_step + col * 8u + (unsigned) (it + NB * m));
					w[m] = cmulp(w[m], twform(cmulp(st, tw_base4)));
				}
			} else if (P.tw_M <= (1ull << 24)) {
				#pragma unroll
				for (int m = 0; m < RLAST; m++) {
					const int k = i + m * PL;
					const unsigned e = (col * (unsigned) k) & twmask;
					float sn, cs;
					sincospif(-2.0f * ((float) e * inv_M), &sn, &cs);
					w[m] = cmulp(w[m], make_float4(cs, sn, -sn, cs));
				}
			} else {
				#pragma unroll
				for (int m = 0; m < RLAST; m++) {
					const int k = i + m * PL;
					const unsigned long long e = ((unsigned long long) col * (unsigned long long) k) & (P.tw_M - 1);
					double dsn, dcs;
					sincospi(-2.0 * ((double) e / (double) P.tw_M), &dsn, &dcs);
					w[m] = cmulp(w[m], make_float4((float) dcs, (float) dsn, -(float) dsn, (float) dcs));
				}
			}
		}
		if constexpr (ACC == 2) {                            // the coherence's sums in double, over the CTA's segments in their order
			if (!(by & 1)) {
				#pragma unroll
				for (int m = 0; m < RLAST; m++) stash[it * RLAST + m] = w[m];
				continue;
			}
			double *row = P.acc + (long long) blockIdx.y * P.acc_bs + out_base + c * (int) P.out_cs;
			#pragma unroll
			for (int m = 0; m < RLAST; m++) {
				const double ax = stash[it * RLAST + m].x, ay = stash[it * RLAST + m].y, bx = w[m].x, bym = w[m].y;
				const double cr = __fma_rn(ax, bx, __dmul_rn(ay, bym)), ci = __fma_rn(ay, bx, -__dmul_rn(ax, bym));   // U+ conj(U-): exact
				double *a = acc + 4 * (it * RLAST + m);
				a[0] = __fma_rn(cr, ph.x, __fma_rn(-ci, ph.y, a[0]));
				a[1] = __fma_rn(cr, ph.y, __fma_rn(ci, ph.x, a[1]));
				a[2] = __fma_rn(ax, ax, __fma_rn(ay, ay, a[2]));
				a[3] = __fma_rn(bx, bx, __fma_rn(bym, bym, a[3]));
				if (last) {
					double *d = row + (i + m * PL) * ks;
					#pragma unroll
					for (int q = 0; q < 4; q++) d[q * plane] = (blockIdx.y < P.acc_keep) ? __dadd_rn(d[q * plane], a[q]) : a[q];
				}
			}
			continue;
		} else if constexpr (ACC == 1) {                     // |X|^2 in double, summed over the CTA's transforms in their order
			double *row = P.acc + (long long) blockIdx.y * P.acc_bs + out_base + c * (int) P.out_cs;
			#pragma unroll
			for (int m = 0; m < RLAST; m++) {
				const double x = w[m].x, y = w[m].y;
				double &a = acc[it * RLAST + m];
				a = __fma_rn(x, x, __fma_rn(y, y, a));
				if (last) { double *d = row + (i + m * PL) * ks; *d = (blockIdx.y < P.acc_keep) ? __dadd_rn(*d, a) : a; }
			}
			continue;
		}
		if (P.out_abs) {
			#pragma unroll
			for (int m = 0; m < RLAST; m++) {
				const float x = w[m].x * P.scale, y = w[m].y * P.scale;
				const float mag = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
				o[(i + m * PL) * ks] = make_float2(mag, 0.0f);
			}
		} else {
			const float sy = P.conj_out ? -P.scale : P.scale;      // inverse transforms: the conjugate on the way out (see bf8)
			#pragma unroll
			for (int m = 0; m < RLAST; m++) if (!(P.dbg & 2) || w[m].x == 1.2345e30f) o[(i + m * PL) * ks] = make_float2(w[m].x * P.scale, w[m].y * sy);
		}
	}
}

template <int LOG2L, bool TMA = false, bool RSPLIT = false, int WIN = 0>
__global__ void __launch_bounds__(512, 3) fft_pass_kernel(const float2 *in, float2 *out, FftPass P, const float2 *__restrict__ stw) {
	fft_pass_body<LOG2L, TMA, RSPLIT, 0, WIN>(in, out, P, stw, blockIdx.y, nullptr, false);
}

// The spectrum's last pass: CTA row blockIdx.y transforms blockIdx.y, blockIdx.y + gridDim.y, ... < P.nseg and adds the sum of their
// |X|^2 (per bin, in that order) to its row of P.acc, so writes are rows x bins whatever the number of transforms.  Every row
// has at least one transform (the caller launches at most nseg rows).  64 registers: room for the eight double sums.
template <int LOG2L>
__global__ void __launch_bounds__(512, 2) fft_acc_kernel(const float2 *in, FftPass P, const float2 *__restrict__ stw) {
	double acc[8];
	#pragma unroll
	for (int j = 0; j < 8; j++) acc[j] = 0.0;
	for (unsigned seg = blockIdx.y; seg < P.nseg; seg += gridDim.y) {
		if (seg != blockIdx.y) __syncthreads();          // the last stage of the previous transform has read the shared buffers
		fft_pass_body<LOG2L, false, false, 1, 1>(in, nullptr, P, stw, seg, acc, seg + gridDim.y >= P.nseg);
	}
}

// The coherence's last pass: CTA row blockIdx.y takes segments j = blockIdx.y, blockIdx.y + gridDim.y, ... < P.nseg / 2, transforms
// 2j (U+, kept in registers) and 2j + 1 (U-) of each, and adds the per-bin sums of U+ conj(U-) e^{-2 pi i alpha s_j / fs}, |U+|^2 and
// |U-|^2 (in that order of segments) to its row of P.acc.  alpha s_j / fs is formed in double from the integer s_j and reduced mod 1
// before the sincospi.  One CTA per SM: the 32 double sums take 64 registers.
template <int LOG2L>
__global__ void __launch_bounds__(512, 1) fft_acc2_kernel(const float2 *in, FftPass P, const float2 *__restrict__ stw, CohPass Q) {
	double acc[32];
	float2 stash[8];
	#pragma unroll
	for (int j = 0; j < 32; j++) acc[j] = 0.0;
	const unsigned nseg = P.nseg / 2;
	for (unsigned seg = blockIdx.y; seg < nseg; seg += gridDim.y) {
		double t = __ddiv_rn(__dmul_rn(Q.alpha, (double) ((Q.seg0 + seg) * Q.hop)), Q.fs);
		t = __dsub_rn(t, floor(t));
		double2 ph;
		sincospi(__dmul_rn(-2.0, t), &ph.y, &ph.x);
		const bool last = seg + gridDim.y >= nseg;
		if (seg != blockIdx.y) __syncthreads();
		fft_pass_body<LOG2L, false, false, 2, 2>(in, nullptr, P, stw, 2 * seg, acc, last, stash, ph, Q.plane);
		__syncthreads();
		fft_pass_body<LOG2L, false, false, 2, 2>(in, nullptr, P, stw, 2 * seg + 1, acc, last, stash, ph, Q.plane);
	}
}

// ---- small elementwise helpers -----------------------------------------------------------------------------
// answer[2i] = real[i], answer[2i+1] = 0 for i in [from, to)          (fft.c:14-22)
__global__ void k_real_to_complex(float2 *answer, const float *real, unsigned long long from, unsigned long long to) {
	for (unsigned long long i = from + (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < to; i += (unsigned long long) gridDim.x * blockDim.x)
		answer[i] = make_float2(real[i], 0.0f);
}
// answer[i] = (|answer[i]|, 0)                                          (fft.c:34-45)
__global__ void k_abs(float2 *answer, unsigned long long from, unsigned long long to) {
	for (unsigned long long i = from + (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < to; i += (unsigned long long) gridDim.x * blockDim.x) {
		const float2 v = answer[i];
		answer[i] = make_float2(mag_exact(v.x, v.y), 0.0f);
	}
}
// ---- the inverse half-size transform's finish (real_split_rn): every one of the N complex outputs of an autocorrelation, for
// callers that want all lags (the frame-rate detector folds the lags it reads into its running means, k_accumulate_half)
__global__ void __launch_bounds__(256) k_real_inv_finish(const float2 *__restrict__ Z, long long z_bs, const float2 *__restrict__ last,
                                                         unsigned half, float2 *__restrict__ Y, long long y_bs) {
	const float2 *z = Z + (long long) blockIdx.y * z_bs;
	float2 *y = Y + (long long) blockIdx.y * y_bs;
	for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < half; k += gridDim.x * blockDim.x) {
		const float2 w = __ldg(last + k);
		float2 x0, x1;
		real_split_rn(z[k], z[(half - k) & (half - 1)], make_float2(w.x, -w.y), x0, x1);
		y[k] = x0; y[k + half] = x1;
	}
}

// a = (aI*bI + aQ*bQ, aI*bQ - aQ*bI)                                   (fft.c:80-89)
__global__ void k_conj_mul(float2 *a, const float2 *b, unsigned long long n) {
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long) gridDim.x * blockDim.x) {
		const float2 x = a[i], y = b[i];
		a[i] = make_float2(__fadd_rn(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y)), __fsub_rn(__fmul_rn(x.x, y.y), __fmul_rn(x.y, y.x)));
	}
}
// running mean of lag magnitudes in double                             (frameratedetector.c:34-62)
__global__ void k_accumulate(double *out, unsigned long long calls, const float2 *in, int startid, int length) {
	const double now_n = (double) calls, before_n = (double) (calls - 1);
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x) {
		const float2 v = in[(size_t) startid + i];
		const double re = (double) v.x, im = (double) v.y;
		const double mag = __dsqrt_rn(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));
		out[i] = (calls == 0) ? mag : __ddiv_rn(__dadd_rn(__dmul_rn(out[i], before_n), mag), now_n);
	}
}
// the same running mean for `batch` consecutive captures in order (one launch instead of `batch`)
__global__ void k_accumulate_batch(double *out, unsigned long long first_calls, const float2 *in, long long in_stride, unsigned batch,
                                   int startid, int length) {
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x) {
		double acc = out[i];
		for (unsigned b = 0; b < batch; b++) {
			const unsigned long long calls = first_calls + b;
			const float2 v = in[(size_t) b * in_stride + startid + i];
			const double re = (double) v.x, im = (double) v.y;
			const double mag = __dsqrt_rn(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));
			acc = (calls == 0) ? mag : __ddiv_rn(__dadd_rn(__dmul_rn(acc, (double) (calls - 1)), mag), (double) calls);
		}
		out[i] = acc;
	}
}
// the same, straight from the half-size inverse's output Z' (captures z_bs apart, `half` points each): the inverse finish is
// folded in, lag k < half is x0 of the split at k, lag k >= half (a window beyond N/2) x1 of the split at k - half, both with
// the conjugate last-stage twiddle, exactly as k_real_inv_finish forms them
__global__ void k_accumulate_half(double *out, unsigned long long first_calls, const float2 *__restrict__ Z, long long z_bs, unsigned batch,
                                  const float2 *__restrict__ last, unsigned half, int startid, int length) {
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < length; i += gridDim.x * blockDim.x) {
		const unsigned k = (unsigned) (startid + i), hi = k >= half, kk = hi ? k - half : k, km = (half - kk) & (half - 1);
		const float2 w = __ldg(last + kk), wc = make_float2(w.x, -w.y);
		double acc = out[i];
		for (unsigned b = 0; b < batch; b++) {
			const unsigned long long calls = first_calls + b;
			const float2 *z = Z + (long long) b * z_bs;
			float2 x0, x1;
			real_split_rn(z[kk], z[km], wc, x0, x1);
			const double re = (double) (hi ? x1.x : x0.x), im = (double) (hi ? x1.y : x0.y);
			const double mag = __dsqrt_rn(__dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im)));
			acc = (calls == 0) ? mag : __ddiv_rn(__dadd_rn(__dmul_rn(acc, (double) (calls - 1)), mag), (double) calls);
		}
		out[i] = acc;
	}
}
// SURVEY 8f-3 on the device: the index of the first strict maximum of each running-mean plot, the pick the GUI makes on the
// host (PlotVisualizer.java:203-236: start from element 0, move on a strict '>').  One CTA per plot; NaN never wins, a NaN in
// element 0 keeps index 0 (nothing compares greater than it), equal values keep the smallest index.
__global__ void __launch_bounds__(1024) k_plot_peaks(const double *p0, int n0, const double *p1, int n1, int *peaks) {
	__shared__ double s_v[32]; __shared__ int s_i[32];
	const double *v = blockIdx.x ? p1 : p0;
	const int n = blockIdx.x ? n1 : n0;
	double best = -INFINITY; int bi = 0x7fffffff;
	for (int i0 = threadIdx.x; i0 < n; i0 += 8 * (int) blockDim.x) {      // eight loads in flight per thread, folded in index order
		double x[8];
		#pragma unroll
		for (int u = 0; u < 8; u++) { const int i = i0 + u * (int) blockDim.x; x[u] = (i < n) ? v[i] : -INFINITY; }
		#pragma unroll
		for (int u = 0; u < 8; u++) { const int i = i0 + u * (int) blockDim.x; if (i < n && (x[u] > best || (x[u] == best && i < bi))) { best = x[u]; bi = i; } }
	}
	for (int o = 16; o > 0; o >>= 1) {
		const double ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
		if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
	}
	if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = best; s_i[threadIdx.x >> 5] = bi; }
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int w = 1; w < (int) (blockDim.x >> 5); w++) if (s_v[w] > best || (s_v[w] == best && s_i[w] < bi)) { best = s_v[w]; bi = s_i[w]; }
		const double first = n > 0 ? v[0] : 0.0;
		peaks[blockIdx.x] = (n <= 0 || first != first || bi == 0x7fffffff) ? 0 : bi;
	}
}
// first difference of magnitudes, out of place                          (superbandwidth.c:67-81)
__global__ void k_abs_diff(const float2 *src, float2 *dst, unsigned long long pairs) {
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < pairs; i += (unsigned long long) gridDim.x * blockDim.x) {
		const float2 v = src[i];
		const float cur = mag_exact(v.x, v.y);
		float prev;
		if (i == 0) prev = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));    // seed without the square root
		else { const float2 u = src[i - 1]; prev = mag_exact(u.x, u.y); }
		dst[i] = make_float2(__fsub_rn(cur, prev), 0.0f);
	}
}
// argmax of |x| over [0, n): first maximum wins                         (superbandwidth.c:100-116)
// Two steps over the whole chip instead of one CTA: every CTA reduces a contiguous chunk to (value, index), the last step
// (one CTA) reduces the partials.  "First maximum" = smallest index among equal values, so the result does not depend on
// how the range is cut; the reference starts from element 0 and only moves on a strict '>' (NaN never wins).
__device__ __forceinline__ void argmax_merge(float &best, unsigned &bi, float ov, unsigned oi) {
	if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
}
__device__ __forceinline__ void argmax_block_reduce(float &best, unsigned &bi, float *s_v, unsigned *s_i) {
	for (int o = 16; o > 0; o >>= 1) argmax_merge(best, bi, __shfl_xor_sync(0xffffffffu, best, o), __shfl_xor_sync(0xffffffffu, bi, o));
	if ((threadIdx.x & 31) == 0) { s_v[threadIdx.x >> 5] = best; s_i[threadIdx.x >> 5] = bi; }
	__syncthreads();
	if (threadIdx.x == 0) for (int w = 1; w < (int) (blockDim.x >> 5); w++) argmax_merge(best, bi, s_v[w], s_i[w]);
}
__global__ void __launch_bounds__(256) k_argmax_partial(const float2 *__restrict__ x, unsigned n, float *__restrict__ pv, unsigned *__restrict__ pi) {
	__shared__ float s_v[8]; __shared__ unsigned s_i[8];
	const unsigned per = (n + gridDim.x - 1) / gridDim.x, lo = blockIdx.x * per, hi = min(n, lo + per);
	float best = -1.0f; unsigned bi = 0xffffffffu;
	for (unsigned i = lo + threadIdx.x; i < hi; i += blockDim.x) {
		const float2 v = __ldg(x + i);
		const float m = mag_exact(v.x, v.y);
		if (m > best) { best = m; bi = i; }              // a thread walks upwards: the first of equal values stays
	}
	argmax_block_reduce(best, bi, s_v, s_i);
	if (threadIdx.x == 0) { pv[blockIdx.x] = best; pi[blockIdx.x] = bi; }
}
__global__ void __launch_bounds__(256) k_argmax_final(const float *__restrict__ pv, const unsigned *__restrict__ pi, unsigned parts, int *result) {
	__shared__ float s_v[8]; __shared__ unsigned s_i[8];
	float best = -1.0f; unsigned bi = 0xffffffffu;
	for (unsigned i = threadIdx.x; i < parts; i += blockDim.x) argmax_merge(best, bi, pv[i], pi[i]);
	argmax_block_reduce(best, bi, s_v, s_i);
	if (threadIdx.x == 0) *result = (bi == 0xffffffffu) ? 0 : (int) bi;
}
// rotate left by *shift complex elements, the shift read from device memory (the lag the kernels before produced)
__global__ void k_rotate_dev(const float2 *src, float2 *dst, unsigned long long n, const int *shift_) {
	const unsigned long long shift = (unsigned long long) *shift_;
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long) gridDim.x * blockDim.x) {
		unsigned long long s = i + shift; if (s >= n) s -= n;
		dst[i] = src[s];
	}
}
// multi-GPU stitch with the alignment folded into the spectrum: rotating hop q left by lag_q samples multiplies its
// spectrum by e^{+2 pi i m lag_q / N}, so ranks exchange RAW spectra and apply the ramp after the gather:
// U_s[m] = e^{+2 pi i m s/(H N)} * sum_q e^{+2 pi i (q s / H + m lag_q / N)} X_q[m]
struct LagSet { int lag[16]; };
__global__ void k_residue_mix_lag(const float2 *gathered, long long block_stride, int H, unsigned n, int s, LagSet lags, float2 *dst) {
	for (unsigned m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x) {
		float accr = 0.0f, acci = 0.0f;
		for (int q = 0; q < H; q++) {
			// phase = 2 pi (q s / H + m lag / N): both terms reduced exactly in integers before the division
			const unsigned long long e = ((unsigned long long) m * (unsigned long long) lags.lag[q]) & (unsigned long long) (n - 1);
			const double frac = (double) e / (double) n + (double) ((q * s) % H) / (double) H;
			float sn, cs;
			sincospif((float) (2.0 * (frac - floor(frac))), &sn, &cs);
			const float2 v = gathered[(size_t) q * block_stride + m];
			accr += cs * v.x - sn * v.y; acci += cs * v.y + sn * v.x;
		}
		double dsn, dcs;
		sincospi(2.0 * ((double) m * (double) s) / ((double) H * (double) n), &dsn, &dcs);
		const float sn = (float) dsn, cs = (float) dcs;
		dst[m] = make_float2(accr * cs - acci * sn, accr * sn + acci * cs);
	}
}

inline unsigned grid1d(unsigned long long n, int sm_count) {
	const unsigned long long want = (n + 255) / 256, cap = (unsigned long long) sm_count * 8;
	return (unsigned) (want < cap ? (want ? want : 1) : cap);
}

// the pass kernels' dynamic shared-memory limit, raised once per context (ctx->mu held): before any of them is launched or has
// its occupancy queried
int pass_attrs(tsdrgpu_ctx_t *ctx) {
	if (ctx->fft_attrs_set) return TSDRGPU_OK;
	const int max_smem = (int) (2 * sizeof(float2) * FFT_MAX_ELEMS);     // ping-pong
#define SET_ATTR(l) CU_TRY(ctx, cudaFuncSetAttribute(fft_pass_kernel<l, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_pass_kernel<l, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_pass_kernel<l, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_pass_kernel<l, false, false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_pass_kernel<l, false, false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_acc_kernel<l>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem)); \
	CU_TRY(ctx, cudaFuncSetAttribute(fft_acc2_kernel<l>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem))
	SET_ATTR(3); SET_ATTR(4); SET_ATTR(5); SET_ATTR(6); SET_ATTR(7); SET_ATTR(8); SET_ATTR(9); SET_ATTR(10); SET_ATTR(11);
#undef SET_ATTR
	ctx->fft_attrs_set = true;
	return TSDRGPU_OK;
}

// The context's twiddle table `key` (tsdrgpu_ctx::fft_tables), n entries computed on the host by fill(h) on first use.  The
// first table also raises the pass kernels' shared-memory limit: every pass launch looks its stage table up first.
enum { TAB_STAGE, TAB_STEP, TAB_LAST };
template <class Fill> int fft_table(tsdrgpu_ctx_t *ctx, FftTableKey key, size_t n, Fill fill, const float2 **out) {
	std::lock_guard<std::mutex> lock(ctx->mu);
	for (auto &t : ctx->fft_tables)
		if (t.key.kind == key.kind && t.key.a == key.a && t.key.b == key.b && t.key.c == key.c && t.key.eps == key.eps) { *out = t.d.ptr; return TSDRGPU_OK; }
	if (const int rc = pass_attrs(ctx)) return rc;
	std::vector<float2> h(n);
	fill(h.data());
	ctx->fft_tables.emplace_back();
	FftTable &t = ctx->fft_tables.back();
	t.key = key;
	cudaError_t e = t.d.assign(n);
	if (e == cudaSuccess) e = cudaMemcpy(t.d.ptr, h.data(), sizeof(float2) * n, cudaMemcpyHostToDevice);
	if (e != cudaSuccess) { ctx->fft_tables.pop_back(); return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "FFT twiddle table", e, __FILE__, __LINE__); }
	*out = t.d.ptr;
	return TSDRGPU_OK;
}

// per-pass layer-twiddle tables (see fft_pass_kernel), built on the host in double precision
int stage_table(tsdrgpu_ctx_t *ctx, int log2L, int l_base, const double *eps_all, const float2 **out) {
	double eps[FFT_MAX_LOG2L + 1];
	int pert = 0;
	for (int sidx = 0; sidx < log2L; sidx++) {
		eps[sidx] = (!tsdrgpu_fft_true_dft() && eps_all && l_base + sidx < 40) ? eps_all[l_base + sidx] : 0.0;
		if (eps[sidx] != 0.0) pert = 1;
	}
	const int L = 1 << log2L;
	return fft_table(ctx, {TAB_STAGE, log2L, pert ? l_base : -1, pert, 0.0}, (size_t) L, [&](float2 *h) {
		for (int sidx = 0; sidx < log2L; sidx++) {
			const int blk = 1 << sidx;
			for (int K = 0; K < blk; K++) {
				const double ang = -3.14159265358979323846 * ((double) K / (double) blk) * (1.0 + eps[sidx]);
				h[(size_t) blk - 1 + K] = make_float2((float) cos(ang), (float) sin(ang));
			}
		}
		h[(size_t) L - 1] = make_float2(1.0f, 0.0f);
	}, out);
}

// W_M^(col * L8 * j) for every column of a pass and j = 0..7 (see fft_pass_kernel), built on the host
int step_table(tsdrgpu_ctx_t *ctx, unsigned long long M, unsigned ncols, unsigned L8, const float2 **out) {
	return fft_table(ctx, {TAB_STEP, (long long) M, ncols, L8, 0.0}, (size_t) ncols * 8, [&](float2 *h) {
		for (unsigned col = 0; col < ncols; col++)
			for (unsigned j = 0; j < 8; j++) {
				const unsigned long long e = ((unsigned long long) col * (unsigned long long) (L8 * j)) & (M - 1);
				const double ang = -2.0 * 3.14159265358979323846 * ((double) e / (double) M);
				h[(size_t) col * 8 + j] = make_float2((float) cos(ang), (float) sin(ang));
			}
	}, out);
}

int bundle_for(int log2L, unsigned long long lines, bool contiguous_lines = false) {
	const int L = 1 << log2L;
	int C = 4096 / L; if (C < 8) C = 8;
	while ((long long) C * L > FFT_MAX_ELEMS) C >>= 1;
	// experiment knob: smaller bundles (more, smaller CTAs per SM) on passes whose lines are contiguous in memory
	static const int small = getenv("TSDRGPU_FFT_SMALL_BUNDLE") ? atoi(getenv("TSDRGPU_FFT_SMALL_BUNDLE")) : 0;
	if (contiguous_lines && small >= 512) while ((long long) C * L > small && C > 1) C >>= 1;
	while ((unsigned long long) C > lines) C >>= 1;
	return C < 1 ? 1 : C;
}

// coh: the coherence's passes (P.win is w+; P.acc: fft_acc2_kernel)
int launch_pass(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, float2 *out, FftPass P, unsigned bundles, int inverse,
                unsigned batch, long long in_bs, long long out_bs, const double *eps_all = NULL, int l_base = 0, const CohPass *coh = NULL) {
	P.in_bs = in_bs; P.out_bs = out_bs;
	P.log2C = 0; while ((1 << P.log2C) < P.C) P.log2C++;
	const int L = 1 << P.log2L, total = P.C * L;
	int threads = (total / 8 + 31) / 32 * 32;            // one radix-8 butterfly (8 elements) per thread and stage
	if (threads < 32) threads = 32;
	if (threads > 512) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "FFT bundle too large", cudaSuccess, __FILE__, __LINE__);
	const int nstages = P.log2L / 3 + ((P.log2L % 3) ? 1 : 0);
	const dim3 grid(bundles, batch);
	if (P.log2L <= 2) {
		if (P.in_real == 3) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "real-split input needs lines of >= 8 points", cudaSuccess, __FILE__, __LINE__);
		if (P.log2L == 1) KL(ctx, "fft_pass_kernel", stream, fft_tiny_kernel<1><<<dim3(1, batch), 32, 0, stream>>>(in, out, P));
		else KL(ctx, "fft_pass_kernel", stream, fft_tiny_kernel<2><<<dim3(1, batch), 32, 0, stream>>>(in, out, P));
		return TSDRGPU_OK;
	}
	const float2 *stw;
	{ int rc = stage_table(ctx, P.log2L, l_base, eps_all, &stw); if (rc) return rc; }
	P.tw_step = NULL;
	if (P.tw_M && P.tw_M <= (1ull << 24) && P.c_fast_out && P.log2L >= 3 && P.tw_lo == P.C && P.tw_cs == 1) {
		// columns of this pass: col = g_lo * C + c, g_lo < G_lo
		const unsigned ncols = P.G_lo * (unsigned) P.C;
		if (ncols <= (1u << 20)) { int rc = step_table(ctx, P.tw_M, ncols, (unsigned) (L >> 3), &P.tw_step); if (rc) return rc; }
	}
	P.dbg = getenv("TSDRGPU_FFT_DBG") ? atoi(getenv("TSDRGPU_FFT_DBG")) : 0;
	P.exact0 = 1;
	for (int sidx = 0; sidx < 3 && sidx < P.log2L; sidx++) if (eps_all && l_base + sidx < 40 && fabs(eps_all[l_base + sidx]) > 1e-10) P.exact0 = 0;
	// bulk copies (TMA) feed the passes whose lines are contiguous and 16-byte aligned; TSDRGPU_FFT_NO_TMA=1 keeps the plain loads
	static const bool no_tma = getenv("TSDRGPU_FFT_NO_TMA") != NULL;
	const bool tma = !no_tma && !P.c_fast_in && !P.in_real && P.in_js == 1 && total * 8 == threads * 64 && !P.acc
	                 && ((reinterpret_cast<unsigned long long>(in) | ((unsigned long long) in_bs * 8ull)) & 15ull) == 0;
	const size_t smem = sizeof(float2) * (size_t) total * ((nstages >= 3 || (tma && nstages == 2)) ? 2 : 1);
	switch (P.log2L) {
#define CASE(l) case l: if (coh && P.acc) KL(ctx, "fft_acc2_kernel", stream, fft_acc2_kernel<l><<<grid, threads, smem, stream>>>(in, P, stw, *coh)); \
	                else if (coh) KL(ctx, "fft_pass_kernel", stream, fft_pass_kernel<l, false, false, 2><<<grid, threads, smem, stream>>>(in, out, P, stw)); \
	                else if (P.acc) KL(ctx, "fft_acc_kernel", stream, fft_acc_kernel<l><<<grid, threads, smem, stream>>>(in, P, stw)); \
	                else if (P.win) KL(ctx, "fft_pass_kernel", stream, fft_pass_kernel<l, false, false, 1><<<grid, threads, smem, stream>>>(in, out, P, stw)); \
	                else if (P.in_real == 3) KL(ctx, "fft_pass_kernel", stream, fft_pass_kernel<l, false, true><<<grid, threads, smem, stream>>>(in, out, P, stw)); \
	                else if (tma) KL(ctx, "fft_pass_kernel", stream, fft_pass_kernel<l, true><<<grid, threads, smem, stream>>>(in, out, P, stw)); \
	                else KL(ctx, "fft_pass_kernel", stream, fft_pass_kernel<l, false><<<grid, threads, smem, stream>>>(in, out, P, stw)); break
	CASE(3); CASE(4); CASE(5); CASE(6); CASE(7); CASE(8); CASE(9); CASE(10); CASE(11);
#undef CASE
	default: return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "unsupported FFT line length", cudaSuccess, __FILE__, __LINE__);
	}
	return TSDRGPU_OK;
}

struct FftOpts {
	const float *real_in; bool out_abs; float scale;
	unsigned batch;                 // independent transforms (grid.y)
	long long data_bs, scratch_bs, real_bs;   // distance between consecutive transforms in data (complex), scratch (complex), real_in (floats)
	const float2 *cplx_in; long long cplx_bs; // the first pass reads its (complex) input from here instead of `data` (which is then output only)
	const float *pair_in; long long pair_bs;  // the same, but the input is pairs of floats with 4-byte alignment only; pair_bs in FLOATS
	const float2 *split_in; long long split_bs;   // the first pass forms its input from this half-size spectrum (FftPass.in_real = 3); must not be `scratch`,
	const float2 *split_last; float split_scale;  // nor `data` on one-pass plans
	const float *win;                             // pair_in only: the first pass multiplies each pair by win[n] (FftPass.win)
	bool exact;                                   // the exact DFT's stage angles (eps = 0) instead of the reference's
	// one- and two-pass plans: the last pass sums |X|^2 of the `batch` transforms into acc_rows rows of acc instead of writing `data`
	// (fft_acc_kernel; acc_rows <= batch)
	double *acc; long long acc_bs; unsigned acc_rows, acc_keep;
	// the coherence: pair_in only, the complex window cwin (FftPass.win, batch = 2 x segments); with acc, the last pass is
	// fft_acc2_kernel
	const float2 *cwin; CohPass coh;
};

// N-point transform of `data` (complex, natural order) through `scratch`; result lands in `data`.
// With opts.real_in the input is read from a real array instead (data is output only).
int fft_run(tsdrgpu_ctx_t *ctx, cudaStream_t stream, float2 *data, float2 *scratch, unsigned log2N, int inverse, FftOpts o) {
	const unsigned long long N = 1ull << log2N;
	const float2 *src0 = o.split_in ? o.split_in : (o.real_in ? reinterpret_cast<const float2 *>(o.real_in) : (o.pair_in ? reinterpret_cast<const float2 *>(o.pair_in) : (o.cplx_in ? o.cplx_in : data)));
	const long long in0_bs = o.split_in ? o.split_bs : (o.real_in ? o.real_bs : (o.pair_in ? o.pair_bs : (o.cplx_in ? o.cplx_bs : o.data_bs)));
	const int in_mode = o.split_in ? 3 : (o.real_in ? 1 : (o.pair_in ? 2 : 0));
	double eps_ref[40];
	tsdrgpu_fft_reference_eps((int) log2N < 40 ? (int) log2N : 40, inverse, eps_ref);
	const double *eps_all = o.exact ? NULL : eps_ref;
	FftPass P; memset(&P, 0, sizeof P);
	P.rs_last = o.split_last; P.rs_half = (unsigned) N; P.rs_scale = o.split_scale;     // (read by the first pass only, with in_real = 3)
	P.win = o.cwin ? reinterpret_cast<const float *>(o.cwin) : o.win;
	const CohPass *coh = o.cwin ? &o.coh : NULL;
	// the last pass of an accumulating plan: grid.y = acc_rows CTA rows walk the `batch` transforms
	auto accumulate = [&](FftPass &Z) { Z.acc = o.acc; Z.acc_bs = o.acc_bs; Z.nseg = o.batch; Z.acc_keep = o.acc_keep; return o.acc ? o.acc_rows : o.batch; };
	if (log2N <= FFT_MAX_LOG2L) {                       // one pass, one CTA
		P.log2L = (int) log2N; P.C = 1; P.G_lo = 1; P.in_js = 1; P.out_ks = 1; P.scale = o.scale;
		P.in_real = in_mode; P.out_abs = o.out_abs;
		P.conj_in = P.conj_out = inverse ? 1 : 0;
		const unsigned rows = accumulate(P);
		return launch_pass(ctx, stream, src0, data, P, 1, inverse, rows, in0_bs, o.data_bs, eps_all, 0, coh);
	}
	int rc;
	// two passes up to 2^21 (1024 x 2048: the 2048-point lines go to the contiguous pass, one TMA bulk copy per 2-line bundle);
	// TSDRGPU_FFT_2PASS_MAX=20 restores three passes at 2^21 for comparison
	static const unsigned two_pass_max = getenv("TSDRGPU_FFT_2PASS_MAX") ? (unsigned) atoi(getenv("TSDRGPU_FFT_2PASS_MAX")) : 21u;
	if (log2N <= two_pass_max && log2N <= 22) {         // N = N1 * N2 ; n = N2*n1 + n2 ; k = k1 + N1*k2
		// odd log2 N: the SHORTER line goes to the strided pass (bundle of 8 columns = 64-byte runs instead of 4 = 32-byte runs on
		// both its loads and its stores); TSDRGPU_FFT_SPLIT=ceil restores the other split for comparison
		static const bool split_ceil = getenv("TSDRGPU_FFT_SPLIT") && !strcmp(getenv("TSDRGPU_FFT_SPLIT"), "ceil");
		const unsigned l1 = split_ceil ? (log2N + 1) / 2 : log2N / 2, l2 = log2N - l1;
		const unsigned long long N1 = 1ull << l1, N2 = 1ull << l2;
		P.log2L = (int) l1; P.C = bundle_for((int) l1, N2); P.c_fast_in = P.c_fast_out = 1;
		P.G_lo = (unsigned) (N2 / P.C);
		P.in_lo = P.C; P.in_cs = 1; P.in_js = (long long) N2;
		P.out_lo = P.C; P.out_cs = 1; P.out_ks = (long long) N2;
		P.tw_M = N; P.tw_lo = P.C; P.tw_cs = 1; P.scale = 1.0f; P.in_real = in_mode;
		P.conj_in = inverse ? 1 : 0;
		if ((rc = launch_pass(ctx, stream, src0, scratch, P, P.G_lo, inverse, o.batch, in0_bs, o.scratch_bs, eps_all, 0, coh))) return rc;
		FftPass Q; memset(&Q, 0, sizeof Q);
		Q.log2L = (int) l2; Q.C = bundle_for((int) l2, N1, true); Q.c_fast_in = 0; Q.c_fast_out = 1;
		Q.G_lo = (unsigned) (N1 / Q.C);
		Q.in_lo = (long long) Q.C * (long long) N2; Q.in_cs = (long long) N2; Q.in_js = 1;
		Q.out_lo = Q.C; Q.out_cs = 1; Q.out_ks = (long long) N1;
		Q.scale = o.scale; Q.out_abs = o.out_abs;
		Q.conj_out = inverse ? 1 : 0;
		const unsigned rows = accumulate(Q);
		return launch_pass(ctx, stream, scratch, data, Q, Q.G_lo, inverse, rows, o.scratch_bs, o.data_bs, eps_all, (int) l1, o.acc ? coh : NULL);
	}
	// N = N1*N2*N3 ; n = N2N3 n1 + N3 n2 + n3 ; k = k1 + N1 k2 + N1N2 k3
	const unsigned l1 = (log2N + 2) / 3, l2 = (log2N - l1 + 1) / 2, l3 = log2N - l1 - l2;
	if (l1 > (unsigned) FFT_MAX_LOG2L) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "FFT too long", cudaSuccess, __FILE__, __LINE__);
	if (o.acc) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "accumulating transforms need a one- or two-pass plan", cudaSuccess, __FILE__, __LINE__);
	const unsigned long long N1 = 1ull << l1, N2 = 1ull << l2, N3 = 1ull << l3, N23 = N2 * N3;
	{   // pass A: length N1 along stride N2N3, bundle over adjacent columns m
		P.log2L = (int) l1; P.C = bundle_for((int) l1, N23); P.c_fast_in = P.c_fast_out = 1;
		P.G_lo = (unsigned) (N23 / P.C);
		P.in_lo = P.C; P.in_cs = 1; P.in_js = (long long) N23;
		P.out_lo = P.C; P.out_cs = 1; P.out_ks = (long long) N23;
		P.tw_M = N; P.tw_lo = P.C; P.tw_cs = 1; P.scale = 1.0f; P.in_real = in_mode;
		P.conj_in = inverse ? 1 : 0;
		if ((rc = launch_pass(ctx, stream, src0, scratch, P, P.G_lo, inverse, o.batch, in0_bs, o.scratch_bs, eps_all, 0))) return rc;
	}
	{   // pass B: for every k1, length N2 along stride N3, bundle over adjacent n3 (in place in scratch)
		FftPass B; memset(&B, 0, sizeof B);
		B.log2L = (int) l2; B.C = bundle_for((int) l2, N3); B.c_fast_in = B.c_fast_out = 1;
		B.G_lo = (unsigned) (N3 / B.C);
		B.in_hi = (long long) N23; B.in_lo = B.C; B.in_cs = 1; B.in_js = (long long) N3;
		B.out_hi = (long long) N23; B.out_lo = B.C; B.out_cs = 1; B.out_ks = (long long) N3;
		B.tw_M = N23; B.tw_lo = B.C; B.tw_cs = 1; B.scale = 1.0f;
		if ((rc = launch_pass(ctx, stream, scratch, scratch, B, (unsigned) (N1 * B.G_lo), inverse, o.batch, o.scratch_bs, o.scratch_bs, eps_all, (int) l1))) return rc;
	}
	{   // pass C: contiguous lines of N3 at (k1,k2); bundle over adjacent k1; output k1 + N1 k2 + N1N2 k3
		FftPass Cc; memset(&Cc, 0, sizeof Cc);
		Cc.log2L = (int) l3; Cc.C = bundle_for((int) l3, N1, true); Cc.c_fast_in = 0; Cc.c_fast_out = 1;
		Cc.G_lo = (unsigned) (N1 / Cc.C);                // g = k2 * G_lo + (k1 / C)
		Cc.in_hi = (long long) N3; Cc.in_lo = (long long) Cc.C * (long long) N23; Cc.in_cs = (long long) N23; Cc.in_js = 1;
		Cc.out_hi = (long long) N1; Cc.out_lo = Cc.C; Cc.out_cs = 1; Cc.out_ks = (long long) (N1 * N2);
		Cc.scale = o.scale; Cc.out_abs = o.out_abs;
		Cc.conj_out = inverse ? 1 : 0;
		return launch_pass(ctx, stream, scratch, data, Cc, (unsigned) (N2 * Cc.G_lo), inverse, o.batch, o.scratch_bs, o.data_bs, eps_all, (int) (l1 + l2));
	}
}

unsigned ilog2(unsigned long long n) { unsigned m = 0; while ((n >>= 1) != 0) m++; return m; }

}  // namespace

// opt out of the reference's stage angles: every transform is the mathematically exact DFT (read once per process)
bool tsdrgpu_fft_true_dft() { static const bool on = getenv("TSDRGPU_FFT_TRUE_DFT") != NULL; return on; }

// internal entry used by other translation units
int tsdrgpu_fft_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, float2 *data, unsigned long long n_pow2, int inverse) {
	int rc;
	if (n_pow2 <= 1) return TSDRGPU_OK;
	void *scratch;
	if ((rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * n_pow2, &scratch))) return rc;
	FftOpts o; memset(&o, 0, sizeof o); o.batch = 1; o.scale = inverse ? 1.0f : 1.0f / (float) n_pow2;
	return fft_run(ctx, stream, data, (float2 *) scratch, ilog2(n_pow2), inverse, o);
}

// out of place: out = FFT(in), both n_pow2 complex, `in` untouched
int tsdrgpu_fft_oop_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, float2 *out, unsigned long long n_pow2, int inverse) {
	int rc;
	if (n_pow2 <= 1) { if (n_pow2 == 1) CU_TRY(ctx, cudaMemcpyAsync(out, in, sizeof(float2), cudaMemcpyDeviceToDevice, stream)); return TSDRGPU_OK; }
	void *scratch;
	if ((rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * n_pow2, &scratch))) return rc;
	FftOpts o; memset(&o, 0, sizeof o); o.batch = 1; o.scale = inverse ? 1.0f : 1.0f / (float) n_pow2;
	o.cplx_in = in; o.cplx_bs = 0;
	return fft_run(ctx, stream, out, (float2 *) scratch, ilog2(n_pow2), inverse, o);
}
// `batch` independent out-of-place transforms (transform b reads in + b*in_bs, writes out + b*out_bs) through a scratch area the
// CALLER owns (batch * n_pow2 complex; NULL: the context's scratch slot 0) -- for callers that run transforms on two streams at once
int tsdrgpu_fft_batch_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, long long in_bs, float2 *out, long long out_bs,
                               float2 *scratch, unsigned long long n_pow2, unsigned batch, int inverse) {
	int rc;
	ARG_TRY(ctx, n_pow2 >= 2 && batch >= 1);
	if (!scratch) {
		void *sc;
		if ((rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * n_pow2 * batch, &sc))) return rc;
		scratch = (float2 *) sc;
	}
	FftOpts o; memset(&o, 0, sizeof o); o.batch = batch; o.scale = inverse ? 1.0f : 1.0f / (float) n_pow2;
	o.cplx_in = in; o.cplx_bs = in_bs; o.data_bs = out_bs; o.scratch_bs = (long long) n_pow2;
	return fft_run(ctx, stream, out, scratch, ilog2(n_pow2), inverse, o);
}
// one transform with the exact DFT's stage angles, from `in` (complex, may be `out`) into `out` through `scratch` (n_pow2 complex of
// the caller's); forward transforms scale by 1/n_pow2, inverse ones are unscaled
int tsdrgpu_fft_exact_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, float2 *out, float2 *scratch, unsigned long long n_pow2,
                               int inverse) {
	ARG_TRY(ctx, n_pow2 >= 2);
	FftOpts o; memset(&o, 0, sizeof o); o.batch = 1; o.scale = inverse ? 1.0f : 1.0f / (float) n_pow2; o.exact = true;
	if (in != out) { o.cplx_in = in; o.cplx_bs = 0; }
	return fft_run(ctx, stream, out, scratch, ilog2(n_pow2), inverse, o);
}
// *d_result = index of the first maximum of |x[0..n)|; d_part: room for 2 * TSDRGPU_ARGMAX_PARTS 32-bit words
int tsdrgpu_argmax_mag_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *x, unsigned n, void *d_part, int *d_result) {
	unsigned parts = (n + 4095) / 4096; if (parts > TSDRGPU_ARGMAX_PARTS) parts = TSDRGPU_ARGMAX_PARTS; if (parts < 1) parts = 1;
	float *pv = (float *) d_part; unsigned *pi = (unsigned *) d_part + TSDRGPU_ARGMAX_PARTS;
	KL(ctx, "k_argmax", stream, k_argmax_partial<<<parts, 256, 0, stream>>>(x, n, pv, pi));
	KL(ctx, "k_argmax", stream, k_argmax_final<<<1, 256, 0, stream>>>(pv, pi, parts, d_result));
	return TSDRGPU_OK;
}

struct tsdrgpu_frd {
	tsdrgpu_ctx_t *ctx;
	DeviceBuf<float> d_big;                       // extbuff (2*size floats), only where the answers are materialised (see frd_run_impl)
	DeviceBuf<double> d_p1, d_p2;                 // the two running means, one element more than the plots
	uint64_t calls; int fresh;
	DeviceBuf<int> d_peaks;                       // first strict maximum of each plot (k_plot_peaks), refreshed with every run
	// overlapped mode (tsdrgpu_frd_set_overlap): everything a run launches goes to an internal stream, behind what the caller's
	// stream held at the call, with work buffers of its own -- the transforms then share the chip with whatever the caller
	// enqueues next (the pass kernels are bound by issue slots, the resampler and the frame stage by other things)
	int overlap, pending;
	cudaStream_t s_side; cudaEvent_t ev_in, ev_done;
	DeviceBuf<float2> w0, w1;
};

extern "C" {

uint32_t tsdrgpu_fft_getrealsize(uint32_t size) {          // fft.c:5-11
	uint32_t m = 0;
	while ((size /= 2) != 0) m++;
	return 1u << m;
}

int tsdrgpu_fft(tsdrgpu_ctx_t *ctx, void *stream, float *d_iq, uint32_t size, int inverse) {
	BIND(ctx); ARG_TRY(ctx, d_iq != NULL);
	if (size == 0) return TSDRGPU_OK;
	return tsdrgpu_fft_internal(ctx, (cudaStream_t) stream, reinterpret_cast<float2 *>(d_iq), tsdrgpu_fft_getrealsize(size), inverse);
}

// batch of independent autocorrelations: transform b reads d_real + b*real_stride (floats) and writes
// d_answer + b*answer_stride (floats, 2*size each).  skip_tail leaves answer[2N .. 2*size) untouched (the
// frame-rate detector never reads lags >= N).
// last[k] = exp(-i pi k / half (1 + eps)), k < half: the reference's final radix-2 stage of an (2 half)-point transform
static int last_stage_table(tsdrgpu_ctx_t *ctx, unsigned half, double eps, const float2 **out) {
	return fft_table(ctx, {TAB_LAST, half, 0, 0, eps}, half, [&](float2 *h) {
		for (unsigned k = 0; k < half; k++) {
			const double ang = -3.14159265358979323846 * ((double) k / (double) half) * (1.0 + eps);
			h[k] = make_float2((float) cos(ang), (float) sin(ang));
		}
	}, out);
}

// Default path (TSDRGPU_AUTOCORR_FULL=1 opts out): both transforms of the autocorrelation at half size.  The capture and |X|/N
// are real; a real sequence of length N is a complex one of length N/2, one N/2-point transform + the reference's last radix-2
// stage (real_split_rn) gives the N-point result.  Neither finish is a pass of its own: the forward's is formed by the inverse's
// first pass as it loads (FftPass.in_real = 3), the inverse's by k_real_inv_finish for callers that want every lag or by
// k_accumulate_half for the frame-rate detector, which only reads its two windows.  profiles/studies/real_input_autocorr_study.py
// measures the only approximation (the mirror identity under perturbed stage angles): 6.6e-10 of the zero-lag peak at 2^20,
// 7.9e-9 at 2^22.
static bool autocorr_half_size(unsigned long long N) { return N >= 16 && getenv("TSDRGPU_AUTOCORR_FULL") == NULL; }     // read per call: the tests flip it inside one process

// How many captures share one pair of work buffers (TSDRGPU_AUTOCORR_GROUP; default: the whole batch).  Small groups would keep
// the intermediates of the four passes inside the L2 instead of streaming them through HBM, but the pass kernel is bound by
// issue slots and shared-memory traffic, not by HBM, and a small group runs in partial waves (128 CTAs per capture against
// three resident CTAs per SM).  profiles/studies/autocorr_group_sweep.py measures the trade; the knob stays for studies.
static unsigned autocorr_group(unsigned long long N, unsigned batch) {
	(void) N;
	const int forced = getenv("TSDRGPU_AUTOCORR_GROUP") ? atoi(getenv("TSDRGPU_AUTOCORR_GROUP")) : 0;       // read per call
	if (forced > 0 && (unsigned) forced < batch) return (unsigned) forced;
	return batch;
}

// the frame-rate detector's two running means (frameratedetector.c:34-62): lags [start1, start1 + len1) into p1, [start2, ...)
// into p2, all below N; the first capture of the batch is call number first_calls
struct RunningMeans { double *p1, *p2; int start1, len1, start2, len2; unsigned long long first_calls; };

struct WorkBufs { float2 *w0, *w1; };                     // caller-owned work buffers (NULL: the context's scratch slots 0 and 1)
// every lag of every capture into ans (rm == NULL), or only the lags of the running means, folded into them (rm != NULL; ans unused)
static int autocorrelation_batch_half(tsdrgpu_ctx_t *ctx, cudaStream_t stream, float2 *ans, long long ans_bs, const float *d_real,
                                      long long real_stride, unsigned long long N, unsigned batch, const RunningMeans *rm, WorkBufs wb) {
	const unsigned log2N = ilog2(N), half = (unsigned) (N >> 1);
	double eps_all[40];
	tsdrgpu_fft_reference_eps((int) log2N, 0, eps_all);
	const float2 *last;
	int rc = last_stage_table(ctx, half, tsdrgpu_fft_true_dft() ? 0.0 : eps_all[log2N - 1], &last);
	if (rc) return rc;
	const unsigned G = autocorr_group(N, batch);
	void *w0_ = wb.w0, *w1_ = wb.w1;
	if (!w0_ && (rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * half * G, &w0_))) return rc;
	if (!w1_ && (rc = tsdrgpu_scratch(ctx, 1, sizeof(float2) * half * G, &w1_))) return rc;
	float2 *W0 = (float2 *) w0_, *W1 = (float2 *) w1_;
	// the inverse's first pass reads Z (in W1) while other CTAs write: to the scratch W0 on multi-pass plans (Z' then lands in
	// W1), to its output on one-pass plans (Z' lands in W0)
	float2 *Zi = (log2N - 1 <= (unsigned) FFT_MAX_LOG2L) ? W0 : W1;
	for (unsigned g0 = 0; g0 < batch; g0 += G) {
		const unsigned gb = (batch - g0 < G) ? (batch - g0) : G;
		// forward: Z = FFT_{N/2}(capture viewed as complex pairs), unscaled: capture -> W0 -> W1
		FftOpts f; memset(&f, 0, sizeof f);
		f.scale = 1.0f; f.batch = gb; f.data_bs = (long long) half; f.scratch_bs = (long long) half;
		const float *cap0 = d_real + (long long) g0 * real_stride;
		if ((real_stride & 1) || (reinterpret_cast<unsigned long long>(cap0) & 7ull)) { f.pair_in = cap0; f.pair_bs = real_stride; }   // odd capture sizes: every other capture starts on an odd sample
		else { f.cplx_in = reinterpret_cast<const float2 *>(cap0); f.cplx_bs = real_stride / 2; }
		if ((rc = fft_run(ctx, stream, W1, W0, log2N - 1, 0, f))) return rc;
		// inverse: Z' = IFFT_{N/2}(z'), z'[n] = (R[2n], R[2n+1]) with R = |X| / N formed from Z on load
		FftOpts gopt; memset(&gopt, 0, sizeof gopt);
		gopt.scale = 1.0f; gopt.batch = gb; gopt.data_bs = (long long) half; gopt.scratch_bs = (long long) half;
		gopt.split_in = W1; gopt.split_bs = (long long) half; gopt.split_last = last; gopt.split_scale = 1.0f / (float) N;
		if ((rc = fft_run(ctx, stream, Zi, W0, log2N - 1, 1, gopt))) return rc;
		if (rm) {                                      // before the next group reuses the work buffers; captures stay in order
			if (rm->len1) KL(ctx, "k_accumulate", stream, k_accumulate_half<<<grid1d((unsigned long long) rm->len1, ctx->sm_count), 256, 0, stream>>>(
				rm->p1, rm->first_calls + g0, Zi, (long long) half, gb, last, half, rm->start1, rm->len1));
			if (rm->len2) KL(ctx, "k_accumulate", stream, k_accumulate_half<<<grid1d((unsigned long long) rm->len2, ctx->sm_count), 256, 0, stream>>>(
				rm->p2, rm->first_calls + g0, Zi, (long long) half, gb, last, half, rm->start2, rm->len2));
		} else KL(ctx, "k_real_inv_finish", stream, k_real_inv_finish<<<dim3(grid1d(half, ctx->sm_count), gb), 256, 0, stream>>>(
			Zi, (long long) half, last, half, ans + (long long) g0 * ans_bs, ans_bs));
	}
	return TSDRGPU_OK;
}

static int autocorrelation_batch(tsdrgpu_ctx_t *ctx, cudaStream_t stream, float *d_answer, long long answer_stride,
                                 const float *d_real, long long real_stride, uint32_t size, unsigned batch, bool skip_tail,
                                 WorkBufs wb = WorkBufs{NULL, NULL}) {
	int rc;
	const unsigned long long N = tsdrgpu_fft_getrealsize(size);
	float2 *ans = reinterpret_cast<float2 *>(d_answer);
	if (N == 1 || !skip_tail) {
		for (unsigned b = 0; b < batch; b++) {       // the part that never enters a transform (fft.c:52-60): (|x|, 0)
			const unsigned long long from = (N == 1) ? 0 : N;
			if (from >= size) break;
			float2 *a = reinterpret_cast<float2 *>(d_answer + (long long) b * answer_stride);
			KL(ctx, "k_real_to_complex", stream, k_real_to_complex<<<grid1d(size - from, ctx->sm_count), 256, 0, stream>>>(a, d_real + (long long) b * real_stride, from, size));
			KL(ctx, "k_abs", stream, k_abs<<<grid1d(size - from, ctx->sm_count), 256, 0, stream>>>(a, from, size));
		}
		if (N == 1) return TSDRGPU_OK;
	}
	// default: both transforms at half size (autocorrelation_batch_half); TSDRGPU_AUTOCORR_FULL=1 keeps the N-point transforms
	if (autocorr_half_size(N) && (answer_stride & 1) == 0)
		return autocorrelation_batch_half(ctx, stream, ans, answer_stride / 2, d_real, real_stride, N, batch, NULL, wb);
	void *scratch = wb.w0;                              // (sized for N * batch by the overlapped detector)
	if (!scratch && (rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * N * batch, &scratch))) return rc;
	// forward transform of the first N samples, real input widened on load, |X|/N on store
	FftOpts f; memset(&f, 0, sizeof f);
	f.real_in = d_real; f.out_abs = true; f.scale = 1.0f / (float) N; f.batch = batch;
	f.data_bs = answer_stride / 2; f.scratch_bs = (long long) N; f.real_bs = real_stride;
	if ((rc = fft_run(ctx, stream, ans, (float2 *) scratch, ilog2(N), 0, f))) return rc;
	FftOpts g; memset(&g, 0, sizeof g);
	g.scale = 1.0f; g.batch = batch; g.data_bs = answer_stride / 2; g.scratch_bs = (long long) N;
	return fft_run(ctx, stream, ans, (float2 *) scratch, ilog2(N), 1, g);
}

int tsdrgpu_autocorrelation(tsdrgpu_ctx_t *ctx, void *stream, float *d_answer, const float *d_real, uint32_t size) {
	BIND(ctx); ARG_TRY(ctx, d_answer != NULL && d_real != NULL);
	if (size == 0) return TSDRGPU_OK;
	return autocorrelation_batch(ctx, (cudaStream_t) stream, d_answer, 2ll * size, d_real, size, size, 1, false);
}

int tsdrgpu_autocorrelation_batch(tsdrgpu_ctx_t *ctx, void *stream, float *d_answers, const float *d_reals, uint32_t size,
                                  uint32_t batch, uint64_t real_stride) {
	BIND(ctx); ARG_TRY(ctx, d_answers != NULL && d_reals != NULL && (size & 1) == 0);
	if (size == 0 || batch == 0) return TSDRGPU_OK;
	return autocorrelation_batch(ctx, (cudaStream_t) stream, d_answers, 2ll * size, d_reals, (long long) real_stride, size, batch, false);
}

int tsdrgpu_crosscorrelation(tsdrgpu_ctx_t *ctx, void *stream_, float *d_a, float *d_b, uint32_t samples) {
	BIND(ctx); ARG_TRY(ctx, d_a != NULL && d_b != NULL);
	if (samples == 0) return TSDRGPU_OK;
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = tsdrgpu_fft_getrealsize(samples);
	int rc;
	if ((rc = tsdrgpu_fft_internal(ctx, stream, reinterpret_cast<float2 *>(d_a), N, 0))) return rc;
	if ((rc = tsdrgpu_fft_internal(ctx, stream, reinterpret_cast<float2 *>(d_b), N, 0))) return rc;
	KL(ctx, "k_conj_mul", stream, k_conj_mul<<<grid1d(N, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<float2 *>(d_a), reinterpret_cast<const float2 *>(d_b), N));
	return tsdrgpu_fft_internal(ctx, stream, reinterpret_cast<float2 *>(d_a), N, 1);
}

int tsdrgpu_accumulate(tsdrgpu_ctx_t *ctx, void *stream, double *d_out, uint64_t calls, const float *d_in, int startid, int length) {
	BIND(ctx); ARG_TRY(ctx, d_out != NULL && d_in != NULL && length >= 0 && startid >= 0);
	if (length == 0) return TSDRGPU_OK;
	KL(ctx, "k_accumulate", (cudaStream_t) stream, k_accumulate<<<grid1d((unsigned long long) length, ctx->sm_count), 256, 0, (cudaStream_t) stream>>>(d_out, calls, reinterpret_cast<const float2 *>(d_in), startid, length));
	return TSDRGPU_OK;
}

// ---- frame-rate detector ---------------------------------------------------------------------------------------
// the side stream and its two events, whichever exist
static void destroy_side(tsdrgpu_frd *f) {
	if (f->s_side) cudaStreamDestroy(f->s_side);
	if (f->ev_in) cudaEventDestroy(f->ev_in);
	if (f->ev_done) cudaEventDestroy(f->ev_done);
	f->s_side = NULL; f->ev_in = f->ev_done = NULL;
}
// a detector whole or half built; its buffers go with the object
static void release(tsdrgpu_frd *f) {
	destroy_side(f);
	delete f;
}

static int create_handles(tsdrgpu_frd *f) {
	CU_TRY(f->ctx, f->d_peaks.assign(64));
	CU_TRY(f->ctx, cudaMemset(f->d_peaks.ptr, 0, 256));
	return TSDRGPU_OK;
}

int tsdrgpu_frd_create(tsdrgpu_ctx_t *ctx, tsdrgpu_frd_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_frd *f = new tsdrgpu_frd();      // value-initialised: every field not set here starts at zero
	f->ctx = ctx; f->fresh = 1;
	const int rc = create_handles(f);
	if (rc) { release(f); return rc; }
	*out = f;
	return TSDRGPU_OK;
}
// the side stream and its two events, all three or none
static int create_side(tsdrgpu_frd *f) {
	tsdrgpu_ctx_t *ctx = f->ctx;
	// the detector's work is background work (a plot every few frames): lowest priority, so that the block scheduler hands free
	// SM resources to the pixel path first and lets the transforms fill what is left (TSDRGPU_FRD_PRIO=high|default for studies)
	int lo = 0, hi = 0;
	CU_TRY(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
	const char *pr = getenv("TSDRGPU_FRD_PRIO");
	const int prio = (pr && !strcmp(pr, "high")) ? hi : ((pr && !strcmp(pr, "default")) ? 0 : lo);
	CU_TRY(ctx, cudaStreamCreateWithPriority(&f->s_side, cudaStreamNonBlocking, prio));
	CU_TRY(ctx, cudaEventCreateWithFlags(&f->ev_in, cudaEventDisableTiming));
	CU_TRY(ctx, cudaEventCreateWithFlags(&f->ev_done, cudaEventDisableTiming));
	return TSDRGPU_OK;
}
// overlapped mode on/off (see struct tsdrgpu_frd).  While it is on, a capture handed to tsdrgpu_frd_run* must stay untouched
// until tsdrgpu_frd_join (or the next synchronising call) has put the caller's stream behind the run.
int tsdrgpu_frd_set_overlap(tsdrgpu_frd_t *f, int on) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	tsdrgpu_ctx_t *ctx = f->ctx;
	BIND(ctx);
	if (on && !f->s_side) {
		const int rc = create_side(f);
		if (rc) { destroy_side(f); return rc; }         // none of the three stays: the next call starts again
	}
	if (!on && f->pending) { CU_TRY(ctx, cudaStreamSynchronize(f->s_side)); f->pending = 0; }
	f->overlap = on ? 1 : 0;
	return TSDRGPU_OK;
}
// `stream` waits (on the device) for the detector's last overlapped run; a no-op otherwise
int tsdrgpu_frd_join(tsdrgpu_frd_t *f, void *stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	BIND(f->ctx);
	if (f->pending) CU_TRY(f->ctx, cudaStreamWaitEvent((cudaStream_t) stream, f->ev_done, 0));
	return TSDRGPU_OK;
}
void tsdrgpu_frd_destroy(tsdrgpu_frd_t *f) {
	if (!f) return;
	cudaSetDevice(f->ctx->device); cudaDeviceSynchronize();
	release(f);
}
int tsdrgpu_frd_reset(tsdrgpu_frd_t *f) { if (!f) return TSDRGPU_EINVAL; f->fresh = 1; return TSDRGPU_OK; }

uint32_t tsdrgpu_frd_capture_size(uint32_t samplerate) { return (uint32_t) (3.1 * samplerate / (double) (55)); }   // frameratedetector.c:160
void tsdrgpu_frd_windows(uint32_t samplerate, int *frame_min, int *frame_max, int *line_min, int *line_max) {
	*frame_max = (int) (samplerate / (double) (55));               // frameratedetector.c:91-95
	*frame_min = (int) (samplerate / (double) (87));
	*line_max = (int) (samplerate / (double) (590 * 55));
	*line_min = (int) (samplerate / (double) (1500 * 87));
}

static int frd_run_impl(tsdrgpu_frd_t *f, void *stream_, uint32_t samplerate, const float *d_capture, uint32_t size,
                        uint32_t batch, uint64_t capture_stride,
                        double *h_frame_plot, int frame_cap, double *h_line_plot, int line_cap, uint64_t *calls, bool synchronise) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	tsdrgpu_ctx_t *ctx = f->ctx;
	BIND(ctx); ARG_TRY(ctx, d_capture != NULL && size > 0 && batch > 0);
	cudaStream_t caller = (cudaStream_t) stream_, stream = caller;
	int fmin, fmax, lmin, lmax;
	tsdrgpu_frd_windows(samplerate, &fmin, &fmax, &lmin, &lmax);
	const int flen = fmax - fmin, llen = lmax - lmin;
	const uint32_t N = tsdrgpu_fft_getrealsize(size);
	ARG_TRY(ctx, (uint64_t) fmax <= (uint64_t) size && flen >= 0 && llen >= 0);
	const bool skip_tail = (uint32_t) fmax <= N;               // always true for the detector's own capture size
	// default: the running means are taken straight from the half-size inverse's output, no lag is stored; otherwise (N-point
	// transforms, or lags beyond the transformed ones) the answers are materialised in d_big and read back
	const bool fold = skip_tail && autocorr_half_size(N);
	WorkBufs wb = WorkBufs{NULL, NULL};
	if (f->overlap) {
		// the internal stream picks up behind everything the caller's stream holds now (the capture is complete there)
		stream = f->s_side;
		const size_t need0 = (size_t) N * batch, need1 = (size_t) (N / 2) * batch + 16;
		if (f->w0.cap < need0 || f->w1.cap < need1) {
			CU_TRY(ctx, cudaStreamSynchronize(f->s_side));
			CU_TRY(ctx, f->w0.assign(need0));
			CU_TRY(ctx, f->w1.assign(need1));
		}
		wb = WorkBufs{f->w0.ptr, f->w1.ptr};
		CU_TRY(ctx, cudaEventRecord(f->ev_in, caller));
		CU_TRY(ctx, cudaStreamWaitEvent(f->s_side, f->ev_in, 0));
	}
	if (f->d_p1.cap <= (size_t) flen || f->fresh) {
		if (f->d_p1.cap <= (size_t) flen) { CU_TRY(ctx, cudaStreamSynchronize(stream)); CU_TRY(ctx, f->d_p1.assign((size_t) flen + 1)); }
		CU_TRY(ctx, cudaMemsetAsync(f->d_p1.ptr, 0, sizeof(double) * (flen + 1), stream));
	}
	if (f->d_p2.cap <= (size_t) llen || f->fresh) {
		if (f->d_p2.cap <= (size_t) llen) { CU_TRY(ctx, cudaStreamSynchronize(stream)); CU_TRY(ctx, f->d_p2.assign((size_t) llen + 1)); }
		CU_TRY(ctx, cudaMemsetAsync(f->d_p2.ptr, 0, sizeof(double) * (llen + 1), stream));
	}
	if (f->fresh) { f->calls = 0; f->fresh = 0; }
	const uint64_t first_calls = f->calls + 1;                  // extbuffer.c:81, one prepare per capture
	f->calls += batch;
	int rc;
	if (fold) {
		// only the two lag windows are ever read (frameratedetector.c:106-109)
		const RunningMeans rm = {f->d_p1.ptr, f->d_p2.ptr, fmin, flen, lmin, llen, first_calls};
		if ((rc = autocorrelation_batch_half(ctx, stream, NULL, 0, d_capture, (long long) capture_stride, N, batch, &rm, wb))) return rc;
	} else {
		const size_t big_need = 2ull * size * batch;
		if (f->d_big.cap < big_need) {
			CU_TRY(ctx, cudaStreamSynchronize(stream));
			CU_TRY(ctx, f->d_big.assign(big_need));
		}
		if ((rc = autocorrelation_batch(ctx, stream, f->d_big.ptr, 2ll * size, d_capture, (long long) capture_stride, size, batch, skip_tail, wb))) return rc;
		if (flen) KL(ctx, "k_accumulate", stream, k_accumulate_batch<<<grid1d((unsigned long long) flen, ctx->sm_count), 256, 0, stream>>>(f->d_p1.ptr, first_calls, reinterpret_cast<const float2 *>(f->d_big.ptr), (long long) size, batch, fmin, flen));
		if (llen) KL(ctx, "k_accumulate", stream, k_accumulate_batch<<<grid1d((unsigned long long) llen, ctx->sm_count), 256, 0, stream>>>(f->d_p2.ptr, first_calls, reinterpret_cast<const float2 *>(f->d_big.ptr), (long long) size, batch, lmin, llen));
	}
	KL(ctx, "k_plot_peaks", stream, k_plot_peaks<<<2, 1024, 0, stream>>>(f->d_p1.ptr, flen, f->d_p2.ptr, llen, f->d_peaks.ptr));
	if (calls) *calls = f->calls;
	if (h_frame_plot || h_line_plot) {
		if (h_frame_plot) CU_TRY(ctx, cudaMemcpyAsync(h_frame_plot, f->d_p1.ptr, sizeof(double) * (size_t) (flen < frame_cap ? flen : frame_cap), cudaMemcpyDeviceToHost, stream));
		if (h_line_plot) CU_TRY(ctx, cudaMemcpyAsync(h_line_plot, f->d_p2.ptr, sizeof(double) * (size_t) (llen < line_cap ? llen : line_cap), cudaMemcpyDeviceToHost, stream));
		if (synchronise) CU_TRY(ctx, cudaStreamSynchronize(stream));
	}
	if (f->overlap) { CU_TRY(ctx, cudaEventRecord(f->ev_done, f->s_side)); f->pending = 1; }
	return TSDRGPU_OK;
}

int tsdrgpu_frd_run(tsdrgpu_frd_t *f, void *stream, uint32_t samplerate, const float *d_capture, uint32_t size,
                    double *h_frame_plot, int frame_cap, double *h_line_plot, int line_cap, uint64_t *calls) {
	return frd_run_impl(f, stream, samplerate, d_capture, size, 1, size, h_frame_plot, frame_cap, h_line_plot, line_cap, calls, true);
}
int tsdrgpu_frd_run_batch(tsdrgpu_frd_t *f, void *stream, uint32_t samplerate, const float *d_captures, uint32_t size, uint32_t batch,
                          uint64_t capture_stride, uint64_t *calls) {
	return frd_run_impl(f, stream, samplerate, d_captures, size, batch, capture_stride, NULL, 0, NULL, 0, calls, false);
}
int tsdrgpu_frd_run_async(tsdrgpu_frd_t *f, void *stream, uint32_t samplerate, const float *d_capture, uint32_t size,
                          double *h_frame_plot_pinned, int frame_cap, double *h_line_plot_pinned, int line_cap, uint64_t *calls) {
	return frd_run_impl(f, stream, samplerate, d_capture, size, 1, size, h_frame_plot_pinned, frame_cap, h_line_plot_pinned, line_cap, calls, false);
}

// dump_autocorrect (frameratedetector.c:64-85): the autocorrelation of ONE capture as a CSV of (lag in ms, 10 log10 |r|) for the
// lags the reference writes (i < fft_getrealsize(2 size) / 2 floats, i.e. the first half of the transformed lags), same header and
// "%f, %f" rows.  A debugging aid of the GUI (PARAM_AUTOCORR_DUMP): one extra autocorrelation with every lag produced, a device-to-
// host copy and a synchronisation, only when asked for.  Does not touch the running means.
int tsdrgpu_frd_dump_csv(tsdrgpu_frd_t *f, void *stream_, uint32_t samplerate, const float *d_capture, uint32_t size, const char *path) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	tsdrgpu_ctx_t *ctx = f->ctx;
	BIND(ctx); ARG_TRY(ctx, d_capture != NULL && size > 0 && path != NULL && samplerate > 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	const uint32_t maxels = tsdrgpu_fft_getrealsize(2u * size) / 2u;           // floats of the answer the reference walks
	std::vector<float> h(maxels);
	{   // the device answer goes at the end of this block, after the stream is done with it
		DeviceBuf<float> d_ans;
		CU_TRY(ctx, d_ans.assign(2ull * size));
		int rc = autocorrelation_batch(ctx, stream, d_ans.ptr, 2ll * size, d_capture, (long long) size, size, 1, false);
		if (rc == TSDRGPU_OK) {
			const cudaError_t e1 = cudaMemcpyAsync(h.data(), d_ans.ptr, sizeof(float) * maxels, cudaMemcpyDeviceToHost, stream);
			const cudaError_t e2 = (e1 == cudaSuccess) ? cudaStreamSynchronize(stream) : e1;
			if (e2 != cudaSuccess) rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "autocorrelation dump: copy", e2, __FILE__, __LINE__);
		} else cudaStreamSynchronize(stream);
		if (rc != TSDRGPU_OK) return rc;
	}
	FILE *fp = fopen(path, "w");
	if (!fp) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "autocorrelation dump: cannot open the file", cudaSuccess, __FILE__, __LINE__);
	fprintf(fp, "%s, %s\n", "ms", "dB");
	for (uint32_t i = 0; i < maxels; i += 2) {
		const double I = (double) h[i], Q = (i + 1 < maxels) ? (double) h[i + 1] : 0.0;
		const double db = 10.0 * log10(sqrt(I * I + Q * Q));
		const double t = 1000.0 * (double) (i / 2) / (double) samplerate;
		fprintf(fp, "%f, %f\n", t, db);
	}
	fclose(fp);
	return TSDRGPU_OK;
}

int tsdrgpu_frd_get_plots(tsdrgpu_frd_t *f, void *stream_, uint32_t samplerate, double *h_frame_plot, int frame_cap,
                          double *h_line_plot, int line_cap) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	tsdrgpu_ctx_t *ctx = f->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	int fmin, fmax, lmin, lmax;
	tsdrgpu_frd_windows(samplerate, &fmin, &fmax, &lmin, &lmax);
	const int flen = fmax - fmin, llen = lmax - lmin;
	ARG_TRY(ctx, f->d_p1.cap > (size_t) flen && f->d_p2.cap > (size_t) llen);
	if (f->pending) CU_TRY(ctx, cudaStreamWaitEvent(stream, f->ev_done, 0));
	if (h_frame_plot) CU_TRY(ctx, cudaMemcpyAsync(h_frame_plot, f->d_p1.ptr, sizeof(double) * (size_t) (flen < frame_cap ? flen : frame_cap), cudaMemcpyDeviceToHost, stream));
	if (h_line_plot) CU_TRY(ctx, cudaMemcpyAsync(h_line_plot, f->d_p2.ptr, sizeof(double) * (size_t) (llen < line_cap ? llen : line_cap), cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	return TSDRGPU_OK;
}

// SURVEY 8f-3: where the two plots peak, picked on the device right after the running means were updated.
// h_peaks[0] = frame plot, [1] = line plot (indices into the plots; add the window offsets for lags).  tsdrgpu_frd_peaks
// synchronises; the _async form needs page-locked memory and is valid once the stream has passed it.
// stage-level entry: the same reduction on any two device-resident plots (synchronises)
int tsdrgpu_plot_peaks(tsdrgpu_ctx_t *ctx, void *stream_, const double *d_frame_plot, int frame_len, const double *d_line_plot, int line_len, int32_t *h_peaks) {
	BIND(ctx); ARG_TRY(ctx, d_frame_plot && d_line_plot && frame_len >= 0 && line_len >= 0 && h_peaks);
	cudaStream_t stream = (cudaStream_t) stream_;
	void *d;
	int rc = tsdrgpu_scratch(ctx, 3, 256, &d);
	if (rc) return rc;
	KL(ctx, "k_plot_peaks", stream, k_plot_peaks<<<2, 1024, 0, stream>>>(d_frame_plot, frame_len, d_line_plot, line_len, (int *) d));
	CU_TRY(ctx, cudaMemcpyAsync(h_peaks, d, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	return TSDRGPU_OK;
}
int tsdrgpu_frd_peaks_async(tsdrgpu_frd_t *f, void *stream, int32_t *h_peaks_pinned) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL && h_peaks_pinned != NULL);
	BIND(f->ctx);
	if (f->pending) CU_TRY(f->ctx, cudaStreamWaitEvent((cudaStream_t) stream, f->ev_done, 0));
	CU_TRY(f->ctx, cudaMemcpyAsync(h_peaks_pinned, f->d_peaks.ptr, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t) stream));
	return TSDRGPU_OK;
}
int tsdrgpu_frd_peaks(tsdrgpu_frd_t *f, void *stream, int32_t *h_peaks) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL && h_peaks != NULL);
	BIND(f->ctx);
	if (f->pending) CU_TRY(f->ctx, cudaStreamWaitEvent((cudaStream_t) stream, f->ev_done, 0));
	CU_TRY(f->ctx, cudaMemcpyAsync(h_peaks, f->d_peaks.ptr, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t) stream));
	CU_TRY(f->ctx, cudaStreamSynchronize((cudaStream_t) stream));
	return TSDRGPU_OK;
}

// ---- superbandwidth ----------------------------------------------------------------------------------------------
int tsdrgpu_complex_to_abs_diff(tsdrgpu_ctx_t *ctx, void *stream_, float *d_data, int size_floats) {
	BIND(ctx); ARG_TRY(ctx, d_data != NULL && size_floats >= 0 && (size_floats & 1) == 0);
	if (size_floats == 0) return TSDRGPU_OK;
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long pairs = (unsigned long long) size_floats / 2;
	void *tmp; int rc;
	if ((rc = tsdrgpu_scratch(ctx, 1, sizeof(float2) * pairs, &tmp))) return rc;
	KL(ctx, "k_abs_diff", stream, k_abs_diff<<<grid1d(pairs, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_data), (float2 *) tmp, pairs));
	CU_TRY(ctx, cudaMemcpyAsync(d_data, tmp, sizeof(float2) * pairs, cudaMemcpyDeviceToDevice, stream));
	return TSDRGPU_OK;
}

// the lag (in complex samples) of hop i against hop 0, left in device memory at d_lag -- no host round trip
static int superb_bestfit_dev(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *d_hop0, const float *d_hopi, int size_floats,
                              int samples_in_frame, int *d_lag) {
	int size = (size_floats / samples_in_frame) * samples_in_frame;      // superbandwidth.c:84-86
	ARG_TRY(ctx, size >= 2);
	size = (int) tsdrgpu_fft_getrealsize((uint32_t) size);
	const unsigned long long pairs = (unsigned long long) size / 2;
	void *wa, *wb, *part; int rc;
	if ((rc = tsdrgpu_scratch(ctx, 1, sizeof(float2) * pairs + 256, &wa))) return rc;
	if ((rc = tsdrgpu_scratch(ctx, 2, sizeof(float2) * pairs + 8 * TSDRGPU_ARGMAX_PARTS + 256, &wb))) return rc;
	KL(ctx, "k_abs_diff", stream, k_abs_diff<<<grid1d(pairs, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hop0), (float2 *) wa, pairs));
	KL(ctx, "k_abs_diff", stream, k_abs_diff<<<grid1d(pairs, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hopi), (float2 *) wb, pairs));
	if ((rc = tsdrgpu_crosscorrelation(ctx, stream, (float *) wa, (float *) wb, (uint32_t) pairs))) return rc;
	part = wb;                                            // wb is free again after the cross-correlation
	return tsdrgpu_argmax_mag_internal(ctx, stream, (const float2 *) wa, (unsigned) pairs, part, d_lag);
}

int tsdrgpu_superb_bestfit(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_hop0, const float *d_hopi, int size_floats,
                           int samples_in_frame, int *h_best_offset) {
	BIND(ctx); ARG_TRY(ctx, d_hop0 && d_hopi && h_best_offset && size_floats > 0 && samples_in_frame > 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	void *res; int rc;
	if ((rc = tsdrgpu_scratch(ctx, 3, 256, &res))) return rc;
	if ((rc = superb_bestfit_dev(ctx, stream, d_hop0, d_hopi, size_floats, samples_in_frame, (int *) res))) return rc;
	int lag = 0;
	CU_TRY(ctx, cudaMemcpyAsync(&lag, res, sizeof(int), cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	*h_best_offset = 2 * lag;
	return TSDRGPU_OK;
}

// superb_ondataready (superbandwidth.c:121-152) on one GPU.  Everything stays on the device: the H-1 alignment lags are left
// in device memory by the grid argmax, the rotations read them from there, and the host sees them once, at the end (one
// synchronisation per stitch instead of one per hop).
int tsdrgpu_superb_stitch(tsdrgpu_ctx_t *ctx, void *stream_, float *const *d_hops, int nhops, int count_pairs, int samples_in_frame,
                          float *d_out, int *h_best_offsets, int *h_total_samples) {
	BIND(ctx); ARG_TRY(ctx, d_hops && nhops > 0 && nhops <= 16 && count_pairs > 0 && d_out && h_best_offsets);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = tsdrgpu_fft_getrealsize((uint32_t) count_pairs);
	int rc;
	void *lags_;
	if ((rc = tsdrgpu_scratch(ctx, 3, 256, &lags_))) return rc;
	int *d_lags = (int *) lags_;
	CU_TRY(ctx, cudaMemsetAsync(d_lags, 0, sizeof(int) * 16, stream));
	for (int i = 1; i < nhops; i++)
		if ((rc = superb_bestfit_dev(ctx, stream, d_hops[0], d_hops[i], (int) (2 * N), samples_in_frame, d_lags + i))) return rc;
	for (int i = 0; i < nhops; i++) {
		float2 *spec = reinterpret_cast<float2 *>(d_out) + (size_t) i * N;
		KL(ctx, "k_rotate", stream, k_rotate_dev<<<grid1d(N, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hops[i]), spec, N, d_lags + i));
		if ((rc = tsdrgpu_fft_internal(ctx, stream, spec, N, 0))) return rc;
	}
	const unsigned long long total = N * (unsigned long long) nhops;
	const unsigned long long tp = 1ull << ilog2(total);            // fft_perform transforms the largest power of two (fft.c:101-105)
	if ((rc = tsdrgpu_fft_internal(ctx, stream, reinterpret_cast<float2 *>(d_out), tp, 1))) return rc;
	int lags[16];
	CU_TRY(ctx, cudaMemcpyAsync(lags, d_lags, sizeof(int) * 16, cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	for (int i = 0; i < nhops; i++) h_best_offsets[i] = 2 * lags[i];
	if (h_total_samples) *h_total_samples = (int) total;
	return TSDRGPU_OK;
}

// ---- one hop per GPU -------------------------------------------------------------------------------------------------
// what a rank contributes to the single all-gather: [ X = FFT_N(raw hop) | D = FFT_nd(first difference of |hop|) ]
int tsdrgpu_superb_local_spectra(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_hop, int count_pairs, int samples_in_frame,
                                 float *d_block, uint32_t *h_n, uint32_t *h_nd) {
	BIND(ctx); ARG_TRY(ctx, d_hop && d_block && count_pairs > 0 && samples_in_frame > 0 && h_n && h_nd);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = tsdrgpu_fft_getrealsize((uint32_t) count_pairs);
	int size = (int) ((2 * N / samples_in_frame) * samples_in_frame);          // superbandwidth.c:84-86 with bufsize = 2N floats
	ARG_TRY(ctx, size >= 2);
	size = (int) tsdrgpu_fft_getrealsize((uint32_t) size);
	const unsigned long long nd = (unsigned long long) size / 2;
	float2 *X = reinterpret_cast<float2 *>(d_block), *D = X + N;
	CU_TRY(ctx, cudaMemcpyAsync(X, d_hop, sizeof(float2) * N, cudaMemcpyDeviceToDevice, stream));
	int rc;
	if ((rc = tsdrgpu_fft_internal(ctx, stream, X, N, 0))) return rc;
	KL(ctx, "k_abs_diff", stream, k_abs_diff<<<grid1d(nd, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hop), D, nd));
	if ((rc = tsdrgpu_fft_internal(ctx, stream, D, nd, 0))) return rc;
	*h_n = (uint32_t) N; *h_nd = (uint32_t) nd;
	return TSDRGPU_OK;
}

// after the all-gather: the alignment lag of every hop against hop 0 (pairs), exact integers.  synchronises
int tsdrgpu_superb_lags(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_gathered, int nhops, uint64_t block_stride_complex,
                        uint32_t n, uint32_t nd, int *h_lags) {
	BIND(ctx); ARG_TRY(ctx, d_gathered && nhops > 0 && nhops <= 16 && h_lags && nd > 0 && (nd & (nd - 1)) == 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	const float2 *G = reinterpret_cast<const float2 *>(d_gathered);
	void *wa, *res; int rc;
	if ((rc = tsdrgpu_scratch(ctx, 1, sizeof(float2) * nd + 256, &wa))) return rc;
	if ((rc = tsdrgpu_scratch(ctx, 2, 256 + 8 * TSDRGPU_ARGMAX_PARTS + 256, &res))) return rc;
	h_lags[0] = 0;
	for (int q = 1; q < nhops; q++) {
		CU_TRY(ctx, cudaMemcpyAsync(wa, G + n, sizeof(float2) * nd, cudaMemcpyDeviceToDevice, stream));            // D_0
		KL(ctx, "k_conj_mul", stream, k_conj_mul<<<grid1d(nd, ctx->sm_count), 256, 0, stream>>>((float2 *) wa, G + (size_t) q * block_stride_complex + n, nd));
		if ((rc = tsdrgpu_fft_internal(ctx, stream, (float2 *) wa, nd, 1))) return rc;
		if ((rc = tsdrgpu_argmax_mag_internal(ctx, stream, (const float2 *) wa, nd, (char *) res + 256, (int *) res + q))) return rc;
	}
	CU_TRY(ctx, cudaMemcpyAsync(h_lags + 1, (int *) res + 1, sizeof(int) * (nhops - 1), cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	return TSDRGPU_OK;
}

// this rank's strided residue of the H*N-point inverse, from the gathered RAW spectra and the lags
int tsdrgpu_superb_residue_ifft_lag(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_gathered, int nhops, uint64_t block_stride_complex,
                                    uint32_t n, int residue, const int *h_lags, float *d_out) {
	BIND(ctx); ARG_TRY(ctx, d_gathered && d_out && h_lags && nhops > 0 && nhops <= 16 && n > 0 && residue >= 0 && residue < nhops && (n & (n - 1)) == 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	LagSet ls; for (int q = 0; q < 16; q++) ls.lag[q] = q < nhops ? h_lags[q] : 0;
	KL(ctx, "k_residue_mix", stream, k_residue_mix_lag<<<grid1d(n, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_gathered), (long long) block_stride_complex, nhops, n, residue, ls, reinterpret_cast<float2 *>(d_out)));
	return tsdrgpu_fft_internal(ctx, stream, reinterpret_cast<float2 *>(d_out), n, 1);
}

}  // extern "C"

// ---- Welch spectrum (definition in tsdrgpu.h) -----------------------------------------------------------------------------
// The segments of a run are windowed on load (FftPass.win), transformed with exact stage angles, and their |X|^2 summed per bin by
// the accumulating last pass (fft_acc_kernel) into rows of partial sums: CTA row r walks segments r, r + rows, ... of a launch, so
// HBM sees each pair about once (the overlapping half of the next segment is read by a neighbouring CTA at about the same time,
// from the L2) and rows x N partial sums instead of a spectrum per segment.  k_spectrum_finish adds the rows in order.
namespace {

constexpr unsigned SP_MIN_SEGS_PER_ROW = 8;                 // a launch of n segments uses at most n / 8 rows (fewer partial sums)
constexpr unsigned long long SP_SCRATCH_POINTS = 1ull << 22; // two-pass plans: segments per first-pass launch x N (32 MB)

// report = scale * (row 0 + row 1 + ...) of acc, bin (i + N/2) mod N into value i
__global__ void __launch_bounds__(256) k_spectrum_finish(const double *__restrict__ acc, long long acc_bs, unsigned rows, unsigned n,
                                                         double scale, double *__restrict__ out) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const unsigned k = (i + n / 2) & (n - 1);
		double s = 0.0;
		for (unsigned r = 0; r < rows; r++) s = __dadd_rn(s, acc[(long long) r * acc_bs + k]);
		out[i] = __dmul_rn(s, scale);
	}
}

// the accumulating last pass of an N-point plan: line length, bundles per transform, threads and shared memory as launch_pass picks them
struct AccShape { int log2L; unsigned bundles; int threads; size_t smem; };
AccShape acc_shape(unsigned log2N) {
	AccShape a;
	int C = 1;
	if (log2N <= (unsigned) FFT_MAX_LOG2L) { a.log2L = (int) log2N; a.bundles = 1; }
	else {
		const unsigned l1 = log2N / 2;
		a.log2L = (int) (log2N - l1);
		C = bundle_for(a.log2L, 1ull << l1, true);
		a.bundles = (unsigned) ((1ull << l1) / C);
	}
	const int total = C << a.log2L, nstages = a.log2L / 3 + ((a.log2L % 3) ? 1 : 0);
	a.threads = (total / 8 + 31) / 32 * 32;
	a.smem = sizeof(float2) * (size_t) total * (nstages >= 3 ? 2 : 1);
	return a;
}
int acc_ctas_per_sm(int log2L, int threads, size_t smem, bool pair) {
	int nb = 0;
	cudaError_t e = cudaErrorInvalidValue;
	switch (log2L) {
#define CASE(l) case l: e = pair ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fft_acc2_kernel<l>, threads, smem) \
	                         : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fft_acc_kernel<l>, threads, smem); break
	CASE(6); CASE(7); CASE(8); CASE(9); CASE(10); CASE(11);
#undef CASE
	default: break;
	}
	return (e == cudaSuccess && nb > 0) ? nb : 1;
}

}  // namespace

// The segmentation the Welch spectrum and the coherence share: segments of N pairs with hop N/2, the open segment (fewer than N
// pairs) carried across runs in d_hist, and reports of K segments, each segment taken as per_seg transforms and summed into `planes`
// planes of N partial sums.  seg_run hands the completed segments of a run to `launch` in pieces of at most seg_chunk segments (all
// of them: 0) that stay inside one report, over at most rows_max rows of partial sums, and calls `finish` for every report completed.
struct SegStream {
	uint32_t N, K;                                // N == 0: no spec set yet
	unsigned per_seg, planes;                     // 1, 1: the spectrum; 2, 4: the coherence (fft_acc2_kernel)
	bool break_report;                            // a discontinuity also discards the report in progress
	int stale;                                    // the device buffers are not those of N yet: the next run (re)builds them
	DeviceBuf<float> d_hist, d_join;              // the open segment; the open segment followed by the head of a block
	DeviceBuf<double> d_acc;                      // rows_max rows of `planes` x N partial sums of the report in progress
	DeviceBuf<float2> d_scratch;                  // two-pass plans: the first pass's output for seg_chunk segments
	uint64_t open;                                // pairs of the open segment (in d_hist, fewer than N)
	uint64_t done;                                // completed segments of the report in progress (< K)
	unsigned rows_used, rows_max, seg_chunk;      // rows of partial sums that hold sums of the report in progress
	void reset() { open = 0; done = 0; rows_used = 0; }
	// reports the next run would complete
	uint32_t plan(uint64_t pairs, int discontinuity) const {
		const uint64_t total = (discontinuity ? 0 : open) + pairs, count = total >= N ? (total - N) / (N / 2) + 1 : 0;
		return (uint32_t) (((discontinuity && break_report ? 0 : done) + count) / K);
	}
};

// launch(src, first, n, rows, keep): n consecutive segments from src (pairs, N/2 apart), segments first .. first + n - 1 of the
// report in progress, summed into `rows` rows of which the first `keep` add to what they hold.  finish(r): report r of the run.
template <class Launch, class Finish>
int seg_run(tsdrgpu_ctx_t *ctx, SegStream &g, cudaStream_t stream, const float *d_iq, uint64_t pairs, int discontinuity, Launch launch,
            Finish finish, uint32_t *h_nreports) {
	int rc;
	*h_nreports = 0;
	if (discontinuity) { if (g.break_report) g.reset(); else g.open = 0; }
	if (pairs == 0) return TSDRGPU_OK;
	const uint64_t N = g.N, H = N / 2, L = g.open, total = L + pairs;
	const uint64_t count = total >= N ? (total - N) / H + 1 : 0;        // segments completed by this run, q = 0 .. count-1
	const uint64_t nj = count < (L + H - 1) / H ? count : (L + H - 1) / H;   // the ones that start in the open segment
	const uint64_t keep = total - count * H;                           // the next open segment: [count H, total)
	// segment q starts at q H of (open segment ++ block): the first nj are formed in d_join, the others read the block in place
	if (nj > 0 || count * H < L) {
		const uint64_t head = pairs < N ? pairs : N;
		if (L) CU_TRY(ctx, cudaMemcpyAsync(g.d_join.ptr, g.d_hist.ptr, sizeof(float) * 2 * L, cudaMemcpyDeviceToDevice, stream));
		CU_TRY(ctx, cudaMemcpyAsync(g.d_join.ptr + 2 * L, d_iq, sizeof(float) * 2 * head, cudaMemcpyDeviceToDevice, stream));
	}
	uint32_t r = 0;
	for (uint64_t q = 0; q < count;) {
		const uint64_t end = q < nj ? nj : count, n = (end - q < g.K - g.done) ? end - q : g.K - g.done;
		const float *src = q < nj ? g.d_join.ptr + 2 * q * H : d_iq + 2 * (q * H - L);
		for (uint64_t q0 = 0; q0 < n;) {
			const uint64_t nq = (g.seg_chunk && n - q0 > g.seg_chunk) ? g.seg_chunk : n - q0;
			uint64_t rows = nq / SP_MIN_SEGS_PER_ROW;
			rows = rows < 1 ? 1 : (rows > g.rows_max ? g.rows_max : rows);
			if ((rc = launch(src + (size_t) q0 * N, g.done + q0, (unsigned) nq, (unsigned) rows, g.rows_used))) return rc;
			if (rows > g.rows_used) g.rows_used = (unsigned) rows;
			q0 += nq;
		}
		g.done += n; q += n;
		if (g.done == g.K) {
			if ((rc = finish(r))) return rc;
			r++; g.done = 0; g.rows_used = 0;
		}
	}
	const float *from = count * H >= L ? d_iq + 2 * (count * H - L) : g.d_join.ptr + 2 * count * H;
	if (keep) CU_TRY(ctx, cudaMemcpyAsync(g.d_hist.ptr, from, sizeof(float) * 2 * keep, cudaMemcpyDeviceToDevice, stream));
	g.open = keep;
	*h_nreports = r;
	return TSDRGPU_OK;
}

// the device buffers of N, once the work that used the old ones on `stream` is done: rows_max rows of partial sums, one CTA per row
// and bundle of the accumulating last pass at its occupancy, and the two-pass plans' scratch for seg_chunk segments
int seg_build(tsdrgpu_ctx_t *ctx, SegStream &g, cudaStream_t stream) {
	const AccShape a = acc_shape(ilog2(g.N));
	{ std::lock_guard<std::mutex> lock(ctx->mu); if (const int rc = pass_attrs(ctx)) return rc; }     // the occupancy below depends on it
	const unsigned ctas = (unsigned) acc_ctas_per_sm(a.log2L, a.threads, a.smem, g.per_seg == 2) * (unsigned) ctx->sm_count;
	const unsigned long long NP = (unsigned long long) g.N * g.per_seg;
	g.rows_max = ctas / a.bundles > 0 ? ctas / a.bundles : 1;
	g.seg_chunk = ilog2(g.N) <= (unsigned) FFT_MAX_LOG2L ? 0u : (unsigned) (SP_SCRATCH_POINTS / NP > 0 ? SP_SCRATCH_POINTS / NP : 1);
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	CU_TRY(ctx, g.d_hist.assign(2 * (size_t) g.N));
	CU_TRY(ctx, g.d_join.assign(4 * (size_t) g.N));
	CU_TRY(ctx, g.d_acc.assign((size_t) g.rows_max * g.planes * g.N));
	if (g.seg_chunk) CU_TRY(ctx, g.d_scratch.assign((size_t) g.seg_chunk * NP));
	return TSDRGPU_OK;
}

// The preamble of both runs: the arguments, the reports the run completes against the output's capacity (`what` names the run in
// the errors), and when stale the buffers of N rebuilt once the work that used the old ones on `stream` is done, `window` putting
// the caller's window in place.
template <class Window>
int seg_begin(tsdrgpu_ctx_t *ctx, const char *what, SegStream &g, cudaStream_t stream, const float *d_iq, uint64_t pairs,
              int discontinuity, const double *d_reports, uint32_t capacity, uint32_t *h_nreports, Window window) {
	char msg[80];
	if (g.N == 0) {
		snprintf(msg, sizeof msg, "%s run before a spec was set", what);
		return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, msg, cudaSuccess, __FILE__, __LINE__);
	}
	ARG_TRY(ctx, h_nreports != NULL && pairs <= (1ull << 40));
	ARG_TRY(ctx, pairs == 0 || (d_iq != NULL && ((uintptr_t) d_iq & 7u) == 0));
	const uint32_t nrep = g.plan(pairs, discontinuity);
	if (nrep > capacity) {
		snprintf(msg, sizeof msg, "%s run: more reports than the output holds", what);
		return tsdrgpu_fail(ctx, TSDRGPU_ECAPACITY, msg, cudaSuccess, __FILE__, __LINE__);
	}
	ARG_TRY(ctx, nrep == 0 || d_reports != NULL);
	if (!g.stale) return TSDRGPU_OK;
	int rc;
	if ((rc = seg_build(ctx, g, stream)) || (rc = window())) return rc;
	g.stale = 0;
	return TSDRGPU_OK;
}

struct tsdrgpu_spectrum {
	tsdrgpu_ctx_t *ctx;
	tsdrgpu_welch_t spec;                         // n == 0: no spec set yet
	uint32_t fs;
	double scale;                                 // 1 / (K (sum w)^2)
	std::vector<float> h_win;                     // the float32 window of spec.n
	SegStream seg;                                // N = spec.n, K
	DeviceBuf<float> d_win;                       // the window
};

extern "C" {

int tsdrgpu_spectrum_create(tsdrgpu_ctx_t *ctx, tsdrgpu_spectrum_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_spectrum *s = new tsdrgpu_spectrum();      // value-initialised; buffers are sized by the first run after a set
	s->ctx = ctx; s->seg.per_seg = 1; s->seg.planes = 1;
	*out = s;
	return TSDRGPU_OK;
}

void tsdrgpu_spectrum_destroy(tsdrgpu_spectrum_t *s) {
	if (!s) return;
	cudaSetDevice(s->ctx->device);
	cudaDeviceSynchronize();
	delete s;
}

int tsdrgpu_spectrum_reset(tsdrgpu_spectrum_t *s) {
	if (!s) return TSDRGPU_EINVAL;
	s->seg.reset();
	return TSDRGPU_OK;
}

int tsdrgpu_spectrum_set(tsdrgpu_spectrum_t *s, const tsdrgpu_welch_t *spec, uint32_t fs) {
	if (!s) return TSDRGPU_EINVAL;
	const uint32_t K = tsdrgpu_spectrum_k(spec, fs);
	if (K == 0) return tsdrgpu_fail(s->ctx, TSDRGPU_EINVAL, "invalid spectrum spec or sample rate (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
	if (spec->n == s->spec.n && spec->rate == s->spec.rate && fs == s->fs) return TSDRGPU_OK;
	if (spec->n != s->spec.n) {
		std::vector<double> w((size_t) spec->n);
		tsdrgpu_spectrum_window(spec->n, w.data());
		s->h_win.resize(w.size());
		double sum = 0.0;
		for (size_t i = 0; i < w.size(); i++) { s->h_win[i] = (float) w[i]; sum += (double) s->h_win[i]; }
		s->scale = 1.0 / (sum * sum);
		s->seg.stale = 1;
	} else s->scale *= (double) s->seg.K;
	s->scale /= (double) K;
	s->spec = *spec; s->fs = fs; s->seg.N = (uint32_t) spec->n; s->seg.K = K;
	return tsdrgpu_spectrum_reset(s);
}

int tsdrgpu_spectrum_plan(const tsdrgpu_spectrum_t *s, uint64_t pairs, int discontinuity, uint32_t *nreports) {
	if (!s || !nreports || s->spec.n == 0) return TSDRGPU_EINVAL;
	*nreports = s->seg.plan(pairs, discontinuity);
	return TSDRGPU_OK;
}

int tsdrgpu_spectrum_run(tsdrgpu_spectrum_t *s, void *stream_, const float *d_iq, uint64_t pairs, int discontinuity,
                         double *d_reports, uint32_t capacity, uint32_t *h_nreports) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	tsdrgpu_ctx_t *ctx = s->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = s->seg.N;
	const int rc = seg_begin(ctx, "spectrum", s->seg, stream, d_iq, pairs, discontinuity, d_reports, capacity, h_nreports, [&]() -> int {
		CU_TRY(ctx, s->d_win.assign(N));
		CU_TRY(ctx, cudaMemcpyAsync(s->d_win.ptr, s->h_win.data(), sizeof(float) * N, cudaMemcpyHostToDevice, stream));
		return TSDRGPU_OK;
	});
	if (rc) return rc;
	auto launch = [&](const float *src, uint64_t, unsigned nq, unsigned rows, unsigned keep) -> int {
		FftOpts o; memset(&o, 0, sizeof o);
		o.scale = 1.0f; o.batch = nq; o.exact = true; o.win = s->d_win.ptr;
		o.pair_in = src; o.pair_bs = (long long) N;
		o.scratch_bs = (long long) N;
		o.acc = s->seg.d_acc.ptr; o.acc_bs = (long long) N; o.acc_rows = rows; o.acc_keep = keep;
		return fft_run(ctx, stream, NULL, s->seg.d_scratch.ptr, ilog2(N), 0, o);
	};
	auto finish = [&](uint32_t r) -> int {
		KL(ctx, "k_spectrum_finish", stream, k_spectrum_finish<<<grid1d(N, ctx->sm_count), 256, 0, stream>>>(
			s->seg.d_acc.ptr, (long long) N, s->seg.rows_used, (unsigned) N, s->scale, d_reports + (size_t) r * N));
		return TSDRGPU_OK;
	};
	return seg_run(ctx, s->seg, stream, d_iq, pairs, discontinuity, launch, finish, h_nreports);
}

}  // extern "C"

// ---- spectral coherence at the line rate (definition in tsdrgpu.h) --------------------------------------------------------------
// Each segment is transformed twice, as a batch of two (x w+ and x w-, the complex window applied on load), and fft_acc2_kernel
// takes both transforms of a segment in one CTA, so the cross term never goes to HBM.  Rows of partial sums as in the spectrum;
// k_coherence_finish adds them in order.
namespace {

// rows 0 .. rows-1 of acc (four planes of n each) added in order, gamma of bin (i + N/2) mod N into value i
__global__ void __launch_bounds__(256) k_coherence_finish(const double *__restrict__ acc, long long acc_bs, unsigned rows, unsigned n,
                                                          double *__restrict__ out) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const unsigned k = (i + n / 2) & (n - 1);
		double cr = 0.0, ci = 0.0, pp = 0.0, pm = 0.0;
		for (unsigned r = 0; r < rows; r++) {
			const double *a = acc + (long long) r * acc_bs + k;
			cr = __dadd_rn(cr, a[0]); ci = __dadd_rn(ci, a[n]); pp = __dadd_rn(pp, a[2 * n]); pm = __dadd_rn(pm, a[3 * n]);
		}
		const double den = __dmul_rn(pp, pm);
		out[i] = den > 0.0 ? __ddiv_rn(__dsqrt_rn(__fma_rn(cr, cr, __dmul_rn(ci, ci))), __dsqrt_rn(den)) : 0.0;
	}
}

}  // namespace

struct tsdrgpu_coherence {
	tsdrgpu_ctx_t *ctx;
	tsdrgpu_coherence_t spec;                     // rate == 0: no spec set yet
	uint32_t fs;
	double alpha;                                 // the last set's; the report in progress uses alpha_rep
	double alpha_rep;                             // the alpha whose window is in d_cwin (0: none yet)
	SegStream seg;                                // planes of partial sums: Re C, Im C, P+, P-
	DeviceBuf<float2> d_cwin;                     // w+ of alpha_rep
	std::vector<float2> h_cwin;
};

extern "C" {

int tsdrgpu_coherence_create(tsdrgpu_ctx_t *ctx, tsdrgpu_coherence_obj_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_coherence *c = new tsdrgpu_coherence();    // value-initialised; buffers are sized by the first run after a set
	c->ctx = ctx; c->seg.per_seg = 2; c->seg.planes = 4;
	c->seg.break_report = true;                        // the time reference of the report is lost with the run
	*out = c;
	return TSDRGPU_OK;
}

void tsdrgpu_coherence_destroy(tsdrgpu_coherence_obj_t *c) {
	if (!c) return;
	cudaSetDevice(c->ctx->device);
	cudaDeviceSynchronize();
	delete c;
}

int tsdrgpu_coherence_reset(tsdrgpu_coherence_obj_t *c) {
	if (!c) return TSDRGPU_EINVAL;
	c->seg.reset();
	return TSDRGPU_OK;
}

int tsdrgpu_coherence_set(tsdrgpu_coherence_obj_t *c, const tsdrgpu_coherence_t *spec, uint32_t fs, double alpha) {
	if (!c) return TSDRGPU_EINVAL;
	const uint32_t N = tsdrgpu_coherence_n(fs, alpha);
	const tsdrgpu_welch_t w = {(int32_t) N, spec ? spec->rate : 0};
	const uint32_t K = N ? tsdrgpu_spectrum_k(&w, fs) : 0;
	if (K == 0) return tsdrgpu_fail(c->ctx, TSDRGPU_EINVAL, "invalid coherence spec, sample rate or line rate (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
	c->alpha = alpha;                             // alone: from the next report on
	if (spec->rate == c->spec.rate && fs == c->fs && N == c->seg.N) return TSDRGPU_OK;
	if (N != c->seg.N) c->seg.stale = 1;
	c->alpha_rep = 0;                             // the window depends on fs: rebuilt at the next report
	c->spec = *spec; c->fs = fs; c->seg.N = N; c->seg.K = K;
	return tsdrgpu_coherence_reset(c);
}

int tsdrgpu_coherence_plan(const tsdrgpu_coherence_obj_t *c, uint64_t pairs, int discontinuity, uint32_t *nreports) {
	if (!c || !nreports || c->spec.rate == 0) return TSDRGPU_EINVAL;
	*nreports = c->seg.plan(pairs, discontinuity);
	return TSDRGPU_OK;
}

int tsdrgpu_coherence_run(tsdrgpu_coherence_obj_t *c, void *stream_, const float *d_iq, uint64_t pairs, int discontinuity,
                          double *d_reports, uint32_t capacity, uint32_t *h_nreports) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, c != NULL);
	tsdrgpu_ctx_t *ctx = c->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned long long N = c->seg.N;
	const int rc = seg_begin(ctx, "coherence", c->seg, stream, d_iq, pairs, discontinuity, d_reports, capacity, h_nreports, [&]() -> int {
		CU_TRY(ctx, c->d_cwin.assign(N));
		c->alpha_rep = 0;                                               // uploaded at the next report's first segment
		return TSDRGPU_OK;
	});
	if (rc) return rc;
	auto launch = [&](const float *src, uint64_t first, unsigned nq, unsigned rows, unsigned keep) -> int {
		if (first == 0 && c->alpha_rep != c->alpha) {                   // alpha is read at the first segment of a report
			std::vector<double> w2(2 * N);
			tsdrgpu_coherence_window((int) N, c->alpha, c->fs, w2.data());
			c->h_cwin.resize(N);
			for (size_t i = 0; i < N; i++) c->h_cwin[i] = make_float2((float) w2[2 * i], (float) w2[2 * i + 1]);
			// pageable source: the copy has taken the host values when it returns
			CU_TRY(ctx, cudaMemcpyAsync(c->d_cwin.ptr, c->h_cwin.data(), sizeof(float2) * N, cudaMemcpyHostToDevice, stream));
			c->alpha_rep = c->alpha;
		}
		FftOpts o; memset(&o, 0, sizeof o);
		o.scale = 1.0f; o.batch = 2 * nq; o.exact = true; o.cwin = c->d_cwin.ptr;
		o.pair_in = src; o.pair_bs = (long long) N;
		o.scratch_bs = (long long) N;
		o.acc = c->seg.d_acc.ptr; o.acc_bs = 4 * (long long) N; o.acc_rows = rows; o.acc_keep = keep;
		o.coh.alpha = c->alpha_rep; o.coh.fs = (double) c->fs; o.coh.seg0 = first; o.coh.hop = N / 2; o.coh.plane = (long long) N;
		return fft_run(ctx, stream, NULL, c->seg.d_scratch.ptr, ilog2(N), 0, o);
	};
	auto finish = [&](uint32_t r) -> int {
		KL(ctx, "k_coherence_finish", stream, k_coherence_finish<<<grid1d(N, ctx->sm_count), 256, 0, stream>>>(
			c->seg.d_acc.ptr, 4 * (long long) N, c->seg.rows_used, (unsigned) N, d_reports + (size_t) r * N));
		return TSDRGPU_OK;
	};
	return seg_run(ctx, c->seg, stream, d_iq, pairs, discontinuity, launch, finish, h_nreports);
}

}  // extern "C"
