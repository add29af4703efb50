// enhance.cu -- the opt-in steps on the frames the frame stage delivers, beyond the reference (definitions in tsdrgpu.h):
// drift-registered averaging (stack.cu), Richardson-Lucy deconvolution along the lines (fs_deblur), non-local means denoising
// (fs_nlm), then contrast-limited adaptive histogram equalisation (fs_clahe_*).  None feeds back into the frame stage.  Built with -fmad=false like the frame stage, so every output bit follows the definitions.
#include "common.cuh"
#include "host_plan.h"

namespace {

// ---------------------------------------------------------------- CLAHE (beyond the reference; the definition is in tsdrgpu.h)
// Per pass of nf frames the histogram buffer holds [frame][tile row][tile column][256] counts, zeroed before fs_clahe_hist;
// fs_clahe_lut overwrites each tile's counts with its LUT (floats) in place, and fs_clahe_map reads the LUTs.
constexpr int CH_BINS = 256;
constexpr int CH_STAGE_BYTES = 96 * 1024;        // fs_clahe_map stages up to three tile rows of LUTs when they fit in this
constexpr size_t CH_PASS_WORDS = (size_t) 1 << 24;   // histogram words per pass (64 MB): frames are processed in passes

__device__ __forceinline__ int ch_bin(float v) { return v <= 0.0f ? 0 : (v >= 1.0f ? CH_BINS - 1 : (int) __fmul_rn(v, 256.0f)); }
// tile bound x_j = floor(j W / T); the tile holding pixel x is the last j with x_j <= x
__device__ __forceinline__ int ch_bound(int j, int W, int T) { return (int) (((long long) j * W) / T); }
__device__ __forceinline__ int ch_tile_of(int x, int W, int T) { return (int) (((long long) (x + 1) * T - 1) / W); }

// interpolation along one axis for pixel x: the two tiles whose centres bracket it and the weight of the second.
// s_j = x_j + x_{j+1} and c = 2x + 1 are twice the centres, so everything is an integer until the one division.
__device__ __forceinline__ void ch_axis(int x, int W, int T, unsigned char *j0, unsigned char *j1, float *wt) {
	const int c = 2 * x + 1;
	const int s_first = ch_bound(0, W, T) + ch_bound(1, W, T), s_last = ch_bound(T - 1, W, T) + ch_bound(T, W, T);
	if (c <= s_first) { *j0 = *j1 = 0; *wt = 0.0f; return; }
	if (c >= s_last) { *j0 = *j1 = (unsigned char) (T - 1); *wt = 0.0f; return; }
	const int t = ch_tile_of(x, W, T);
	const int j = (ch_bound(t, W, T) + ch_bound(t + 1, W, T) <= c) ? t : t - 1;     // s_{t+1} > c and s_{t-1} < c always
	const int a = ch_bound(j, W, T) + ch_bound(j + 1, W, T), b = ch_bound(j + 1, W, T) + ch_bound(j + 2, W, T);
	*j0 = (unsigned char) j; *j1 = (unsigned char) (j + 1);
	*wt = __fdiv_rn((float) (c - a), (float) (b - a));
}

// histograms: grid (TY * parts, frames).  CTA (i * parts + p, f) counts part p of tile row i of frame f into TX shared
// histograms, and adds its non-zero counts to the pass buffer once at the end.  Dynamic shared memory: TX * 1 KB + W bytes.
__global__ void __launch_bounds__(256) fs_clahe_hist(const float *__restrict__ in, int W, int H, int TX, int TY, int parts,
                                                     unsigned *__restrict__ hist) {
	extern __shared__ __align__(16) unsigned ch_smem[];
	unsigned *s_h = ch_smem;
	unsigned char *s_col = reinterpret_cast<unsigned char *>(s_h + TX * CH_BINS);
	const int f = blockIdx.y, i = blockIdx.x / parts, p = blockIdx.x % parts;
	const int y0 = ch_bound(i, H, TY), rows = ch_bound(i + 1, H, TY) - y0;
	const int r0 = y0 + (int) ((long long) p * rows / parts), r1 = y0 + (int) ((long long) (p + 1) * rows / parts);
	for (int k = threadIdx.x; k < TX * CH_BINS; k += blockDim.x) s_h[k] = 0;
	for (int x = threadIdx.x; x < W; x += blockDim.x) s_col[x] = (unsigned char) ch_tile_of(x, W, TX);
	__syncthreads();
	const float *src = in + (size_t) f * W * H + (size_t) r0 * W;
	const F4Split band(src, (size_t) (r1 - r0) * W);
	const unsigned uw = (unsigned) W;
	const int lane = threadIdx.x & 31;
	if (threadIdx.x < band.head) { const float v = src[threadIdx.x]; if (px_valid(v)) atomicAdd(&s_h[s_col[threadIdx.x % uw] * CH_BINS + ch_bin(v)], 1u); }
	if (threadIdx.x < band.n - band.tail0) {
		const unsigned q = (unsigned) (band.tail0 + threadIdx.x);
		const float v = src[q];
		if (px_valid(v)) atomicAdd(&s_h[s_col[q % uw] * CH_BINS + ch_bin(v)], 1u);
	}
	auto key_of = [&](float v, int x) { return px_valid(v) ? s_col[x] * CH_BINS + ch_bin(v) : -1; };
	const float4 *src4 = reinterpret_cast<const float4 *>(src + band.head);
	for (size_t base = threadIdx.x & ~31u; base < band.nbody; base += blockDim.x) {      // warp-uniform trip count
		const size_t k = base + lane;
		int key[4] = {-1, -1, -1, -1};
		if (k < band.nbody) {
			const float4 v = __ldg(src4 + k);
			int x = (int) ((unsigned) (band.head + 4 * k) % uw);
			key[0] = key_of(v.x, x); x = (x + 1 == W) ? 0 : x + 1;
			key[1] = key_of(v.y, x); x = (x + 1 == W) ? 0 : x + 1;
			key[2] = key_of(v.z, x); x = (x + 1 == W) ? 0 : x + 1;
			key[3] = key_of(v.w, x);
		}
		// a warp whose valid pixels all share one (tile, bin), as in blanking and flat areas, adds them with one atomic;
		// otherwise each lane adds one atomic per run of equal keys among its four pixels
		const int k0 = __shfl_sync(0xffffffffu, key[0], 0);
		unsigned mine = 0;
		bool only = true;
#pragma unroll
		for (int p = 0; p < 4; p++) { if (key[p] == k0) mine++; else if (key[p] >= 0) only = false; }
		if (__all_sync(0xffffffffu, only) && k0 >= 0) {
			const unsigned total = __reduce_add_sync(0xffffffffu, mine);
			if (lane == 0) atomicAdd(&s_h[k0], total);
		} else {
			int run = key[0];
			unsigned cnt = 1;
#pragma unroll
			for (int p = 1; p < 4; p++) {
				if (key[p] == run) cnt++;
				else { if (run >= 0) atomicAdd(&s_h[run], cnt); run = key[p]; cnt = 1; }
			}
			if (run >= 0) atomicAdd(&s_h[run], cnt);
		}
	}
	__syncthreads();
	unsigned *g = hist + ((size_t) f * TY + i) * TX * CH_BINS;
	for (int k = threadIdx.x; k < TX * CH_BINS; k += blockDim.x) if (s_h[k]) atomicAdd(g + k, s_h[k]);
}

__device__ __forceinline__ unsigned ch_block_sum(unsigned v, unsigned *s_w) {
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	__syncthreads();                                     // s_w is free again
	if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
	__syncthreads();
	unsigned t = 0;
	for (int k = 0; k < CH_BINS / 32; k++) t += s_w[k];
	return t;
}

// LUTs: one 256-thread CTA per (tile, frame), thread b owns bin b.  Clip at L, spread the excess in OpenCV's integer scheme
// (closed form of its residual loop), inclusive scan, one IEEE division per bin.  The LUT overwrites the counts.
__global__ void __launch_bounds__(CH_BINS) fs_clahe_lut(unsigned *hist, int clip_centi) {
	__shared__ unsigned s_w[CH_BINS / 32];
	unsigned *h = hist + ((size_t) blockIdx.y * gridDim.x + blockIdx.x) * CH_BINS;
	const unsigned b = threadIdx.x;
	unsigned c = h[b];
	const unsigned nt = ch_block_sum(c, s_w);
	float lut;
	if (nt == 0) lut = __fdiv_rn((float) b, 255.0f);
	else {                                               // block-uniform branch
		const unsigned long long l = (unsigned long long) clip_centi * nt / 25600ull;
		const unsigned L = l > 1ull ? (unsigned) l : 1u;
		const unsigned excess = ch_block_sum(c > L ? c - L : 0u, s_w);
		c = (c < L ? c : L) + excess / CH_BINS;
		const unsigned r = excess % CH_BINS;
		if (r) { const unsigned step = (CH_BINS / r > 1u) ? CH_BINS / r : 1u; if (b % step == 0 && b / step < r) c++; }
		unsigned s = c;
		const int lane = b & 31, wid = b >> 5;
		for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
		__syncthreads();
		if (lane == 31) s_w[wid] = s;
		__syncthreads();
		for (int k = 0; k < wid; k++) s += s_w[k];
		lut = __fdiv_rn((float) s, (float) nt);
	}
	h[b] = __float_as_uint(lut);
}

// mapping: grid (bands, frames), band rows [b * bh, min(H, (b + 1) * bh)).  Per-column and per-row (tile pair, weight) tables
// in shared memory; the LUTs of the tile rows the band touches are staged in shared memory when there are at most stage_rows
// of them, otherwise gathered from global memory (L1).  VEC: in and out share their 16-byte phase, so the body is float4s.
template <bool VEC>
__global__ void __launch_bounds__(256) fs_clahe_map(const float *in, float *out, int W, int H, int TX, int TY, int bh,
                                                    int stage_rows, const float *__restrict__ luts) {
	extern __shared__ __align__(16) float ch_fsmem[];
	const int f = blockIdx.y, r0 = blockIdx.x * bh, r1 = (r0 + bh < H) ? r0 + bh : H;
	float *s_lut = ch_fsmem, *s_cw = s_lut + (size_t) stage_rows * TX * CH_BINS, *s_rw = s_cw + W;
	uchar2 *s_cj = reinterpret_cast<uchar2 *>(s_rw + bh), *s_rj = s_cj + W;
	for (int x = threadIdx.x; x < W; x += blockDim.x) { uchar2 j; ch_axis(x, W, TX, &j.x, &j.y, &s_cw[x]); s_cj[x] = j; }
	for (int y = threadIdx.x; y < r1 - r0; y += blockDim.x) { uchar2 j; ch_axis(r0 + y, H, TY, &j.x, &j.y, &s_rw[y]); s_rj[y] = j; }
	__syncthreads();
	const int i_lo = s_rj[0].x, i_hi = s_rj[r1 - r0 - 1].y, tile_row = TX * CH_BINS;
	const float *g = luts + (size_t) f * TY * tile_row;
	const float *L = g;
	int base_row = 0;
	if (i_hi - i_lo + 1 <= stage_rows) {                 // block-uniform
		const float4 *s4 = reinterpret_cast<const float4 *>(g + (size_t) i_lo * tile_row);
		float4 *d4 = reinterpret_cast<float4 *>(s_lut);
		for (int k = threadIdx.x; k < (i_hi - i_lo + 1) * tile_row / 4; k += blockDim.x) d4[k] = __ldg(s4 + k);
		__syncthreads();
		L = s_lut; base_row = i_lo;
	}
	auto map = [&](float v, int x, int yy) -> float {
		if (!px_valid(v)) return v;
		const int bin = ch_bin(v);
		const uchar2 cj = s_cj[x], rj = s_rj[yy];
		const float wx = s_cw[x], wy = s_rw[yy];
		const float *l0 = L + (rj.x - base_row) * tile_row + bin, *l1 = L + (rj.y - base_row) * tile_row + bin;
		const float a = l0[cj.x * CH_BINS], b = l0[cj.y * CH_BINS], c = l1[cj.x * CH_BINS], d = l1[cj.y * CH_BINS];
		const float top = __fadd_rn(a, __fmul_rn(wx, __fsub_rn(b, a)));
		const float bot = __fadd_rn(c, __fmul_rn(wx, __fsub_rn(d, c)));
		return __fadd_rn(top, __fmul_rn(wy, __fsub_rn(bot, top)));
	};
	const size_t off = (size_t) f * W * H + (size_t) r0 * W;
	const float *src = in + off;
	float *dst = out + off;
	const unsigned uw = (unsigned) W, count = (unsigned) ((r1 - r0) * W);
	if (!VEC) {
		for (unsigned q = threadIdx.x; q < count; q += blockDim.x) dst[q] = map(src[q], (int) (q % uw), (int) (q / uw));
		return;
	}
	const F4Split band(src, count);
	if (threadIdx.x < band.head) { const unsigned q = threadIdx.x; dst[q] = map(src[q], (int) (q % uw), (int) (q / uw)); }
	if (threadIdx.x < band.n - band.tail0) {
		const unsigned q = (unsigned) (band.tail0 + threadIdx.x);
		dst[q] = map(src[q], (int) (q % uw), (int) (q / uw));
	}
	const float4 *src4 = reinterpret_cast<const float4 *>(src + band.head);
	float4 *dst4 = reinterpret_cast<float4 *>(dst + band.head);
	auto map4 = [&](float4 v, size_t k) {
		const unsigned q = (unsigned) (band.head + 4 * k);
		int x = (int) (q % uw), y = (int) (q / uw);
		v.x = map(v.x, x, y); if (++x == W) { x = 0; y++; }
		v.y = map(v.y, x, y); if (++x == W) { x = 0; y++; }
		v.z = map(v.z, x, y); if (++x == W) { x = 0; y++; }
		v.w = map(v.w, x, y);
		dst4[k] = v;
	};
	// two float4s per thread and iteration, both loaded before either is stored (in place, the stores could alias later loads)
	for (size_t k = threadIdx.x; k < band.nbody; k += 2 * blockDim.x) {
		const size_t k2 = k + blockDim.x;
		const float4 v = src4[k], u = (k2 < band.nbody) ? src4[k2] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		map4(v, k);
		if (k2 < band.nbody) map4(u, k2);
	}
}

// ---------------------------------------------------------------- non-local means (beyond the reference; the definition is in tsdrgpu.h)
// A CTA of NL_TW x NL_BY threads owns an output tile of NL_TW columns by NL_BY K rows of one frame (frames on grid.y).  Shared
// memory holds the tile's guide g_c with a fixed halo of R_max + P_max and its (masked value, mask) pairs with a fixed halo of
// R_max, so the row pitches are constants and every shared load is a register base plus an immediate; only the rows and
// columns the actual R and P reach are filled.  A thread owns one column and K consecutive rows.  The guide values of its
// centre patches (K + 2P rows by 2P + 1 columns) stay in registers for all offsets.  Along dx the neighbours' guide values
// slide through a rotating register window (the dx loop is unrolled by 2P + 1, so the slot of every column is a constant),
// which takes one new column, K + 2P loads, per offset.  Each offset then costs per pixel one LDS.64 of (v_n, m) and the
// arithmetic of the definition; the mask multiplies the weight (w m is w or +0, and adding +0 leaves either accumulator as
// it was, since neither can be -0), so no branch or select depends on the neighbour.
constexpr int NL_TW = 64, NL_BY = 4;
constexpr int NL_GH = TSDRGPU_NLM_MAX_R + TSDRGPU_NLM_MAX_P, NL_VH = TSDRGPU_NLM_MAX_R;
constexpr int NL_GW = NL_TW + 2 * NL_GH, NL_VW = NL_TW + 2 * NL_VH;       // row pitches of the guide and value planes
template <int K> constexpr size_t nl_smem_bytes() {
	return sizeof(float) * NL_GW * (NL_BY * K + 2 * NL_GH) + sizeof(float2) * NL_VW * (NL_BY * K + 2 * NL_VH);
}

template <int P, int K>
__global__ void __launch_bounds__(NL_TW * NL_BY) fs_nlm(const float *__restrict__ in, float *__restrict__ out, int W, int H,
                                                       int tiles_x, int R, float inv) {
	constexpr int TH = NL_BY * K, WN = 2 * P + 1, ROWS = K + 2 * P;
	extern __shared__ __align__(16) float nl_smem[];
	float *sG = nl_smem;
	float2 *sV = reinterpret_cast<float2 *>(nl_smem + NL_GW * (TH + 2 * NL_GH));
	const int x0 = (int) (blockIdx.x % (unsigned) tiles_x) * NL_TW, y0 = (int) (blockIdx.x / (unsigned) tiles_x) * TH;
	const int tx = threadIdx.x, ty = threadIdx.y;
	const float *src = in + (size_t) blockIdx.y * W * H;
	const int hg = R + P;
	for (int r = NL_GH - hg + ty; r < NL_GH + TH + hg; r += NL_BY) {
		const int yy = min(max(y0 - NL_GH + r, 0), H - 1);
		const float *row = src + (size_t) yy * W;
		for (int c = NL_GH - hg + tx; c < NL_GH + NL_TW + hg; c += NL_TW) {
			const float v = __ldg(row + min(max(x0 - NL_GH + c, 0), W - 1));
			sG[r * NL_GW + c] = px_valid(v) ? fminf(fmaxf(v, 0.0f), 1.0f) : 0.0f;
		}
	}
	for (int r = NL_VH - R + ty; r < NL_VH + TH + R; r += NL_BY) {
		const int yy = y0 - NL_VH + r;
		for (int c = NL_VH - R + tx; c < NL_VH + NL_TW + R; c += NL_TW) {
			const int xx = x0 - NL_VH + c;
			float2 q = make_float2(0.0f, 0.0f);
			if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
				const float v = __ldg(src + (size_t) yy * W + xx);
				if (px_valid(v)) q = make_float2(v, 1.0f);
			}
			sV[r * NL_VW + c] = q;
		}
	}
	__syncthreads();
	const int x = x0 + tx, yt = y0 + ty * K;
	if (x >= W || yt >= H) return;
	const float *cg = sG + (NL_GH + ty * K - P) * NL_GW + NL_GH + tx - P;     // top-left of the thread's centre patches
	float cw[ROWS][WN];
#pragma unroll
	for (int j = 0; j < ROWS; j++)
#pragma unroll
		for (int c = 0; c < WN; c++) cw[j][c] = cg[j * NL_GW + c];
	float aw[K], av[K];
#pragma unroll
	for (int i = 0; i < K; i++) { aw[i] = 0.0f; av[i] = 0.0f; }
	for (int dy = -R; dy <= R; dy++) {
		const float *nb = cg + dy * NL_GW - R;                          // neighbour window of dx = -R, column 0
		const float2 *vb = sV + (NL_VH + ty * K + dy) * NL_VW + NL_VH + tx - R;
		float nw[ROWS][WN];
#pragma unroll
		for (int j = 0; j < ROWS; j++)
#pragma unroll
			for (int c = 0; c < WN - 1; c++) nw[j][c] = nb[j * NL_GW + c];
		for (int kb = 0; kb <= 2 * R; kb += WN) {
#pragma unroll
			for (int r = 0; r < WN; r++) {
				const int k = kb + r;                                   // dx = k - R
				if (k > 2 * R) break;
#pragma unroll
				for (int j = 0; j < ROWS; j++) nw[j][(r + WN - 1) % WN] = nb[j * NL_GW + k + WN - 1];
				float s[ROWS];
#pragma unroll
				for (int j = 0; j < ROWS; j++) {
#pragma unroll
					for (int c = 0; c < WN; c++) {
						const float d = __fsub_rn(cw[j][c], nw[j][(r + c) % WN]);
						const float e = __fmul_rn(d, d);
						s[j] = (c == 0) ? e : __fadd_rn(s[j], e);
					}
				}
#pragma unroll
				for (int i = 0; i < K; i++) {
					float d = s[i];
#pragma unroll
					for (int p = 1; p < WN; p++) d = __fadd_rn(d, s[i + p]);
					const float u = __fsub_rn(1.0f, fminf(__fmul_rn(d, inv), 1.0f));
					const float2 q = vb[i * NL_VW + k];
					const float wm = __fmul_rn(__fmul_rn(u, u), q.y);
					aw[i] = __fadd_rn(aw[i], wm);
					av[i] = __fadd_rn(av[i], __fmul_rn(wm, q.x));
				}
			}
		}
	}
#pragma unroll
	for (int i = 0; i < K; i++) {
		if (yt + i >= H) break;
		const size_t o = (size_t) (yt + i) * W + x;
		const float v = __ldg(src + o);
		out[(size_t) blockIdx.y * W * H + o] = px_valid(v) ? __fdiv_rn(av[i], aw[i]) : v;
	}
}

// ---------------------------------------------------------------- Richardson-Lucy deconvolution along the lines (beyond the reference; the definition is in tsdrgpu.h)
// A CTA holds up to DB_SPAN pixels of content in shared memory: either several whole lines (lines of at most DB_SPAN pixels,
// stored R apart so the zeros between them stand for "outside the line"), or one segment of a longer line with a halo of 2 R I
// pixels on each side, clamped to the line.  It runs all I iterations there and writes the lines or the segment once.  Four
// planes: d, u, q and rn, with rn = 0 where m = 0, so every plane is 0 wherever m is (u_0 = d = 0 there, q = d / max(b, eps) = 0,
// u (B(q) rn) = 0): the masked correlation is then a plain one over zeros, and the gaps and pads need no test.  Each thread
// computes four adjacent outputs from one float4-aligned register window of the plane it correlates.  Where a segment is cut,
// the plane is correct one R further in after each correlation, so each pass computes only the range the output still needs.
constexpr int DB_SPAN = 6144;                         // content pixels per CTA: 4 planes of 24 KB, two CTAs per SM
constexpr int DB_THREADS = 256;
struct DbTaps { float k[2 * TSDRGPU_DEBLUR_MAX_R + 1]; };

// plane pitch in floats: pads of P = R rounded up to 4 (zeros) around DB_SPAN of content
__host__ __device__ constexpr int db_pad(int R) { return (R + 3) & ~3; }
__host__ __device__ constexpr int db_pitch(int R) { return db_pad(R) + DB_SPAN + db_pad(R) + 4; }

// sum_j k_j a(x + t + j), j from -R to R left to right, for t = 0..3; `a` points at content position x (16-byte aligned)
template <int R, int P>
__device__ __forceinline__ float4 db_corr4(const float *a, const DbTaps &tp) {
	constexpr int NW = 2 * P / 4 + 1;
	float v[4 * NW];
	const float4 *a4 = reinterpret_cast<const float4 *>(a - P);
#pragma unroll
	for (int i = 0; i < NW; i++) { const float4 f = a4[i]; v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w; }
	float s[4];
#pragma unroll
	for (int t = 0; t < 4; t++) {
		s[t] = __fmul_rn(tp.k[0], v[P + t - R]);
#pragma unroll
		for (int j = 1; j <= 2 * R; j++) s[t] = __fadd_rn(s[t], __fmul_rn(tp.k[j], v[P + t - R + j]));
	}
	return make_float4(s[0], s[1], s[2], s[3]);
}

// grid.x = CTAs.  Whole lines (seg == 0): CTA c takes lines [c L, min((c + 1) L, lines)) of w pixels, stored at content
// position l (w + R).  Segments (seg > 0): CTA c takes segment c % segs of line c / segs, [s0, s0 + seg), loaded with its halo.
template <int R>
__global__ void __launch_bounds__(DB_THREADS, 2) fs_deblur(const float *__restrict__ in, float *__restrict__ out, int w,
                                                          long long lines, int L, int seg, int segs, int iters, DbTaps tp) {
	constexpr int P = db_pad(R), PITCH = db_pitch(R);
	extern __shared__ __align__(16) float db_smem[];
	float *sd = db_smem, *su = sd + PITCH, *sq = su + PITCH, *srn = sq + PITCH;
	long long g0;                                        // first global pixel of the content
	int span, cutl = 0, cutr = 0, nl = 1, s_out0 = 0, n_out;
	if (seg == 0) {
		const long long l0 = (long long) blockIdx.x * L;
		nl = (int) ((lines - l0 < L) ? lines - l0 : L);
		g0 = l0 * w;
		span = nl * (w + R) - R;
		n_out = nl * w;
	} else {
		const long long line = blockIdx.x / (unsigned) segs;
		const int s0 = (int) (blockIdx.x % (unsigned) segs) * seg, s1 = min(s0 + seg, w), halo = 2 * R * iters;
		const int a = max(s0 - halo, 0), b = min(s1 + halo, w);
		cutl = a > 0; cutr = b < w;
		g0 = line * w + a;
		span = b - a;
		s_out0 = s0 - a;
		n_out = s1 - s0;
	}
	const int span4 = (span + 3) & ~3;
	const float *src = in + g0;
	// load: d, u = d, m into sq (B(m) gives rn), zeros in the pads and gaps
	for (int p = threadIdx.x; p < PITCH; p += DB_THREADS) {
		const int x = p - P;
		float v = 0.0f, mv = 0.0f;
		if (x >= 0 && x < span) {
			const int l = x / (w + R), c = x - l * (w + R);
			if (c < w) {
				const float f = __ldg(src + (long long) l * w + c);
				if (px_valid(f)) { mv = 1.0f; v = f > 0.0f ? fminf(f, 1.0f) : 0.0f; }
			}
		}
		sd[p] = v; su[p] = v; sq[p] = mv; srn[p] = 0.0f;
	}
	__syncthreads();
	for (int g = threadIdx.x; g < span4 / 4; g += DB_THREADS) {
		const int x = 4 * g;
		const float4 b = db_corr4<R, P>(sq + P + x, tp), m = *reinterpret_cast<const float4 *>(sq + P + x);
		float4 r;
		r.x = m.x != 0.0f ? __fdiv_rn(1.0f, b.x) : 0.0f;
		r.y = m.y != 0.0f ? __fdiv_rn(1.0f, b.y) : 0.0f;
		r.z = m.z != 0.0f ? __fdiv_rn(1.0f, b.z) : 0.0f;
		r.w = m.w != 0.0f ? __fdiv_rn(1.0f, b.w) : 0.0f;
		*reinterpret_cast<float4 *>(srn + P + x) = r;
	}
	__syncthreads();
	const float eps = TSDRGPU_DEBLUR_EPS;
	for (int it = 0, k = 1; it < iters; it++, k += 2) {
		// pass 1: q = d / max(B(u) rn, eps), on the range correct after k correlations
		int lo = cutl ? (k * R) & ~3 : 0, hi = cutr ? min((span - k * R + 3) & ~3, span4) : span4;
		for (int g = lo / 4 + threadIdx.x; g < hi / 4; g += DB_THREADS) {
			const int x = 4 * g;
			const float4 b = db_corr4<R, P>(su + P + x, tp);
			const float4 rn = *reinterpret_cast<const float4 *>(srn + P + x), d = *reinterpret_cast<const float4 *>(sd + P + x);
			float4 q;
			q.x = __fdiv_rn(d.x, fmaxf(__fmul_rn(b.x, rn.x), eps));
			q.y = __fdiv_rn(d.y, fmaxf(__fmul_rn(b.y, rn.y), eps));
			q.z = __fdiv_rn(d.z, fmaxf(__fmul_rn(b.z, rn.z), eps));
			q.w = __fdiv_rn(d.w, fmaxf(__fmul_rn(b.w, rn.w), eps));
			*reinterpret_cast<float4 *>(sq + P + x) = q;
		}
		__syncthreads();
		// pass 2: u = u (B(q) rn), in place (each output reads only its own u)
		lo = cutl ? ((k + 1) * R) & ~3 : 0; hi = cutr ? min((span - (k + 1) * R + 3) & ~3, span4) : span4;
		for (int g = lo / 4 + threadIdx.x; g < hi / 4; g += DB_THREADS) {
			const int x = 4 * g;
			const float4 c = db_corr4<R, P>(sq + P + x, tp);
			const float4 rn = *reinterpret_cast<const float4 *>(srn + P + x);
			float4 u = *reinterpret_cast<const float4 *>(su + P + x);
			u.x = __fmul_rn(u.x, __fmul_rn(c.x, rn.x));
			u.y = __fmul_rn(u.y, __fmul_rn(c.y, rn.y));
			u.z = __fmul_rn(u.z, __fmul_rn(c.z, rn.z));
			u.w = __fmul_rn(u.w, __fmul_rn(c.w, rn.w));
			*reinterpret_cast<float4 *>(su + P + x) = u;
		}
		__syncthreads();
	}
	// output: the lines or the segment, at any 4-byte phase
	const float *osrc = src + s_out0;
	float *dst = out + g0 + s_out0;
	for (int e = threadIdx.x; e < n_out; e += DB_THREADS) {
		const int l = e / w, c = e - l * w;
		const float v = __ldg(osrc + e);
		dst[e] = px_valid(v) ? fminf(su[P + s_out0 + l * (w + R) + c], 1.0f) : v;
	}
}

}  // namespace

// deblur of nframes frames of w x h, in -> out (no overlap), on `stream`
static int fs_deblur_batch(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h,
                           int sigma_centi, int iters) {
	DbTaps tp = {};
	int R = 0;
	if (tsdrgpu_deblur_taps(sigma_centi, tp.k, &R) != TSDRGPU_OK) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "deblur sigma", cudaSuccess, __FILE__, __LINE__);
	const long long lines = (long long) nframes * h;
	int L = 0, seg = 0, segs = 0;
	long long ctas;
	if (w <= DB_SPAN) {                                  // whole lines, R apart
		L = (DB_SPAN + R) / (w + R);
		ctas = (lines + L - 1) / L;
	} else {                                             // segments with a halo of 2 R I on each side
		seg = DB_SPAN - 4 * R * iters;
		segs = (w + seg - 1) / seg;
		ctas = lines * segs;
	}
	ARG_TRY(ctx, ctas <= 0x7fffffffLL);
	using K = void (*)(const float *, float *, int, long long, int, int, int, int, DbTaps);
	static const K kernels[TSDRGPU_DEBLUR_MAX_R] = {fs_deblur<1>, fs_deblur<2>, fs_deblur<3>, fs_deblur<4>, fs_deblur<5>, fs_deblur<6>,
	                                                fs_deblur<7>, fs_deblur<8>, fs_deblur<9>, fs_deblur<10>, fs_deblur<11>, fs_deblur<12>};
	const K kern = kernels[R - 1];
	const size_t smem = sizeof(float) * 4 * (size_t) db_pitch(R);
	CU_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	KL(ctx, "fs_deblur", stream, kern<<<(unsigned) ctas, DB_THREADS, smem, stream>>>(in, out, w, lines, L, seg, segs, iters, tp));
	return TSDRGPU_OK;
}

// CLAHE: effective tile grid, frames per pass and the words one pass of the histogram buffer needs
struct ChGeom { int tx, ty, fpp; size_t words; };
static ChGeom ch_geom(const EnhanceState *st, int nframes, int w, int h) {
	ChGeom g;
	g.tx = st->tx < w ? st->tx : w; g.ty = st->ty < h ? st->ty : h;
	const size_t per_frame = (size_t) g.tx * g.ty * CH_BINS;
	size_t fpp = CH_PASS_WORDS / per_frame;
	if (fpp > (size_t) nframes) fpp = (size_t) nframes;
	if (fpp > 65535) fpp = 65535;
	g.fpp = fpp ? (int) fpp : 1;
	g.words = (size_t) g.fpp * per_frame;
	return g;
}

template <int P, int K>
static int nl_launch(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h, int r,
                     float inv) {
	const int tiles_x = (w + NL_TW - 1) / NL_TW, tiles_y = (h + NL_BY * K - 1) / (NL_BY * K);
	const size_t smem = nl_smem_bytes<K>(), n = (size_t) w * h;
	CU_TRY(ctx, cudaFuncSetAttribute(fs_nlm<P, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem));
	for (int f0 = 0; f0 < nframes; f0 += 65535) {
		const int nf = (nframes - f0 < 65535) ? nframes - f0 : 65535;
		KL(ctx, "fs_nlm", stream, (fs_nlm<P, K><<<dim3((unsigned) (tiles_x * tiles_y), (unsigned) nf), dim3(NL_TW, NL_BY), smem, stream>>>(
			in + f0 * n, out + f0 * n, w, h, tiles_x, r, inv)));
	}
	return TSDRGPU_OK;
}

// non-local means of nframes frames of w x h, in -> out (no overlap), on `stream`
static int fs_nlm_batch(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h, int h_milli,
                        int r, int p) {
	const float inv = (float) (1e6 / (4.0 * (double) h_milli * (double) h_milli * (double) ((2 * p + 1) * (2 * p + 1))));
	if (p == 1) return nl_launch<1, 8>(ctx, stream, in, out, nframes, w, h, r, inv);
	if (p == 2) return nl_launch<2, 6>(ctx, stream, in, out, nframes, w, h, r, inv);
	return nl_launch<3, 4>(ctx, stream, in, out, nframes, w, h, r, inv);
}

// CLAHE of nframes frames of w x h, in -> out (in == out allowed), on `stream`; per pass: zero, histograms, LUTs, mapping
static int fs_clahe_batch(tsdrgpu_ctx_t *ctx, const EnhanceState *st, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h) {
	const ChGeom g = ch_geom(st, nframes, w, h);
	const size_t n = (size_t) w * h;
	const int target = ctx->sm_count * 4;                // histogram CTAs per launch: about four per SM over the pass
	const size_t hist_smem = sizeof(unsigned) * g.tx * CH_BINS + (size_t) ((w + 3) & ~3);
	const int stage_rows = (3 * g.tx * CH_BINS * (int) sizeof(float) <= CH_STAGE_BYTES) ? 3 : 0;
	const bool vec = ((reinterpret_cast<unsigned long long>(in) ^ reinterpret_cast<unsigned long long>(out)) & 15ull) == 0;
	CU_TRY(ctx, cudaFuncSetAttribute(fs_clahe_hist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) hist_smem));
	for (int f0 = 0; f0 < nframes; f0 += g.fpp) {
		const int nf = (nframes - f0 < g.fpp) ? nframes - f0 : g.fpp;
		CU_TRY(ctx, cudaMemsetAsync(st->d_clahe.ptr, 0, sizeof(unsigned) * nf * g.tx * g.ty * CH_BINS, stream));
		int parts = (target + nf * g.ty - 1) / (nf * g.ty);
		if (parts > h / g.ty) parts = h / g.ty;          // every part keeps at least one row
		if (parts < 1) parts = 1;
		KL(ctx, "fs_clahe_hist", stream, fs_clahe_hist<<<dim3((unsigned) (g.ty * parts), nf), 256, hist_smem, stream>>>(in + f0 * n, w, h, g.tx, g.ty, parts, st->d_clahe.ptr));
		KL(ctx, "fs_clahe_lut", stream, fs_clahe_lut<<<dim3((unsigned) (g.tx * g.ty), nf), CH_BINS, 0, stream>>>(st->d_clahe.ptr, st->clip_centi));
		int bands = (2 * target + nf - 1) / nf;          // mapping CTAs: about eight per SM
		if (bands > h) bands = h;
		const int bh = (h + bands - 1) / bands;
		bands = (h + bh - 1) / bh;
		const size_t map_smem = sizeof(float) * ((size_t) stage_rows * g.tx * CH_BINS + w + bh) + sizeof(uchar2) * ((size_t) w + bh);
		const float *luts = reinterpret_cast<const float *>(st->d_clahe.ptr);
		const auto map = vec ? fs_clahe_map<true> : fs_clahe_map<false>;
		CU_TRY(ctx, cudaFuncSetAttribute(map, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) map_smem));
		KL(ctx, "fs_clahe_map", stream, map<<<dim3((unsigned) bands, nf), 256, map_smem, stream>>>(in + f0 * n, out + f0 * n, w, h, g.tx, g.ty, bh, stage_rows, luts));
	}
	return TSDRGPU_OK;
}

// the buffers the enabled steps need, each grown to exactly its size when short; nothing may be in flight on them
int enhance_reserve(tsdrgpu_ctx_t *ctx, EnhanceState *st, int nframes, int w, int h) {
	const size_t nlm = (size_t) nframes * w * h;
	if (st->stack.mode != TSDRGPU_STACK_OFF) {
		const int rc = stack_reserve(ctx, &st->stack, nframes, w, h);
		if (rc) return rc;
		if (st->d_stack.cap < nlm) { CU_TRY(ctx, cudaDeviceSynchronize()); CU_TRY(ctx, st->d_stack.assign(nlm)); }
	}
	if (st->deblur == TSDRGPU_DEBLUR_RL && st->d_deblur.cap < nlm) { CU_TRY(ctx, cudaDeviceSynchronize()); CU_TRY(ctx, st->d_deblur.assign(nlm)); }
	if (st->denoise == TSDRGPU_DENOISE_NLM && st->d_nlm.cap < nlm) { CU_TRY(ctx, cudaDeviceSynchronize()); CU_TRY(ctx, st->d_nlm.assign(nlm)); }
	if (st->contrast != TSDRGPU_CONTRAST_CLAHE) return TSDRGPU_OK;
	const size_t words = ch_geom(st, nframes, w, h).words;
	if (st->d_clahe.cap < words) { CU_TRY(ctx, cudaDeviceSynchronize()); CU_TRY(ctx, st->d_clahe.assign(words)); }
	return TSDRGPU_OK;
}

// The stack, deblur, NLM, then CLAHE, in place on nframes frames of w x h, on `stream`.  None of the first three can run in place:
// each writes its own buffer (d_stack, d_deblur, d_nlm) when it reads the frames themselves, and the frames when it reads a buffer,
// and CLAHE or one copy brings the frames back.  Only `stream` ever touches these buffers and the stack's state: the frame stage passes the stream its output becomes
// valid on, and in overlap mode its main stream is already filling d_t1 and the other phase's T2 with the next batch, so neither
// can be borrowed.
int enhance_run(tsdrgpu_ctx_t *ctx, EnhanceState *st, cudaStream_t stream, float *d_frames, int nframes, int w, int h) {
	const bool stack = st->stack.mode != TSDRGPU_STACK_OFF;
	const bool nlm = st->denoise == TSDRGPU_DENOISE_NLM, clahe = st->contrast == TSDRGPU_CONTRAST_CLAHE;
	float *cur = d_frames;
	int rc;
	if (stack) {
		if ((rc = stack_run(ctx, &st->stack, stream, cur, st->d_stack.ptr, nframes, w, h))) return rc;
		cur = st->d_stack.ptr;
	}
	if (st->deblur == TSDRGPU_DEBLUR_RL) {
		float *dst = (cur == d_frames) ? st->d_deblur.ptr : d_frames;
		if ((rc = fs_deblur_batch(ctx, stream, cur, dst, nframes, w, h, st->sigma_centi, st->iters))) return rc;
		cur = dst;
	}
	if (nlm) {
		float *dst = (cur == d_frames) ? st->d_nlm.ptr : d_frames;
		if ((rc = fs_nlm_batch(ctx, stream, cur, dst, nframes, w, h, st->h_milli, st->r, st->p))) return rc;
		cur = dst;
	}
	if (clahe) return fs_clahe_batch(ctx, st, stream, cur, d_frames, nframes, w, h);
	return cur == d_frames ? TSDRGPU_OK : fs_copy_async(ctx, stream, cur, d_frames, (size_t) nframes * w * h);
}

extern "C" {

int tsdrgpu_clahe(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_in, float *d_out, int w, int h, int nframes, int clip_centi,
                  int tx, int ty) {
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in && d_out && nframes > 0 && w > 0 && h > 0 && w <= 8192 && h <= 8192);     // tsdrgpu.h
	ARG_TRY(ctx, (size_t) w * h <= TSDRGPU_MAX_FRAME_PIXELS && ((((uintptr_t) d_in) | ((uintptr_t) d_out)) & 3) == 0);
	ARG_TRY(ctx, contrast_ok(TSDRGPU_CONTRAST_CLAHE, clip_centi, tx, ty));
	cudaStream_t stream = (cudaStream_t) stream_;
	EnhanceState st = {TSDRGPU_CONTRAST_CLAHE, clip_centi, tx, ty};           // the rest zero: no denoise, no buffers yet
	int rc = enhance_reserve(ctx, &st, nframes, w, h);
	if (rc == TSDRGPU_OK) rc = fs_clahe_batch(ctx, &st, stream, d_in, d_out, nframes, w, h);
	const cudaError_t e = cudaStreamSynchronize(stream);          // before the buffers go with st
	if (rc == TSDRGPU_OK && e != cudaSuccess) rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "tsdrgpu_clahe", e, __FILE__, __LINE__);
	return rc;
}

int tsdrgpu_nlm(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_in, float *d_out, int w, int h, int nframes, int h_milli, int r,
                int p) {
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in && d_out && nframes > 0 && w > 0 && h > 0 && (size_t) w * h <= TSDRGPU_MAX_FRAME_PIXELS);
	ARG_TRY(ctx, ((((uintptr_t) d_in) | ((uintptr_t) d_out)) & 3) == 0 && denoise_ok(TSDRGPU_DENOISE_NLM, h_milli, r, p));
	const uintptr_t bytes = (uintptr_t) sizeof(float) * w * h * nframes;
	ARG_TRY(ctx, (uintptr_t) d_out >= (uintptr_t) d_in + bytes || (uintptr_t) d_in >= (uintptr_t) d_out + bytes);
	cudaStream_t stream = (cudaStream_t) stream_;
	int rc = fs_nlm_batch(ctx, stream, d_in, d_out, nframes, w, h, h_milli, r, p);
	if (rc == TSDRGPU_OK) CU_TRY(ctx, cudaStreamSynchronize(stream));
	return rc;
}

int tsdrgpu_deblur(tsdrgpu_ctx_t *ctx, void *stream_, const float *d_in, float *d_out, int w, int h, int nframes, int sigma_centi,
                   int iterations) {
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in && d_out && nframes > 0 && w > 0 && h > 0 && (size_t) w * h <= TSDRGPU_MAX_FRAME_PIXELS);
	ARG_TRY(ctx, ((((uintptr_t) d_in) | ((uintptr_t) d_out)) & 3) == 0 && deblur_ok(TSDRGPU_DEBLUR_RL, sigma_centi, iterations));
	const uintptr_t bytes = (uintptr_t) sizeof(float) * w * h * nframes;
	ARG_TRY(ctx, (uintptr_t) d_out >= (uintptr_t) d_in + bytes || (uintptr_t) d_in >= (uintptr_t) d_out + bytes);
	cudaStream_t stream = (cudaStream_t) stream_;
	int rc = fs_deblur_batch(ctx, stream, d_in, d_out, nframes, w, h, sigma_centi, iterations);
	if (rc == TSDRGPU_OK) CU_TRY(ctx, cudaStreamSynchronize(stream));
	return rc;
}

}  // extern "C"
