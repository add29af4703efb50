// stack.cu -- drift-registered frame averaging on the frames the frame stage delivers, beyond the reference (definition in
// tsdrgpu.h).  Frames are taken one after the other; per frame, three launches on one stream: st_score adds every candidate's
// partial scores, st_pick chooses s* and the sub-pixel offset and keeps the offsets on the device, st_blend warps the frame into
// the accumulator and writes the output.  The adaptive mode replaces st_blend by three: st_tile_sums measures every tile's
// residual and marks the changed ones, st_decide restarts them and their neighbours and sets each tile's weights, and
// st_blend_tiles blends with those.  The tracking mode keeps st_tile_sums and replaces the other two: st_track_search looks for
// where each changed tile's content came from, st_track_decide restarts the tiles that changed and did not move (and their
// neighbours), and st_track_blend gathers the accumulator and the per-pixel counts along each tile's move into the second
// planes, which the host swaps with the first after every frame.  The glitch-tolerant mode keeps the tracking mode's first two
// and replaces the other two: st_robust_decide (one CTA) adds the debounce, counts the held tiles and decides a glitch frame, and
// st_robust_blend adds the pixel gate.  No host round trip inside a batch, and no CTA waits for another.  Built with -fmad=false;
// the float arithmetic is spelled with __f*_rn anyway, so every output bit follows the definition.
#include "common.cuh"
#include "host_plan.h"

#include <utility>

namespace {

constexpr int ST_THREADS = 256;
constexpr int ST_WPT = 4;                                   // words (four pixels each) of the accumulator per thread in st_score
constexpr int ST_TILE_WORDS = ST_THREADS * ST_WPT;
constexpr int ST_TILE = 4 * ST_TILE_WORDS;                  // pixels per st_score CTA
// the window of qF one dy row of candidates reads: the tile, 2 rx more bytes, and one word so that byte_perm may read past the end
constexpr int ST_WIN_WORDS = ST_TILE_WORDS + TSDRGPU_STACK_MAX_RX / 2 + 2;
constexpr int ST_MAX_CAND = (2 * TSDRGPU_STACK_MAX_RX + 1) * (2 * TSDRGPU_STACK_MAX_RY + 1);

struct StackOffsets { double o1, o2; };
size_t st_tiles_x(int w) { return ((size_t) w + TSDRGPU_STACK_TILE - 1) / TSDRGPU_STACK_TILE; }
size_t st_tiles_y(int h) { return ((size_t) h + TSDRGPU_STACK_TILE - 1) / TSDRGPU_STACK_TILE; }

__device__ __forceinline__ unsigned st_q(float v) {         // Q(v) of a valid v
	return (unsigned) (int) __fadd_rn(__fmul_rn(fminf(fmaxf(v, 0.0f), 1.0f), 255.0f), 0.5f);
}
__device__ __forceinline__ double st_round(double x) { return floor(x + 0.5); }
__device__ __forceinline__ unsigned st_wrap(long long x, long long n) { const long long r = x % n; return (unsigned) (r < 0 ? r + n : r); }
// the base of the search, b = R(o1) + (m >= 2 ? R(o1) - R(o2) : 0)
__device__ __forceinline__ double st_base(const StackOffsets *o, int m2) {
	const double r1 = st_round(o->o1);
	return m2 ? r1 + (r1 - st_round(o->o2)) : r1;
}

// scores: one CTA per ST_TILE pixels q of the accumulator.  The CTA packs qA of its tile into registers (four pixels per word,
// the lowest byte first); per dy it stages the window of qF the row of candidates reads, packed the same way, and every dx is then
// a byte_perm of two neighbouring words and one __dp4a per word.  A warp's per-candidate sum (at most 512 * 255^2) goes through
// __reduce_add_sync into the CTA's counts (at most ST_TILE * 255^2 < 2^32), and those into the 64-bit scores.
__global__ void __launch_bounds__(ST_THREADS) st_score(const float *__restrict__ F, const float *__restrict__ A, unsigned n, int W,
                                                       int rx, int ry, int m2, const StackOffsets *__restrict__ off,
                                                       unsigned long long *__restrict__ scores) {
	__shared__ unsigned s_win[ST_WIN_WORDS];
	__shared__ unsigned s_sc[ST_MAX_CAND];
	const int nx = 2 * rx + 1, ncand = nx * (2 * ry + 1);
	const unsigned q0 = blockIdx.x * (unsigned) ST_TILE;
	for (int c = threadIdx.x; c < ncand; c += ST_THREADS) s_sc[c] = 0;
	unsigned a[ST_WPT];
#pragma unroll
	for (int i = 0; i < ST_WPT; i++) {
		const unsigned q = q0 + 4u * (threadIdx.x + ST_THREADS * i);
		unsigned word = 0;
#pragma unroll
		for (int k = 0; k < 4; k++) if (q + k < n) word |= st_q(A[q + k]) << (8 * k);
		a[i] = word;
	}
	const long long b = (long long) st_base(off, m2);
	const int win_words = ST_TILE_WORDS + (2 * rx) / 4 + 2;
	const unsigned sel[4] = {0x3210u, 0x4321u, 0x5432u, 0x6543u};
	const int lane = threadIdx.x & 31;
	for (int dy = -ry; dy <= ry; dy++) {
		const unsigned base = q0 + st_wrap(b + (long long) dy * W - rx, n);    // window byte e holds qF[base + e]
		__syncthreads();                                     // the previous row's window is no longer read
		for (int e4 = threadIdx.x; e4 < win_words; e4 += ST_THREADS) {
			unsigned word = 0;
#pragma unroll
			for (int k = 0; k < 4; k++) {
				unsigned g = base + 4u * e4 + k;
				if (g >= n) g %= n;
				const float v = __ldg(F + g);
				if (px_valid(v)) word |= st_q(v) << (8 * k);
			}
			s_win[e4] = word;
		}
		__syncthreads();
		unsigned *row = s_sc + (dy + ry) * nx;
		for (int k = 0; 4 * k < nx; k++) {
			unsigned lo[ST_WPT], hi[ST_WPT];
#pragma unroll
			for (int i = 0; i < ST_WPT; i++) {
				const int w = threadIdx.x + ST_THREADS * i + k;
				lo[i] = s_win[w]; hi[i] = s_win[w + 1];
			}
#pragma unroll
			for (int r = 0; r < 4; r++) {
				const int j = 4 * k + r;                     // dx = j - rx
				if (j >= nx) break;
				unsigned acc = 0;
#pragma unroll
				for (int i = 0; i < ST_WPT; i++) acc = __dp4a(__byte_perm(lo[i], hi[i], sel[r]), a[i], acc);
				acc = __reduce_add_sync(0xffffffffu, acc);
				if (lane == 0 && acc) atomicAdd(&row[j], acc);
			}
		}
	}
	__syncthreads();
	for (int c = threadIdx.x; c < ncand; c += ST_THREADS) if (s_sc[c]) atomicAdd(scores + c, (unsigned long long) s_sc[c]);
}

// s* (largest score, first in loop order on a tie), the sub-pixel fit and the offsets; the frame's record; the scores back to 0
__global__ void __launch_bounds__(1024) st_pick(unsigned long long *scores, int W, int rx, int ry, int m2, StackOffsets *off,
                                                tsdrgpu_stack_record_t *rec) {
	__shared__ unsigned long long s_best[32];
	__shared__ int s_idx[32];
	const int nx = 2 * rx + 1, ncand = nx * (2 * ry + 1);
	unsigned long long best = 0;
	int idx = 0x7fffffff;
	for (int c = threadIdx.x; c < ncand; c += blockDim.x) {
		const unsigned long long s = scores[c];
		if (idx == 0x7fffffff || s > best) { best = s; idx = c; }          // c rises: the first of equal scores stays
	}
	auto better = [](unsigned long long s, int i, unsigned long long t, int j) { return j != 0x7fffffff && (i == 0x7fffffff || t > s || (t == s && j < i)); };
	for (int o = 16; o > 0; o >>= 1) {
		const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
		const int j = __shfl_xor_sync(0xffffffffu, idx, o);
		if (better(best, idx, t, j)) { best = t; idx = j; }
	}
	if ((threadIdx.x & 31) == 0) { s_best[threadIdx.x >> 5] = best; s_idx[threadIdx.x >> 5] = idx; }
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int k = 1; k < (int) (blockDim.x >> 5); k++) if (better(best, idx, s_best[k], s_idx[k])) { best = s_best[k]; idx = s_idx[k]; }
		const int dy = idx / nx - ry, dx = idx % nx - rx;
		const double sstar = st_base(off, m2) + (double) ((long long) dy * W + dx);
		double delta = 0.0;
		if (dx > -rx && dx < rx) {
			const double a = (double) scores[idx - 1], c = (double) scores[idx + 1], M = (double) best;
			const double den = (a - 2.0 * M) + c;
			if (den < 0.0) delta = fmin(fmax((a - c) / (2.0 * den), -0.5), 0.5);
		}
		const double o = sstar + delta;
		off->o2 = off->o1; off->o1 = o;
		tsdrgpu_stack_record_t r;
		r.offset = o; r.score = (int64_t) best; r.dx = dx; r.dy = dy; r.restarted = 0; r.changed = 0;
		*rec = r;
	}
	__syncthreads();
	for (int c = threadIdx.x; c < ncand; c += blockDim.x) scores[c] = 0;
}

// the warp of step 5 for o = off->o1: the Catmull-Rom weights, q's first tap q + I - 1 and the output shift R(o), both mod n
struct StackWarp { float wm1, w0, w1, w2; unsigned im1, ro; };
__device__ __forceinline__ StackWarp st_warp(const StackOffsets *off, unsigned n) {
	const double o = off->o1, I = floor(o);
	const float t = (float) (o - I);
	StackWarp c;
	c.wm1 = __fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(-0.5f, t), 1.0f), t), 0.5f), t);
	c.w0 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.5f, t), 2.5f), t), t), 1.0f);
	c.w1 = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(-1.5f, t), 2.0f), t), 0.5f), t);
	c.w2 = __fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(0.5f, t), 0.5f), t), t);
	c.im1 = st_wrap((long long) I - 1, n); c.ro = st_wrap((long long) st_round(o), n);
	return c;
}
__device__ __forceinline__ unsigned st_wrapu(unsigned g, unsigned n) { while (g >= n) g -= n; return g; }    // g < 2n + 3: a few steps
// x[q] into *x when all four taps are valid
__device__ __forceinline__ bool st_tap(const float *__restrict__ F, const StackWarp &c, unsigned q, unsigned n, float *x) {
	const unsigned g = st_wrapu(q + c.im1, n);
	const float f0 = __ldg(F + g), f1 = __ldg(F + st_wrapu(g + 1, n)), f2 = __ldg(F + st_wrapu(g + 2, n)), f3 = __ldg(F + st_wrapu(g + 3, n));
	if (!(px_valid(f0) && px_valid(f1) && px_valid(f2) && px_valid(f3))) return false;
	*x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.wm1, f0), __fmul_rn(c.w0, f1)), __fmul_rn(c.w1, f2)), __fmul_rn(c.w2, f3));
	return true;
}

// warp frame F by o = off->o1 into the accumulator where all four taps are valid, then out[q + R(o)] from the new A[q].  The taps
// are spelled out here rather than taken through st_tap, which keeps this kernel's machine code as it was before the adaptive mode.
__global__ void __launch_bounds__(ST_THREADS) st_blend(const float *__restrict__ F, float *__restrict__ A, float *__restrict__ out,
                                                       unsigned n, float wo, float wn, const StackOffsets *__restrict__ off) {
	const StackWarp c = st_warp(off, n);
	for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
		const unsigned g = st_wrapu(q + c.im1, n);
		const float f0 = __ldg(F + g), f1 = __ldg(F + st_wrapu(g + 1, n)), f2 = __ldg(F + st_wrapu(g + 2, n)), f3 = __ldg(F + st_wrapu(g + 3, n));
		float acc = A[q];
		if (px_valid(f0) && px_valid(f1) && px_valid(f2) && px_valid(f3)) {
			const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(c.wm1, f0), __fmul_rn(c.w0, f1)), __fmul_rn(c.w1, f2)), __fmul_rn(c.w2, f3));
			acc = __fadd_rn(__fmul_rn(acc, wo), __fmul_rn(x, wn));
			A[q] = acc;
		}
		const unsigned p = st_wrapu(q + c.ro, n);
		const float fp = __ldg(F + p);
		out[p] = px_valid(fp) ? acc : fp;
	}
}

// adapt, step 6a-b: one CTA per tile (ST_THREADS = TILE^2 threads, thread i at (i mod TILE, i div TILE) of the tile).  D_t (at
// most TILE^2 * 255^2 < 2^32) and C_t by warp sums; the tile's r and its flag against its level e_t, which st_decide updates.
constexpr int ST_TILE_PX = TSDRGPU_STACK_TILE;
constexpr unsigned ST_NO_LEVEL = 0xffffffffu;
static_assert(ST_TILE_PX * ST_TILE_PX == ST_THREADS, "one thread per pixel of a tile");
__global__ void __launch_bounds__(ST_THREADS) st_tile_sums(const float *__restrict__ F, const float *__restrict__ A, unsigned n,
                                                           int W, int H, int tx, const StackOffsets *__restrict__ off,
                                                           StackTile *__restrict__ tiles) {
	__shared__ unsigned s_d[ST_THREADS / 32], s_c[ST_THREADS / 32];
	const StackWarp c = st_warp(off, n);
	const int t = blockIdx.x;
	const int X = (t % tx) * ST_TILE_PX + (int) (threadIdx.x % ST_TILE_PX), Y = (t / tx) * ST_TILE_PX + (int) (threadIdx.x / ST_TILE_PX);
	unsigned d2 = 0, cnt = 0;
	float x;
	if (X < W && Y < H) {
		const unsigned q = (unsigned) Y * (unsigned) W + (unsigned) X;
		if (st_tap(F, c, q, n, &x)) {
			const int d = (int) st_q(x) - (int) st_q(A[q]);
			d2 = (unsigned) (d * d); cnt = 1;
		}
	}
	d2 = __reduce_add_sync(0xffffffffu, d2);
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if ((threadIdx.x & 31) == 0) { s_d[threadIdx.x >> 5] = d2; s_c[threadIdx.x >> 5] = cnt; }
	__syncthreads();
	if (threadIdx.x == 0) {
		unsigned long long D = 0, C = 0;
		for (int k = 0; k < ST_THREADS / 32; k++) { D += s_d[k]; C += s_c[k]; }
		const unsigned long long e = tiles[t].e;
		int flag = 0;
		unsigned r = 0;
		if (C) {
			r = (unsigned) (16ull * D / C);
			flag = e != ST_NO_LEVEL && 16ull * D > TSDRGPU_STACK_ADAPT_RATIO * e * C && D > TSDRGPU_STACK_ADAPT_FLOOR * C ? 2 : 1;
		}
		tiles[t].r = r; tiles[t].flag = flag;
	}
}

// adapt, step 6b-c: one thread per tile.  A tile restarts when it or one of its 8 neighbours changed; its weights for this frame,
// its new count and level; the frame's record counts the restarts (integer atomics: the same total in any order).
__global__ void __launch_bounds__(ST_THREADS) st_decide(StackTile *__restrict__ tiles, int tx, int ty, int depth,
                                                        tsdrgpu_stack_record_t *rec) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	bool restart = false;
	if (t < tx * ty) {
		const int X = t % tx, Y = t / tx;
		for (int y = max(Y - 1, 0); y <= min(Y + 1, ty - 1); y++)
			for (int x = max(X - 1, 0); x <= min(X + 1, tx - 1); x++) restart |= tiles[y * tx + x].flag == 2;
	}
	if (t < tx * ty) {                                       // nothing here writes a flag, so neighbours may read them meanwhile
		StackTile &s = tiles[t];
		int m = s.m;
		unsigned e = s.e;
		if (restart) { m = 0; e = ST_NO_LEVEL; }
		else if (s.flag) e = e == ST_NO_LEVEL ? s.r : (unsigned) ((7ull * e + s.r) / 8);
		const int k = min(m + 1, depth);
		s.wn = (float) (1.0 / (double) k); s.wo = (float) (1.0 - 1.0 / (double) k);
		s.m = k; s.e = e;
	}
	const unsigned cnt = __reduce_add_sync(0xffffffffu, restart ? 1u : 0u);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&rec->changed, (int) cnt);
}

// adapt, step 6d and 7: st_blend with the weights of q's tile
__global__ void __launch_bounds__(ST_THREADS) st_blend_tiles(const float *__restrict__ F, float *__restrict__ A, float *__restrict__ out,
                                                             unsigned n, unsigned W, int tx, const StackTile *__restrict__ tiles,
                                                             const StackOffsets *__restrict__ off) {
	const StackWarp c = st_warp(off, n);
	for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
		float acc = A[q], x;
		if (st_tap(F, c, q, n, &x)) {
			const unsigned y = q / W;
			const StackTile &s = tiles[(y / ST_TILE_PX) * tx + (q - y * W) / ST_TILE_PX];
			acc = __fadd_rn(__fmul_rn(acc, s.wo), __fmul_rn(x, s.wn));
			A[q] = acc;
		}
		const unsigned p = st_wrapu(q + c.ro, n);
		const float fp = __ldg(F + p);
		out[p] = px_valid(fp) ? acc : fp;
	}
}

// adapt, a restart frame: every m_t = 1, e_t = none
__global__ void __launch_bounds__(ST_THREADS) st_tile_init(StackTile *tiles, int ntiles) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t < ntiles) { tiles[t].m = 1; tiles[t].e = ST_NO_LEVEL; }
}

// a restart frame: A = valid ? F : 0, out = F, o1 = o2 = 0
__global__ void __launch_bounds__(ST_THREADS) st_restart(const float *__restrict__ F, float *__restrict__ A, float *__restrict__ out,
                                                         unsigned n, StackOffsets *off, tsdrgpu_stack_record_t *rec) {
	for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		const float v = __ldg(F + p);
		A[p] = px_valid(v) ? v : 0.0f;
		out[p] = v;
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		off->o1 = 0.0; off->o2 = 0.0;
		tsdrgpu_stack_record_t r;
		r.offset = 0.0; r.score = 0; r.dx = 0; r.dy = 0; r.restarted = 1; r.changed = 0;
		*rec = r;
	}
}

// track, step 6t: one CTA per tile, returning at once unless the tile changed.  The CTA stages Q(x) of its tile (four pixels per
// word, lowest byte first) with a byte mask of the pixels whose taps are valid, and the window of Q(A) every candidate reads:
// (16 + 2 LX) x (16 + 2 LY) bytes, 0 outside the raster, one spare word per row so that byte_perm may read past the end.  Each
// thread takes candidates in loop order; per word of the tile, byte_perm takes the candidate's horizontal phase, vabsdiffu4 the
// distance, the mask the pixels of p and s both in the sum, and dp4a adds d^2 (D <= 256 * 255^2 < 2^32).  C(v) is the mask's
// population.  The best candidate of a thread, of a warp and of the CTA, by the definition's exact order.
constexpr int TK_LX = TSDRGPU_STACK_TRACK_LX, TK_LY = TSDRGPU_STACK_TRACK_LY;
constexpr int TK_NX = 2 * TK_LX + 1, TK_NCAND = TK_NX * (2 * TK_LY + 1);
constexpr int TK_WIN_ROWS = ST_TILE_PX + 2 * TK_LY;
constexpr int TK_WIN_WORDS = (ST_TILE_PX + 2 * TK_LX) / 4 + 1;          // words per window row
static_assert(TK_LX % 4 == 0 && ST_TILE_PX % 4 == 0, "window rows start on a word");
struct TrackBest { unsigned d, c; int l1, idx; };                         // idx < 0: none
__device__ __forceinline__ bool tk_better(const TrackBest &a, const TrackBest &b) {   // a before b in the definition's order
	if (a.idx < 0) return false;
	if (b.idx < 0) return true;
	const unsigned long long l = (unsigned long long) a.d * b.c, r = (unsigned long long) b.d * a.c;
	return l != r ? l < r : a.l1 != b.l1 ? a.l1 < b.l1 : a.idx < b.idx;
}
__global__ void __launch_bounds__(ST_THREADS) st_track_search(const float *__restrict__ F, const float *__restrict__ A, unsigned n,
                                                              int W, int H, int tx, const StackOffsets *__restrict__ off,
                                                              const StackTile *__restrict__ tiles, StackTrack *__restrict__ track) {
	__shared__ __align__(4) unsigned char s_q[ST_TILE_PX * ST_TILE_PX], s_m[ST_TILE_PX * ST_TILE_PX];
	__shared__ __align__(4) unsigned char s_win[TK_WIN_ROWS * TK_WIN_WORDS * 4];
	__shared__ TrackBest s_best[ST_THREADS / 32];
	const int t = blockIdx.x;
	if (tiles[t].flag != 2) return;
	const StackWarp cw = st_warp(off, n);
	const int X0 = (t % tx) * ST_TILE_PX, Y0 = (t / tx) * ST_TILE_PX;
	{
		const int X = X0 + (int) (threadIdx.x % ST_TILE_PX), Y = Y0 + (int) (threadIdx.x / ST_TILE_PX);
		unsigned char qv = 0, mv = 0;
		float x;
		if (X < W && Y < H && st_tap(F, cw, (unsigned) Y * (unsigned) W + (unsigned) X, n, &x)) { qv = (unsigned char) st_q(x); mv = 0xff; }
		s_q[threadIdx.x] = qv; s_m[threadIdx.x] = mv;
	}
	for (int e = threadIdx.x; e < TK_WIN_ROWS * TK_WIN_WORDS * 4; e += ST_THREADS) {
		const int r = e / (TK_WIN_WORDS * 4), b = e - r * (TK_WIN_WORDS * 4);
		const int X = X0 - TK_LX + b, Y = Y0 - TK_LY + r;
		s_win[e] = (b < ST_TILE_PX + 2 * TK_LX && X >= 0 && X < W && Y >= 0 && Y < H)
		           ? (unsigned char) st_q(A[(unsigned) Y * (unsigned) W + (unsigned) X]) : 0;
	}
	const int c0 = __syncthreads_count(s_m[threadIdx.x] != 0);
	const unsigned *q4 = reinterpret_cast<const unsigned *>(s_q), *m4 = reinterpret_cast<const unsigned *>(s_m);
	const unsigned *w4 = reinterpret_cast<const unsigned *>(s_win);
	TrackBest best = {0u, 0u, 0, -1};
	for (int idx = threadIdx.x; idx < TK_NCAND; idx += ST_THREADS) {
		const int vy = idx / TK_NX - TK_LY, vx = idx % TK_NX - TK_LX;
		if (vx == 0 && vy == 0) continue;
		// the tile's rows y and columns x whose source Y0 + y - vy, X0 + x - vx lies inside the raster
		const int ylo = max(0, vy - Y0), yhi = min(ST_TILE_PX, H - Y0 + vy);
		const int xlo = max(0, vx - X0), xhi = min(ST_TILE_PX, W - X0 + vx);
		if (ylo >= yhi || xlo >= xhi) continue;
		const unsigned cols = (0xffffu >> (ST_TILE_PX - xhi)) & (0xffffu << xlo);
		unsigned cm[ST_TILE_PX / 4];
#pragma unroll
		for (int j = 0; j < ST_TILE_PX / 4; j++) {
			const unsigned b = cols >> (4 * j);
			cm[j] = (b & 1u ? 0xffu : 0u) | (b & 2u ? 0xff00u : 0u) | (b & 4u ? 0xff0000u : 0u) | (b & 8u ? 0xff000000u : 0u);
		}
		const int sh = TK_LX - vx;                                       // byte of the window row under the tile's column 0
		const unsigned sel = 0x3210u + 0x1111u * (unsigned) (sh & 3);
		unsigned D = 0, Cb = 0;
		for (int y = ylo; y < yhi; y++) {
			const unsigned *wr = w4 + (y - vy + TK_LY) * TK_WIN_WORDS + (sh >> 2);
#pragma unroll
			for (int j = 0; j < ST_TILE_PX / 4; j++) {
				const unsigned m = m4[y * (ST_TILE_PX / 4) + j] & cm[j];
				const unsigned d = __vabsdiffu4(q4[y * (ST_TILE_PX / 4) + j], __byte_perm(wr[j], wr[j + 1], sel)) & m;
				D = __dp4a(d, d, D);
				Cb += __popc(m);
			}
		}
		const unsigned C = Cb >> 3;
		if (C == 0 || 2 * C < (unsigned) c0) continue;
		const TrackBest cand = {D, C, abs(vx) + abs(vy), idx};
		if (tk_better(cand, best)) best = cand;
	}
	for (int o = 16; o > 0; o >>= 1) {
		TrackBest b;
		b.d = __shfl_xor_sync(0xffffffffu, best.d, o); b.c = __shfl_xor_sync(0xffffffffu, best.c, o);
		b.l1 = __shfl_xor_sync(0xffffffffu, best.l1, o); b.idx = __shfl_xor_sync(0xffffffffu, best.idx, o);
		if (tk_better(b, best)) best = b;
	}
	if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int k = 1; k < ST_THREADS / 32; k++) if (tk_better(s_best[k], best)) best = s_best[k];
		StackTrack r = {0, 0, 0u, 0u, 0, 0, 0, 0};
		if (best.idx >= 0) {
			const unsigned long long e = tiles[t].e, D = best.d, C = best.c;
			r.vx = best.idx % TK_NX - TK_LX; r.vy = best.idx / TK_NX - TK_LY; r.d = best.d; r.c = best.c;
			r.moved = !(16ull * D > TSDRGPU_STACK_ADAPT_RATIO * e * C && D > TSDRGPU_STACK_ADAPT_FLOOR * C);
		}
		track[t].vx = r.vx; track[t].vy = r.vy; track[t].d = r.d; track[t].c = r.c; track[t].moved = r.moved;
	}
}

// track, steps 6b-c: one thread per tile, as st_decide.  Restarts spread from tiles that changed and did not move; the move and
// the restart the blend takes; the record counts the restarts.
__global__ void __launch_bounds__(ST_THREADS) st_track_decide(StackTile *__restrict__ tiles, StackTrack *__restrict__ track, int tx,
                                                              int ty, tsdrgpu_stack_record_t *rec) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	bool restart = false;
	if (t < tx * ty) {
		const int X = t % tx, Y = t / tx;
		for (int y = max(Y - 1, 0); y <= min(Y + 1, ty - 1); y++)
			for (int x = max(X - 1, 0); x <= min(X + 1, tx - 1); x++) restart |= tiles[y * tx + x].flag == 2 && !track[y * tx + x].moved;
	}
	if (t < tx * ty) {                                       // flag and moved are only read here, e, bx, by, restart only written
		StackTile &s = tiles[t];
		StackTrack &k = track[t];
		unsigned e = s.e;
		int bx = 0, by = 0;
		if (restart) e = ST_NO_LEVEL;
		else if (s.flag == 2) {                              // changed and not restarting: it moved
			e = (unsigned) ((7ull * e + 16ull * k.d / k.c) / 8);
			bx = k.vx; by = k.vy;
		} else if (s.flag) e = e == ST_NO_LEVEL ? s.r : (unsigned) ((7ull * e + s.r) / 8);
		s.e = e; k.bx = bx; k.by = by; k.restart = restart;
	}
	const unsigned cnt = __reduce_add_sync(0xffffffffu, restart ? 1u : 0u);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&rec->changed, (int) cnt);
}

// track, steps 6d and 7: A' and c' at q from A and c at q's source, then out[q + R(o)] from A'[q]
__global__ void __launch_bounds__(ST_THREADS) st_track_blend(const float *__restrict__ F, const float *__restrict__ A,
                                                             float *__restrict__ A2, const uint16_t *__restrict__ cnt,
                                                             uint16_t *__restrict__ cnt2, float *__restrict__ out, unsigned n,
                                                             int W, int H, int tx, int depth, const StackTrack *__restrict__ track,
                                                             const StackOffsets *__restrict__ off) {
	const StackWarp c = st_warp(off, n);
	for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
		const int Y = (int) (q / (unsigned) W), X = (int) (q - (unsigned) Y * (unsigned) W);
		const StackTrack &T = track[(Y / ST_TILE_PX) * tx + X / ST_TILE_PX];
		unsigned s = q;
		int cs = 0;
		if (!T.restart) {
			const int sx = X - T.bx, sy = Y - T.by;
			if (sx >= 0 && sx < W && sy >= 0 && sy < H) { s = (unsigned) sy * (unsigned) W + (unsigned) sx; cs = cnt[s]; }
		}
		const int k = min(cs + 1, depth);
		float acc = A[s], x;
		if (st_tap(F, c, q, n, &x)) {
			const float wn = (float) (1.0 / (double) k), wo = (float) (1.0 - 1.0 / (double) k);
			acc = __fadd_rn(__fmul_rn(acc, wo), __fmul_rn(x, wn));
		}
		A2[q] = acc;
		cnt2[q] = (uint16_t) k;
		const unsigned p = st_wrapu(q + c.ro, n);
		const float fp = __ldg(F + p);
		out[p] = px_valid(fp) ? acc : fp;
	}
}

// track, a restart frame: every c = 1 and no tile moved
__global__ void __launch_bounds__(ST_THREADS) st_track_init(uint16_t *cnt, unsigned n, StackTrack *track, int ntiles) {
	for (unsigned p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) cnt[p] = 1;
	for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < ntiles; t += gridDim.x * blockDim.x) {
		track[t].bx = 0; track[t].by = 0; track[t].restart = 0;
	}
}

// robust, steps 6r, 6h and 6c: one CTA for the whole tile grid, so that the held count and the glitch-frame decision need no
// second launch.  Pass 1 marks the confirmed tiles, pass 2 spreads their restarts and counts the held tiles, pass 3 sets each
// tile's level, move, restart, gate level and pend for the blend.  Thread 0 then keeps a glitch frame's prediction as the
// offset (st_warp in st_robust_blend reads it for the output) and the record's, and leaves the next frame's prediction.
constexpr int RB_THREADS = 1024;
constexpr uint16_t RB_GATED = 0x8000u, RB_COUNT = 0x7fffu;
__global__ void __launch_bounds__(RB_THREADS) st_robust_decide(StackTile *__restrict__ tiles, StackTrack *__restrict__ track,
                                                               StackRobust *__restrict__ rob, int tx, int ty, StackOffsets *off,
                                                               StackRobustFrame *fr, tsdrgpu_stack_record_t *rec) {
	__shared__ int s_held, s_restarts;
	const int ntiles = tx * ty;
	if (threadIdx.x == 0) { s_held = 0; s_restarts = 0; }
	for (int t = threadIdx.x; t < ntiles; t += RB_THREADS)
		rob[t].confirmed = tiles[t].flag == 2 && !track[t].moved && rob[t].pend;
	__syncthreads();
	int held = 0;
	for (int t = threadIdx.x; t < ntiles; t += RB_THREADS) {
		const int X = t % tx, Y = t / tx;
		bool restart = false;
		for (int y = max(Y - 1, 0); y <= min(Y + 1, ty - 1); y++)
			for (int x = max(X - 1, 0); x <= min(X + 1, tx - 1); x++) restart |= rob[y * tx + x].confirmed != 0;
		const bool h = tiles[t].flag == 2 && !track[t].moved && !rob[t].pend && !restart;
		track[t].restart = restart;
		rob[t].held = h;
		held += h;
	}
	held = (int) __reduce_add_sync(0xffffffffu, (unsigned) held);
	if ((threadIdx.x & 31) == 0 && held) atomicAdd(&s_held, held);
	__syncthreads();
	const bool hold = 2 * s_held > ntiles;
	int restarts = 0;
	for (int t = threadIdx.x; t < ntiles; t += RB_THREADS) {   // every read and write here is of tile t's own entries
		StackTile &s = tiles[t];
		StackTrack &k = track[t];
		StackRobust &r = rob[t];
		unsigned e = s.e, ge = ST_NO_LEVEL;
		int bx = 0, by = 0;
		bool restart = k.restart && !hold;
		if (restart) e = ST_NO_LEVEL;
		else if (!hold && !r.held) {
			ge = e;
			if (s.flag == 2) {                                 // changed, not restarting, not held: it moved
				e = (unsigned) ((7ull * e + 16ull * k.d / k.c) / 8);
				bx = k.vx; by = k.vy;
			} else if (s.flag) e = e == ST_NO_LEVEL ? s.r : (unsigned) ((7ull * e + s.r) / 8);
		}
		s.e = e; k.bx = bx; k.by = by; k.restart = restart;
		r.gate_e = ge; r.pend = s.flag == 2 && !k.moved;
		restarts += restart;
	}
	restarts = (int) __reduce_add_sync(0xffffffffu, (unsigned) restarts);
	if ((threadIdx.x & 31) == 0 && restarts) atomicAdd(&s_restarts, restarts);
	__syncthreads();
	if (threadIdx.x == 0) {
		if (hold) { off->o1 = fr->b; rec->offset = fr->b; }
		rec->changed = s_restarts;
		fr->held = s_held; fr->hold = hold; fr->gated = 0;
		fr->b = st_base(off, 1);                              // every later frame has m >= 2
	}
}

// robust, steps 6d and 7: track's gather and blend with the pixel gate; held tiles and a glitch frame copy A and c over
__global__ void __launch_bounds__(ST_THREADS) st_robust_blend(const float *__restrict__ F, const float *__restrict__ A,
                                                              float *__restrict__ A2, const uint16_t *__restrict__ cnt,
                                                              uint16_t *__restrict__ cnt2, float *__restrict__ out, unsigned n,
                                                              int W, int H, int tx, int depth, const StackTrack *__restrict__ track,
                                                              const StackRobust *__restrict__ rob,
                                                              StackRobustFrame *fr, const StackOffsets *__restrict__ off) {
	const StackWarp c = st_warp(off, n);                      // on a glitch frame o1 = b already: the output moves by R(b)
	const bool hold = fr->hold;
	unsigned gated = 0;
	for (unsigned q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
		const int Y = (int) (q / (unsigned) W), X = (int) (q - (unsigned) Y * (unsigned) W);
		const int t = (Y / ST_TILE_PX) * tx + X / ST_TILE_PX;
		float acc;
		unsigned c2;
		if (hold || rob[t].held) { acc = A[q]; c2 = cnt[q]; }
		else {
			const StackTrack &T = track[t];
			unsigned s = q, cs = 0, g = 0;
			bool inside = false;
			if (!T.restart) {
				const int sx = X - T.bx, sy = Y - T.by;
				if (sx >= 0 && sx < W && sy >= 0 && sy < H) {
					s = (unsigned) sy * (unsigned) W + (unsigned) sx;
					cs = cnt[s]; g = cs & RB_GATED; cs &= RB_COUNT; inside = true;
				}
			}
			const int k = min((int) cs + 1, depth);
			acc = A[s]; c2 = (unsigned) k;
			float x;
			if (st_tap(F, c, q, n, &x)) {
				const unsigned ge = rob[t].gate_e;
				const int d = (int) st_q(x) - (int) st_q(acc);
				if (inside && ge != ST_NO_LEVEL && (unsigned) (d * d) > max(ge, (unsigned) TSDRGPU_STACK_ROBUST_GATE_MIN)) {
					gated++;
					if (g) { acc = x; c2 = 1; }
					else c2 = cs | RB_GATED;
				} else {
					const float wn = (float) (1.0 / (double) k), wo = (float) (1.0 - 1.0 / (double) k);
					acc = __fadd_rn(__fmul_rn(acc, wo), __fmul_rn(x, wn));
				}
			}
		}
		A2[q] = acc;
		cnt2[q] = (uint16_t) c2;
		const unsigned p = st_wrapu(q + c.ro, n);
		const float fp = __ldg(F + p);
		out[p] = px_valid(fp) ? acc : fp;
	}
	gated = __reduce_add_sync(0xffffffffu, gated);
	if ((threadIdx.x & 31) == 0 && gated) atomicAdd(&fr->gated, (unsigned long long) gated);
}

// robust, a restart frame (after st_track_init): every pend_t = 0, and the next frame's prediction b = R(0) = 0
__global__ void __launch_bounds__(ST_THREADS) st_robust_init(StackRobust *rob, int ntiles, StackRobustFrame *fr) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t < ntiles) { rob[t].pend = 0; rob[t].confirmed = 0; rob[t].held = 0; rob[t].gate_e = ST_NO_LEVEL; }
	if (t == 0) { fr->b = 0.0; fr->held = 0; fr->hold = 0; fr->gated = 0; }
}

template <class T> void st_swap(DeviceBuf<T> &a, DeviceBuf<T> &b) { std::swap(a.ptr, b.ptr); std::swap(a.cap, b.cap); }

}  // namespace

// the accumulator (restarted when the geometry changes), the offsets, the scores and nframes records; in adapt, track and robust
// modes the tiles, in track and robust modes the second accumulator, the count planes and the search results, in robust mode
// the debounce state; nothing may be in flight
int stack_reserve(tsdrgpu_ctx_t *ctx, StackState *st, int nframes, int w, int h) {
	if (st->mode == TSDRGPU_STACK_OFF) return TSDRGPU_OK;
	const size_t n = (size_t) w * h;
	const bool robust = st->mode == TSDRGPU_STACK_ROBUST, track = st->mode == TSDRGPU_STACK_TRACK || robust;
	const size_t ntiles = st->mode == TSDRGPU_STACK_ADAPT || track ? st_tiles_x(w) * st_tiles_y(h) : 0;
	const size_t n2 = track ? n : 0, ntrack = track ? ntiles : 0, nrobust = robust ? ntiles : 0;
	if (w != st->w || h != st->h) { st->w = w; st->h = h; st->m = 0; }
	const bool grow = st->d_acc.cap < n || !st->d_off.ptr || st->d_rec.cap < (size_t) nframes || st->d_tiles.cap < ntiles ||
	                  st->d_acc2.cap < n2 || st->d_cnt.cap < n2 || st->d_cnt2.cap < n2 || st->d_track.cap < ntrack ||
	                  st->d_robust.cap < nrobust || (robust && !st->d_rframe.ptr);
	if (grow) CU_TRY(ctx, cudaDeviceSynchronize());
	if (st->d_acc.cap < n) CU_TRY(ctx, st->d_acc.assign(n));
	if (st->d_tiles.cap < ntiles) CU_TRY(ctx, st->d_tiles.assign(ntiles));
	if (st->d_acc2.cap < n2) CU_TRY(ctx, st->d_acc2.assign(n2));
	if (st->d_cnt.cap < n2) CU_TRY(ctx, st->d_cnt.assign(n2));
	if (st->d_cnt2.cap < n2) CU_TRY(ctx, st->d_cnt2.assign(n2));
	if (st->d_track.cap < ntrack) CU_TRY(ctx, st->d_track.assign(ntrack));
	if (st->d_robust.cap < nrobust) CU_TRY(ctx, st->d_robust.assign(nrobust));
	if (robust && !st->d_rframe.ptr) CU_TRY(ctx, st->d_rframe.assign(1));
	if (st->d_rec.cap < (size_t) nframes) CU_TRY(ctx, st->d_rec.assign(nframes));
	if (!st->d_off.ptr) {
		CU_TRY(ctx, st->d_off.assign(2));
		CU_TRY(ctx, st->d_scores.assign(ST_MAX_CAND));
		CU_TRY(ctx, cudaMemset(st->d_scores.ptr, 0, sizeof(unsigned long long) * ST_MAX_CAND));    // st_pick leaves them at 0
		CU_TRY(ctx, cudaDeviceSynchronize());
	}
	return TSDRGPU_OK;
}

// nframes frames of w x h, in -> out (no overlap), on `stream`; stack_reserve has been called for this geometry and batch
int stack_run(tsdrgpu_ctx_t *ctx, StackState *st, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h) {
	const unsigned n = (unsigned) ((size_t) w * h);
	StackOffsets *off = reinterpret_cast<StackOffsets *>(st->d_off.ptr);
	const unsigned tiles = (n + ST_TILE - 1) / ST_TILE;
	unsigned grid = (n + ST_THREADS - 1) / ST_THREADS;
	if (grid > (unsigned) ctx->sm_count * 8) grid = (unsigned) ctx->sm_count * 8;
	const bool adapt = st->mode == TSDRGPU_STACK_ADAPT, robust = st->mode == TSDRGPU_STACK_ROBUST;
	const bool track = st->mode == TSDRGPU_STACK_TRACK || robust;
	const int tx = (int) st_tiles_x(w), ty = (int) st_tiles_y(h), ntiles = tx * ty;
	const unsigned tgrid = (unsigned) (ntiles + ST_THREADS - 1) / ST_THREADS;
	for (int f = 0; f < nframes; f++) {
		const float *F = in + (size_t) f * n;
		float *O = out + (size_t) f * n;
		tsdrgpu_stack_record_t *rec = st->d_rec.ptr + f;
		if (st->m == 0) {
			KL(ctx, "st_restart", stream, st_restart<<<grid, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, O, n, off, rec));
			if (adapt || track) KL(ctx, "st_tile_init", stream, st_tile_init<<<tgrid, ST_THREADS, 0, stream>>>(st->d_tiles.ptr, ntiles));
			if (track) KL(ctx, "st_track_init", stream, st_track_init<<<grid, ST_THREADS, 0, stream>>>(st->d_cnt.ptr, n, st->d_track.ptr, ntiles));
			if (robust) KL(ctx, "st_robust_init", stream, st_robust_init<<<tgrid, ST_THREADS, 0, stream>>>(st->d_robust.ptr, ntiles, st->d_rframe.ptr));
		} else {
			const int m2 = st->m >= 2;
			const long long k = st->m + 1 < st->depth ? st->m + 1 : st->depth;
			const float wn = (float) (1.0 / (double) k), wo = (float) (1.0 - 1.0 / (double) k);
			KL(ctx, "st_score", stream, st_score<<<tiles, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, n, w, st->rx, st->ry, m2, off, st->d_scores.ptr));
			KL(ctx, "st_pick", stream, st_pick<<<1, 1024, 0, stream>>>(st->d_scores.ptr, w, st->rx, st->ry, m2, off, rec));
			if (track) {
				KL(ctx, "st_tile_sums", stream, st_tile_sums<<<ntiles, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, n, w, h, tx, off, st->d_tiles.ptr));
				KL(ctx, "st_track_search", stream, st_track_search<<<ntiles, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, n, w, h, tx, off,
				                                                                                   st->d_tiles.ptr, st->d_track.ptr));
				if (robust) {
					KL(ctx, "st_robust_decide", stream, st_robust_decide<<<1, RB_THREADS, 0, stream>>>(st->d_tiles.ptr, st->d_track.ptr, st->d_robust.ptr,
					                                                                                 tx, ty, off, st->d_rframe.ptr, rec));
					KL(ctx, "st_robust_blend", stream, st_robust_blend<<<grid, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, st->d_acc2.ptr, st->d_cnt.ptr,
					                                                                                  st->d_cnt2.ptr, O, n, w, h, tx, st->depth, st->d_track.ptr,
					                                                                                  st->d_robust.ptr, st->d_rframe.ptr, off));
				} else {
					KL(ctx, "st_track_decide", stream, st_track_decide<<<tgrid, ST_THREADS, 0, stream>>>(st->d_tiles.ptr, st->d_track.ptr, tx, ty, rec));
					KL(ctx, "st_track_blend", stream, st_track_blend<<<grid, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, st->d_acc2.ptr, st->d_cnt.ptr,
					                                                                                st->d_cnt2.ptr, O, n, w, h, tx, st->depth, st->d_track.ptr, off));
				}
				st_swap(st->d_acc, st->d_acc2);                  // host-side: the next launches on this stream read the new planes
				st_swap(st->d_cnt, st->d_cnt2);
			} else if (adapt) {
				KL(ctx, "st_tile_sums", stream, st_tile_sums<<<ntiles, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, n, w, h, tx, off, st->d_tiles.ptr));
				KL(ctx, "st_decide", stream, st_decide<<<tgrid, ST_THREADS, 0, stream>>>(st->d_tiles.ptr, tx, ty, st->depth, rec));
				KL(ctx, "st_blend_tiles", stream, st_blend_tiles<<<grid, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, O, n, (unsigned) w, tx, st->d_tiles.ptr, off));
			} else KL(ctx, "st_blend", stream, st_blend<<<grid, ST_THREADS, 0, stream>>>(F, st->d_acc.ptr, O, n, wo, wn, off));
		}
		if (st->m <= st->depth) st->m++;                     // past N only "m >= 2" and k = N matter
	}
	st->last_frames = nframes;
	return TSDRGPU_OK;
}

// a new mode or window restarts the accumulator; the same settings again leave it running
int stack_set(StackState *st, int mode, int depth, int rx, int ry) {
	if (mode == TSDRGPU_STACK_OFF) depth = rx = ry = 0;
	if (mode != st->mode || depth != st->depth || rx != st->rx || ry != st->ry) st->m = 0;
	st->mode = mode; st->depth = depth; st->rx = rx; st->ry = ry;
	return TSDRGPU_OK;
}

struct tsdrgpu_stack {
	tsdrgpu_ctx_t *ctx;
	StackState st;
};

extern "C" {

int tsdrgpu_stack_create(tsdrgpu_ctx_t *ctx, tsdrgpu_stack_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_stack *s = new tsdrgpu_stack();                // value-initialised: off, m = 0, no buffers
	s->ctx = ctx;
	*out = s;
	return TSDRGPU_OK;
}

void tsdrgpu_stack_destroy(tsdrgpu_stack_t *s) {
	if (!s) return;
	cudaSetDevice(s->ctx->device);
	cudaDeviceSynchronize();
	delete s;
}

int tsdrgpu_stack_reset(tsdrgpu_stack_t *s) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	s->st.m = 0;
	return TSDRGPU_OK;
}

int tsdrgpu_stack_set(tsdrgpu_stack_t *s, int mode, int depth, int rx, int ry) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	ARG_TRY(s->ctx, stack_ok(mode, depth, rx, ry));
	return stack_set(&s->st, mode, depth, rx, ry);
}

int tsdrgpu_stack_vectors(tsdrgpu_stack_t *s, int32_t *h_v, int ntiles) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	tsdrgpu_ctx_t *ctx = s->ctx;
	BIND(ctx);
	const StackState &st = s->st;
	ARG_TRY(ctx, h_v && (st.mode == TSDRGPU_STACK_TRACK || st.mode == TSDRGPU_STACK_ROBUST) && st.m > 0 && st.d_track.ptr);
	ARG_TRY(ctx, (size_t) ntiles == st_tiles_x(st.w) * st_tiles_y(st.h));
	CU_TRY(ctx, cudaDeviceSynchronize());
	CU_TRY(ctx, cudaMemcpy2D(h_v, 2 * sizeof(int32_t), &st.d_track.ptr[0].bx, sizeof(StackTrack), 2 * sizeof(int32_t), (size_t) ntiles,
	                         cudaMemcpyDeviceToHost));
	return TSDRGPU_OK;
}

int tsdrgpu_stack_robust_counts(tsdrgpu_stack_t *s, int32_t *held_tiles, uint64_t *gated_pixels, int32_t *frame_held) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	tsdrgpu_ctx_t *ctx = s->ctx;
	BIND(ctx);
	const StackState &st = s->st;
	ARG_TRY(ctx, held_tiles && gated_pixels && frame_held && st.mode == TSDRGPU_STACK_ROBUST && st.m > 0 && st.d_rframe.ptr);
	StackRobustFrame fr;
	CU_TRY(ctx, cudaDeviceSynchronize());
	CU_TRY(ctx, cudaMemcpy(&fr, st.d_rframe.ptr, sizeof fr, cudaMemcpyDeviceToHost));
	*held_tiles = fr.held; *gated_pixels = fr.gated; *frame_held = fr.hold;
	return TSDRGPU_OK;
}

int tsdrgpu_stack_run(tsdrgpu_stack_t *s, void *stream_, const float *d_in, float *d_out, int w, int h, int nframes,
                      tsdrgpu_stack_record_t *h_records_pinned) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, s != NULL);
	tsdrgpu_ctx_t *ctx = s->ctx;
	BIND(ctx);
	if (nframes == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in && d_out && nframes > 0 && w > 0 && h > 0 && (size_t) w * h <= TSDRGPU_MAX_FRAME_PIXELS);
	ARG_TRY(ctx, ((((uintptr_t) d_in) | ((uintptr_t) d_out)) & 3) == 0);
	const uintptr_t bytes = (uintptr_t) sizeof(float) * w * h * nframes;
	ARG_TRY(ctx, (uintptr_t) d_out >= (uintptr_t) d_in + bytes || (uintptr_t) d_in >= (uintptr_t) d_out + bytes);
	cudaStream_t stream = (cudaStream_t) stream_;
	if (s->st.mode == TSDRGPU_STACK_OFF) return fs_copy_async(ctx, stream, d_in, d_out, (size_t) nframes * w * h);
	int rc = stack_reserve(ctx, &s->st, nframes, w, h);
	if (rc == TSDRGPU_OK) rc = stack_run(ctx, &s->st, stream, d_in, d_out, nframes, w, h);
	if (rc == TSDRGPU_OK && h_records_pinned)
		CU_TRY(ctx, cudaMemcpyAsync(h_records_pinned, s->st.d_rec.ptr, sizeof(tsdrgpu_stack_record_t) * nframes, cudaMemcpyDeviceToHost, stream));
	return rc;
}

}  // extern "C"
