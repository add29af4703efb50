// channel.cu -- the channel filter: one complex FIR on the interleaved IQ stream before AM demodulation (definition in tsdrgpu.h).
//
// cf_fir is compute-bound: every tap of every output costs 4 FMUL and 4 FADD (no contraction: the products are rounded on their own,
// tsdrgpu.h), 8 T FP32 instructions per pair against 16 bytes of traffic.  So the kernel is built for instruction issue:
//   * the taps sit in shared memory as float2 and are read as broadcasts;
//   * the CTA's input tile plus its T-1 history halo sit in shared memory;
//   * each thread computes CF_K consecutive outputs with a sliding register window: per tap one broadcast load of the tap and one
//     load of the one new input sample, against 8 CF_K FP32 instructions.  CF_K is odd, so the window loads of a half-warp (stride
//     CF_K float2) fall into distinct bank pairs.
// The outputs are staged back through shared memory so that the stores are coalesced.
#include "common.cuh"

namespace {

constexpr int CF_THREADS = 256;
constexpr int CF_K = 9;                                   // outputs per thread
constexpr int CF_P = CF_THREADS * CF_K;                   // outputs per CTA
constexpr int CF_TMAX = TSDRGPU_CHANNEL_MAX_TAPS;
constexpr int CF_HMAX = CF_TMAX - 1;
constexpr unsigned long long CF_MAX_PAIRS = 1ull << 36;

__device__ __forceinline__ constexpr int cf_slot(int k, int t) { return ((k - t) % CF_K + CF_K) % CF_K; }

// x[m_k - t] of output k lives in r[cf_slot(k, t)]: stepping to t + 1 only renames registers, and the one new sample x[m_0 - t - 1]
// overwrites the slot of x[m_{K-1} - t], which no output needs any more.  J counts (t - 1) mod CF_K, so slots are compile-time.
template <bool TAIL>
__device__ __forceinline__ void cf_chunk(int t0, int T, const float2 *__restrict__ s_h, const float2 *__restrict__ s_xb, float2 (&r)[CF_K],
                                         float (&yr)[CF_K], float (&yi)[CF_K]) {
#pragma unroll
	for (int j = 0; j < CF_K; j++) {
		const int t = t0 + j;
		if (TAIL && t >= T) break;
		const float2 h = s_h[t];
#pragma unroll
		for (int k = 0; k < CF_K; k++) {
			const float2 x = r[cf_slot(k, 1 + j)];
			const float pr = __fsub_rn(__fmul_rn(x.x, h.x), __fmul_rn(x.y, h.y));
			const float pi = __fadd_rn(__fmul_rn(x.x, h.y), __fmul_rn(x.y, h.x));
			yr[k] = __fadd_rn(yr[k], pr);
			yi[k] = __fadd_rn(yi[k], pi);
		}
		if (!TAIL || t + 1 < T) r[cf_slot(0, 2 + j)] = s_xb[-(t + 1)];
	}
}

__global__ void __launch_bounds__(CF_THREADS) cf_fir(const float2 *__restrict__ in, float2 *__restrict__ out, unsigned long long pairs,
                                                      const float2 *__restrict__ taps, int T, const float2 *__restrict__ hist_in,
                                                      float2 *__restrict__ hist_out) {
	__shared__ float2 s_x[CF_P + CF_HMAX];
	__shared__ float2 s_h[CF_TMAX];
	const int H = T - 1;
	const long long n0 = (long long) blockIdx.x * CF_P;
	const int nvalid = (int) ((unsigned long long) CF_P < pairs - (unsigned long long) n0 ? CF_P : pairs - (unsigned long long) n0);
	for (int i = threadIdx.x; i < T; i += CF_THREADS) s_h[i] = taps[i];
	// s_x[j] = x[n0 - H + j]; before the run's first pair the history
	for (int j = threadIdx.x; j < nvalid + H; j += CF_THREADS) {
		const long long g = n0 - H + j;
		s_x[j] = g < 0 ? hist_in[H + g] : __ldg(in + g);
	}
	// the history the next run reads: the last H pairs of everything seen so far
	if (blockIdx.x == 0)
		for (int i = threadIdx.x; i < H; i += CF_THREADS) {
			const long long g = (long long) pairs - H + i;
			hist_out[i] = g < 0 ? hist_in[H + g] : __ldg(in + g);
		}
	__syncthreads();

	// thread outputs m = tid K + k (tile-relative); x[m - t] is s_x[m + H - t]
	const float2 *s_xb = s_x + threadIdx.x * CF_K + H;
	float2 r[CF_K];
	float yr[CF_K], yi[CF_K];
	{                                                         // t = 0 sets the sums: yr = pr (0 + pr would turn -0 into +0)
		const float2 h = s_h[0];
#pragma unroll
		for (int k = 0; k < CF_K; k++) {
			const float2 x = s_xb[k];
			r[cf_slot(k, 0)] = x;
			yr[k] = __fsub_rn(__fmul_rn(x.x, h.x), __fmul_rn(x.y, h.y));
			yi[k] = __fadd_rn(__fmul_rn(x.x, h.y), __fmul_rn(x.y, h.x));
		}
		r[cf_slot(0, 1)] = s_xb[-1];                          // T >= 9: tap 1 exists
	}
	// whole chunks while the chunk's last tap is not the last one (that tap loads no new sample: s_xb[-T] lies before the tile)
	int t0 = 1;
	for (; t0 + CF_K < T; t0 += CF_K) cf_chunk<false>(t0, T, s_h, s_xb, r, yr, yi);
	cf_chunk<true>(t0, T, s_h, s_xb, r, yr, yi);

	__syncthreads();                                          // everyone is done reading the tile: stage the outputs there
#pragma unroll
	for (int k = 0; k < CF_K; k++) s_x[threadIdx.x * CF_K + k] = make_float2(yr[k], yi[k]);
	__syncthreads();
	for (int j = threadIdx.x; j < nvalid; j += CF_THREADS) out[n0 + j] = s_x[j];
}

}  // namespace

struct tsdrgpu_chanfilt {
	tsdrgpu_ctx_t *ctx;
	int T;                                    // 0: no spec set yet
	float h_taps[2 * CF_TMAX];                // the taps of the current spec (host copy)
	DeviceBuf<float2> d_taps; int taps_dirty; // device copy, uploaded by the next run when dirty
	DeviceBuf<float2> d_hist[2]; int hist_cur; int hist_zero;      // last T-1 pairs: runs read d_hist[hist_cur], write the other
};

extern "C" {

static int create_handles(tsdrgpu_chanfilt *f) {
	CU_TRY(f->ctx, f->d_taps.assign(CF_TMAX));
	for (DeviceBuf<float2> &h : f->d_hist) {
		CU_TRY(f->ctx, h.assign(CF_HMAX));
		CU_TRY(f->ctx, cudaMemset(h.ptr, 0, sizeof(float2) * CF_HMAX));
	}
	return TSDRGPU_OK;
}

int tsdrgpu_chanfilt_create(tsdrgpu_ctx_t *ctx, tsdrgpu_chanfilt_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	tsdrgpu_chanfilt *f = new tsdrgpu_chanfilt();      // value-initialised: every field not set here starts at zero
	f->ctx = ctx;
	const int rc = create_handles(f);
	if (rc) { delete f; return rc; }                   // no stream or event of its own: its buffers go with it
	*out = f;
	return TSDRGPU_OK;
}

void tsdrgpu_chanfilt_destroy(tsdrgpu_chanfilt_t *f) {
	if (!f) return;
	cudaSetDevice(f->ctx->device);
	cudaDeviceSynchronize();
	delete f;
}

int tsdrgpu_chanfilt_reset(tsdrgpu_chanfilt_t *f, void *stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	BIND(f->ctx);
	CU_TRY(f->ctx, cudaMemsetAsync(f->d_hist[f->hist_cur].ptr, 0, sizeof(float2) * CF_HMAX, (cudaStream_t) stream));
	f->hist_zero = 0;
	return TSDRGPU_OK;
}

int tsdrgpu_chanfilt_set(tsdrgpu_chanfilt_t *f, const tsdrgpu_channel_t *spec, uint32_t fs) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	float h[2 * CF_TMAX];
	int T = 0;
	if (!spec || spec->taps == 0 || tsdrgpu_channel_taps(spec, fs, h, &T) != TSDRGPU_OK)
		return tsdrgpu_fail(f->ctx, TSDRGPU_EINVAL, "invalid channel filter spec or sample rate (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
	if (T == f->T && memcmp(h, f->h_taps, sizeof(float) * 2 * T) == 0) return TSDRGPU_OK;      // same taps: the history stays
	memcpy(f->h_taps, h, sizeof(float) * 2 * T);
	f->T = T; f->taps_dirty = 1; f->hist_zero = 1;
	return TSDRGPU_OK;
}

int tsdrgpu_chanfilt_run(tsdrgpu_chanfilt_t *f, void *stream_, const float *d_in, uint64_t pairs, float *d_out) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, f != NULL);
	tsdrgpu_ctx_t *ctx = f->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	if (f->T == 0) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "channel filter run before a spec was set", cudaSuccess, __FILE__, __LINE__);
	ARG_TRY(ctx, pairs <= CF_MAX_PAIRS);
	if (pairs == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_in != NULL && d_out != NULL);
	const uintptr_t a = (uintptr_t) d_in, b = (uintptr_t) d_out, bytes = (uintptr_t) (8 * pairs);
	ARG_TRY(ctx, (a & 7u) == 0 && (b & 7u) == 0);
	ARG_TRY(ctx, a + bytes <= b || b + bytes <= a);           // no overlap
	if (f->taps_dirty) {                                      // pageable source: the copy is staged before the call returns
		CU_TRY(ctx, cudaMemcpyAsync(f->d_taps.ptr, f->h_taps, sizeof(float) * 2 * f->T, cudaMemcpyHostToDevice, stream));
		f->taps_dirty = 0;
	}
	if (f->hist_zero) { CU_TRY(ctx, cudaMemsetAsync(f->d_hist[f->hist_cur].ptr, 0, sizeof(float2) * CF_HMAX, stream)); f->hist_zero = 0; }
	const unsigned grid = (unsigned) ((pairs + CF_P - 1) / CF_P);
	KL(ctx, "cf_fir", stream, cf_fir<<<grid, CF_THREADS, 0, stream>>>(reinterpret_cast<const float2 *>(d_in), reinterpret_cast<float2 *>(d_out), pairs,
	                                                              f->d_taps.ptr, f->T, f->d_hist[f->hist_cur].ptr, f->d_hist[f->hist_cur ^ 1].ptr));
	f->hist_cur ^= 1;
	return TSDRGPU_OK;
}

}  // extern "C"
