// common.cuh -- shared plumbing of libtsdrgpu (context, error handling, exact-arithmetic helpers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <deque>
#include <mutex>
#include <vector>

#include "../../include/tsdrgpu.h"
#include "devbuf.h"

// a twiddle table of the transforms (fft.cu): which one, and its device copy
struct FftTableKey { int kind; long long a, b, c; double eps; };
struct FftTable { FftTableKey key; DeviceBuf<float2> d; };

struct tsdrgpu_ctx {
	int device;
	int sm_count;
	char err[512];
	uint64_t launches;
	// scratch owned by the context (grown on demand, reused across calls on the same stream)
	DeviceBuf<unsigned char> scratch[4];
	PinnedBuf<unsigned char> pinned;      // small pinned staging area for descriptor uploads / scalar read-backs
	std::mutex mu;                        // guards the profiling records and the FFT tables
	// the transforms' twiddle tables, built on first use (a deque never moves them: DeviceBuf cannot move), and whether the
	// pass kernels' shared-memory limit has been raised
	std::deque<FftTable> fft_tables; bool fft_attrs_set = false;
	// optional per-kernel timing (bench.py's roofline): CUDA events on the launching stream around named launches
	bool profiling;
	struct ProfRec { int id; cudaEvent_t a, b; };
	std::vector<ProfRec> prof_recs;
	std::vector<cudaEvent_t> prof_pool;
	char prof_names[48][48];
	int prof_nnames;
};

void tsdrgpu_prof_begin(tsdrgpu_ctx_t *ctx, const char *name, cudaStream_t stream);
void tsdrgpu_prof_end(tsdrgpu_ctx_t *ctx, cudaStream_t stream);
// wrap a kernel launch: KL(ctx, "name", stream, kernel<<<...>>>(...));
#define KL(ctx, name, stream, ...) do { if ((ctx)->profiling) tsdrgpu_prof_begin((ctx), (name), (stream)); __VA_ARGS__; \
	if ((ctx)->profiling) tsdrgpu_prof_end((ctx), (stream)); LAUNCH_CHECK(ctx); } while (0)

extern thread_local char g_tsdrgpu_err[512];

static inline int tsdrgpu_fail(tsdrgpu_ctx_t *ctx, int code, const char *what, cudaError_t e, const char *file, int line) {
	char *dst = ctx ? ctx->err : g_tsdrgpu_err;
	if (e != cudaSuccess) { snprintf(dst, 512, "%s: %s (%s:%d)", what, cudaGetErrorString(e), file, line); cudaGetLastError(); /* reported here: do not let it resurface at the next launch check */ }
	else snprintf(dst, 512, "%s (%s:%d)", what, file, line);
	return code;
}

#define CU_TRY(ctx, expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
	return tsdrgpu_fail((ctx), TSDRGPU_ECUDA, #expr, e_, __FILE__, __LINE__); } while (0)
#define ARG_TRY(ctx, cond) do { if (!(cond)) \
	return tsdrgpu_fail((ctx), TSDRGPU_EINVAL, "invalid argument: " #cond, cudaSuccess, __FILE__, __LINE__); } while (0)
#define LAUNCH_CHECK(ctx) do { (ctx)->launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) \
	return tsdrgpu_fail((ctx), TSDRGPU_ECUDA, "kernel launch", e_, __FILE__, __LINE__); } while (0)

static inline int tsdrgpu_bind(tsdrgpu_ctx_t *ctx) {
	if (!ctx) return tsdrgpu_fail(NULL, TSDRGPU_EINVAL, "null context", cudaSuccess, __FILE__, __LINE__);
	CU_TRY(ctx, cudaSetDevice(ctx->device));
	return TSDRGPU_OK;
}
#define BIND(ctx) do { int rc_ = tsdrgpu_bind(ctx); if (rc_ != TSDRGPU_OK) return rc_; } while (0)

// grow-only scratch slot
int tsdrgpu_scratch(tsdrgpu_ctx_t *ctx, int slot, size_t bytes, void **out);
int tsdrgpu_pinned(tsdrgpu_ctx_t *ctx, size_t bytes, void **out);

// ---- exact single-precision magnitude: fl(sqrt(fl(fl(I*I) + fl(Q*Q)))), no contraction (TSDRLibrary.c:260)
__device__ __forceinline__ float mag_exact(float i, float q) {
	return __fsqrt_rn(__fadd_rn(__fmul_rn(i, i), __fmul_rn(q, q)));
}

__device__ __forceinline__ float2 ldg_stream_f2(const float2 *p) {
	float2 v;
	asm("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
	return v;
}
__device__ __forceinline__ float4 ldg_stream_f4(const float4 *p) {
	float4 v;
	asm("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
	             : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
	return v;
}
__device__ __forceinline__ float ldg_stream_f1(const float *p) {
	float v;
	asm("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
	return v;
}

// ---- pixels of the frame stage
__device__ __forceinline__ bool px_is_marker(float v) { return v > 250.0f || v < -250.0f; }   // dsp.c:57
// the pixels the clip auto-gain, CLAHE and NLM work on (tsdrgpu.h): neither a marker nor NaN
__device__ __forceinline__ bool px_valid(float v) { return !px_is_marker(v) && v == v; }

// n floats from src cut on the ADDRESS into a scalar head up to the next 16-byte boundary, a float4 body and a scalar tail
// from tail0: frames of an odd number of pixels start at any of the four 4-byte phases
struct F4Split {
	size_t head, nbody, tail0, n;
	__device__ F4Split(const float *src, size_t count) : n(count) {
		head = (size_t) ((4u - (unsigned) ((reinterpret_cast<unsigned long long>(src) >> 2) & 3ull)) & 3u);
		if (head > n) head = n;
		nbody = (n - head) >> 2; tail0 = head + (nbody << 2);
	}
};

// ---- internal entry points shared between translation units (fft.cu owns the transforms, framestage.cu fs_copy)
constexpr unsigned TSDRGPU_ARGMAX_PARTS = 1024;
int tsdrgpu_fft_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, float2 *data, unsigned long long n_pow2, int inverse);
int tsdrgpu_fft_oop_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, float2 *out, unsigned long long n_pow2, int inverse);
int tsdrgpu_fft_batch_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, long long in_bs, float2 *out, long long out_bs,
                               float2 *scratch, unsigned long long n_pow2, unsigned batch, int inverse);
int tsdrgpu_fft_exact_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *in, float2 *out, float2 *scratch, unsigned long long n_pow2,
                               int inverse);
bool tsdrgpu_fft_true_dft();          // TSDRGPU_FFT_TRUE_DFT: the exact DFT's stage angles instead of the reference's
int tsdrgpu_argmax_mag_internal(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float2 *x, unsigned n, void *d_part, int *d_result);
int fs_copy_async(tsdrgpu_ctx_t *ctx, cudaStream_t stream, const float *in, float *out, size_t total);
// stack.cu: drift-registered frame averaging.  m (frames since the last restart) is counted on the host, as every launch knows it;
// the offsets o1, o2 stay on the device, as does the adaptive mode's per-tile state.
struct StackTile {
	unsigned e;                                  // e_t, the residual level (0xffffffff: none)
	int m;                                       // m_t, counted up to N
	unsigned r;                                  // this frame's floor(16 D_t / C_t)
	int flag;                                    // this frame: 0 no measured pixel (C_t = 0), 1 measured, 2 changed
	float wo, wn;                                // this frame's blend weights
};
struct StackTrack {                              // track: one per tile of the accumulator, this frame's
	int vx, vy;                                  // search: v* ((0, 0): no admissible candidate)
	unsigned d, c;                               // search: D(v*), C(v*)
	int moved;                                   // search: moved_t (meaningful where the tile's flag is 2)
	int bx, by;                                  // decide: the move the blend takes, (0, 0) unless moved and not restarting
	int restart;                                 // decide: the tile restarts
};
struct StackRobust {                             // robust: one per tile of the accumulator
	int pend;                                    // pend_t: the tile was new in the last frame
	int confirmed;                               // decide: confirmed_t of this frame
	int held;                                    // decide: the tile is held this frame
	unsigned gate_e;                             // decide: e_t before this frame's 6c where the gate applies, else 0xffffffff
};
struct StackRobustFrame {                        // robust: the frame in flight
	double b;                                    // step 3's prediction b of the next frame
	int held, hold;                              // held tiles, and 1 on a glitch frame
	unsigned long long gated;                    // gated pixels
};
struct StackState {
	int mode, depth, rx, ry;                     // TSDRGPU_STACK_* and its parameters (N, rx, ry)
	int w, h;                                    // the accumulator's geometry
	int m;                                       // frames since the last restart, counted up to depth + 1
	int last_frames;                             // frames of the last run (its records are in d_rec)
	DeviceBuf<float> d_acc;                      // A
	DeviceBuf<double> d_off;                     // o1, o2
	DeviceBuf<unsigned long long> d_scores;      // S of every candidate of the frame in flight
	DeviceBuf<tsdrgpu_stack_record_t> d_rec;     // the records of a batch
	DeviceBuf<StackTile> d_tiles;                // adapt, track, robust: one per tile of the accumulator
	DeviceBuf<float> d_acc2;                     // track, robust: A', swapped with d_acc after every frame
	DeviceBuf<uint16_t> d_cnt, d_cnt2;           // track, robust: c and c', swapped likewise
	DeviceBuf<StackTrack> d_track;               // track, robust: one per tile of the accumulator
	DeviceBuf<StackRobust> d_robust;             // robust: one per tile of the accumulator
	DeviceBuf<StackRobustFrame> d_rframe;        // robust: one
};
int stack_reserve(tsdrgpu_ctx_t *ctx, StackState *st, int nframes, int w, int h);
int stack_run(tsdrgpu_ctx_t *ctx, StackState *st, cudaStream_t stream, const float *in, float *out, int nframes, int w, int h);
int stack_set(StackState *st, int mode, int depth, int rx, int ry);
// enhance.cu: stack, deblur, NLM, then CLAHE on delivered frames, modes and parameters as the frame stage's setters take them
struct EnhanceState {
	int contrast, clip_centi, tx, ty;            // TSDRGPU_CONTRAST_* and its parameters
	int denoise, h_milli, r, p;                  // TSDRGPU_DENOISE_* and its parameters (R, P)
	int deblur, sigma_centi, iters;              // TSDRGPU_DEBLUR_* and its parameters (sigma, I)
	DeviceBuf<unsigned> d_clahe;                 // CLAHE histograms / LUTs of one pass
	DeviceBuf<float> d_nlm;                      // NLM output of a batch
	StackState stack;                            // the stack's mode and state
	DeviceBuf<float> d_stack;                    // stack output of a batch
	DeviceBuf<float> d_deblur;                   // deblur output of a batch
};
// framestage.cu, for the pipeline: restart != 0 restarts the stack; h_records_pinned (may be NULL) receives the stack records of
// the next run, copied on the stream its output becomes valid on
extern "C" int framestage_stack_next(tsdrgpu_framestage_t *fs, int restart, tsdrgpu_stack_record_t *h_records_pinned);
int enhance_reserve(tsdrgpu_ctx_t *ctx, EnhanceState *st, int nframes, int w, int h);
int enhance_run(tsdrgpu_ctx_t *ctx, EnhanceState *st, cudaStream_t stream, float *d_frames, int nframes, int w, int h);
