// superb_mgpu.cu -- a22 with one hop per GPU: superb_ondataready (superbandwidth.c:121-152) sharded over H GPUs of one node.
//
// The reference aligns H hops against hop 0 (H-1 cross-correlations), transforms each hop, concatenates the spectra and runs
// one H*N-point inverse fft_perform: bit reversal, then radix-2 decimation-in-time stages 0 .. log2(HN)-1, each with ITS OWN
// slightly wrong angle (fft.c:161; tsdrgpu_fft_reference_eps: 2.6e-5 relative at stage 22).  The sharding follows exactly that
// structure, so the result tracks the reference as closely as the one-GPU path does (1e-6 of the peak), not merely the true DFT:
// after bit reversal, block rev(t) of the big array holds the inputs k = H u + t, and the first log2 N stages turn it into the
// N-point transform of that decimated sub-sequence; the last log2 H stages combine the H blocks position by position.
//
//   phase 1  local    X_q = FFT_N(hop_q)/N  (fft_perform on the hop, as superbandwidth.c:138-140);
//                     lag_q: P = conj(D_0) D_q, IFFT_nd, grid argmax, D = FFT_nd(first difference of |hop|)/nd.  D_0 comes from the
//                     rank's OWN copy of hop 0 when the caller keeps the alignment reference on every device (d_hop0: the
//                     pipeline copies the first hop to all devices while the later hops are still being recorded; a small
//                     redundant transform instead of a broadcast whose source link carries (H-1) x 8 nd bytes); without it D_0
//                     is READ FROM RANK 0 over NVLink inside the multiply, after an extra barrier (SPEC).
//                     Rotating the hop by lag_q samples (superbandwidth.c:135-137) is a phase ramp on its spectrum: applied
//                     here, locally, while the spectrum is re-ordered for the exchange:
//                         Xp_q[t][u'] = X_q[t + H u'] e^{2 pi i (t + H u') lag_q / N}         -> own window, one run per destination t
//   barrier  LAG      (flags in peer memory; the lag rides along for the record)
//   phase 2  blocks   all-to-all #1: rank t PULLS its run from every rank (contiguous N/H values each) -> B_t[u] = X~[H u + t],
//                     then A_t = IDFT_N(B_t) with the reference's stage angles (the one-GPU transform, unchanged) -> own window
//   barrier  MIX
//   phase 3  combine  all-to-all #2: rank r owns the positions v in [r N/H, (r+1) N/H).  It PULLS A_t[v] from every rank, runs
//                     the reference's last log2 H radix-2 stages across the H blocks (their perturbed angles, twiddles in double),
//                     takes |y| (am_demod, TSDRLibrary.c:244-262: what process() does to superb_run's output) and PUSHES
//                     y[v + N c], c = 0..H-1, as float32 into the ROOT's window -- already time-contiguous, in runs of N/H
//                     samples (SURVEY 8e option B: 4 B per sample)
//   barrier  RES      (root only waits)
//   phase 4  root     one device-to-device copy of the stream to where the caller wants it -> decimator -> frames
//   NVLink traffic per rank: 2 (H-1)/H N complex in (an all-gather would be (H-1) N), the root takes (H-1) N floats.
//
// Synchronisation between ranks never touches the host and never calls a collective library: every window starts with a
// small header of epoch-valued flags; a one-CTA kernel between phases stores this rank's flag into every peer (release,
// system scope, after the kernels before it have completed in stream order) and spins (acquire, bounded by a timeout that
// raises a status word instead of hanging the GPU) until every peer's flag for the phase carries this stitch's epoch.  The
// same kernels run whether the peers are other processes (windows mapped with CUDA IPC: torchrun, one process per GPU) or
// other devices of this process (cudaDeviceEnablePeerAccess: the C host library with TSDR_CUDA_DEVICES).
//
// Parity: lags exact (same float operations as the one-GPU path up to the transform, first-maximum argmax); samples are
// tolerance-based like every FFT result here: within float32 rounding units of a float64 model of this dataflow, and of
// superb_ondataready + am_demod's model within that plus a pinned deviation (tests/test_superb_sweep.py, DESIGN.md section 6).
#include "common.cuh"
#include <math.h>
#include <stdlib.h>

namespace {

constexpr int SBM_MAX_RANKS = 16;
enum { PH_SPEC = 0, PH_LAG = 1, PH_MIX = 2, PH_RES = 3, PH_COUNT = 4 };

struct WinHeader {                                   // first 4 KB of every window
	unsigned flag[PH_COUNT][SBM_MAX_RANKS];          // flag[phase][src] = epoch of the last stitch in which src finished `phase`
	int lag[SBM_MAX_RANKS];                          // lag[q] in complex samples, stored by rank q before its PH_LAG flag
	unsigned status;                                 // != 0: a wait timed out (phase + 1 in the low byte, the missing rank above it)
	unsigned pad[1024 - PH_COUNT * SBM_MAX_RANKS - SBM_MAX_RANKS - 1];
};
static_assert(sizeof(WinHeader) == 4096, "window header layout");

struct Peers { unsigned char *win[SBM_MAX_RANKS]; };

__device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p) { unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ float2 ld_peer_f2(const float2 *p) { float2 v; asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p)); return v; }
__device__ __forceinline__ float4 ld_peer_f4(const float4 *p) { float4 v; asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p)); return v; }

// One CTA, one thread per rank.  signal: tell every rank in `to_mask` that this rank has finished `phase` of stitch `epoch`
// (everything the stream ran before this kernel is complete; the fence + release store publish it system-wide).  wait: spin
// until every rank in `from_mask` has said the same to us.  `lag_value` (phase LAG) rides along with the flag.
__global__ void __launch_bounds__(32) sbm_sync(Peers peers, int nranks, int rank, int phase, unsigned epoch, unsigned to_mask, unsigned from_mask,
                                               const int *lag_value, long long timeout_cycles) {
	const int q = threadIdx.x;
	if (q >= nranks) return;
	WinHeader *mine = reinterpret_cast<WinHeader *>(peers.win[rank]);
	if (to_mask & (1u << q)) {
		WinHeader *theirs = reinterpret_cast<WinHeader *>(peers.win[q]);
		if (lag_value) *reinterpret_cast<volatile int *>(&theirs->lag[rank]) = *lag_value;
		__threadfence_system();
		st_release_sys(&theirs->flag[phase][rank], epoch);
	}
	if (from_mask & (1u << q)) {
		const long long t0 = clock64();
		while (ld_acquire_sys(&mine->flag[phase][q]) != epoch) {
			if (clock64() - t0 > timeout_cycles) { atomicCAS(&mine->status, 0u, (unsigned) (phase + 1) | ((unsigned) q << 8)); break; }
			__nanosleep(200);
		}
	}
}

// first difference of magnitudes (superbandwidth.c:67-81), out of place
__global__ void __launch_bounds__(256) sbm_abs_diff(const float2 *__restrict__ src, float2 *__restrict__ dst, unsigned n) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float2 v = src[i];
		const float cur = mag_exact(v.x, v.y);
		float prev;
		if (i == 0) prev = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));    // seed without the square root (superbandwidth.c:70)
		else { const float2 u = src[i - 1]; prev = mag_exact(u.x, u.y); }
		dst[i] = make_float2(__fsub_rn(cur, prev), 0.0f);
	}
}

// the same for two signals in one launch (blockIdx.y picks the signal): dst = [ diff(src0) | diff(src1) ], n each
__global__ void __launch_bounds__(256) sbm_abs_diff2(const float2 *__restrict__ src0, const float2 *__restrict__ src1, float2 *__restrict__ dst, unsigned n) {
	const float2 *src = blockIdx.y ? src1 : src0;
	float2 *d = dst + (size_t) blockIdx.y * n;
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float2 v = src[i];
		const float cur = mag_exact(v.x, v.y);
		float prev;
		if (i == 0) prev = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
		else { const float2 u = src[i - 1]; prev = mag_exact(u.x, u.y); }
		d[i] = make_float2(__fsub_rn(cur, prev), 0.0f);
	}
}

// P = (aI bI + aQ bQ, aI bQ - aQ bI) (fft.c:80-89) with a = D_0 in RANK 0's window (NVLink loads), b = D_q local
__global__ void __launch_bounds__(256) sbm_xcorr_pull(const float4 *__restrict__ d0_remote, const float4 *__restrict__ dq, float4 *__restrict__ out, unsigned n2 /* pairs of complex */) {
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) {
		const float4 a = ld_peer_f4(d0_remote + i), b = __ldg(dq + i);
		float4 r;
		r.x = __fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); r.y = __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x));
		r.z = __fadd_rn(__fmul_rn(a.z, b.z), __fmul_rn(a.w, b.w)); r.w = __fsub_rn(__fmul_rn(a.z, b.w), __fmul_rn(a.w, b.z));
		out[i] = r;
	}
}

// phase 1 epilogue: Xp[t][u'] = X[t + H u'] e^{2 pi i (t + H u') lag / N} -- the spectrum re-ordered so that what rank t will
// pull is one contiguous run, with this hop's alignment ramp applied (the argument is reduced exactly in integers)
__global__ void __launch_bounds__(256) sbm_permute_ramp(const float2 *__restrict__ X, float2 *__restrict__ Xp, unsigned n, int log2H, const int *__restrict__ lag_) {
	const unsigned lag = (unsigned) *lag_, per = n >> log2H;
	const float inv_n = 1.0f / (float) n;             // n is a power of two: exact
	for (unsigned o = blockIdx.x * blockDim.x + threadIdx.x; o < n; o += gridDim.x * blockDim.x) {
		const unsigned t = o / per, up = o - t * per, m = t + (up << log2H);
		const float2 x = __ldg(X + m);
		const unsigned e = (unsigned) (((unsigned long long) m * (unsigned long long) lag) & (unsigned long long) (n - 1));
		float sn, cs;
		sincospif(2.0f * ((float) e * inv_n), &sn, &cs);
		Xp[o] = make_float2(x.x * cs - x.y * sn, x.x * sn + x.y * cs);
	}
}

// phase 2: B_t = [ run t of rank 0 | run t of rank 1 | ... ]  (N/H complex from each peer, 16-byte loads over NVLink)
struct PullArgs { Peers peers; size_t off_xp; int H, rank; unsigned per; };
__global__ void __launch_bounds__(256) sbm_pull_blocks(PullArgs A, float4 *__restrict__ dst) {
	const unsigned per2 = A.per >> 1, total = per2 * (unsigned) A.H;       // float4 = two complex values
	for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
		const unsigned q = i / per2, j = i - q * per2;
		const float4 *src = reinterpret_cast<const float4 *>(A.peers.win[q] + A.off_xp) + (size_t) A.rank * per2 + j;
		dst[i] = ld_peer_f4(src);
	}
}

// phase 3: the reference's last log2 H radix-2 decimation-in-time stages across the H blocks, for this rank's positions v.
// Block b of the big array is A_{rev(b)}; at stage s (fft_perform's stage l = log2 N + s) blocks b and b + 2^s (bit s of b clear)
// meet with the twiddle exp(+i pi (v + N beta) / (N 2^s) (1 + eps_l)), beta = b mod 2^s.  Output block c is y[v + N c].
struct FinalArgs { Peers peers; size_t off_a, off_r; int H, log2H, rank, root; unsigned n; double eps[4]; };
template <int H>
__global__ void __launch_bounds__(256) sbm_final(FinalArgs A) {
	constexpr int LOG2H = (H == 2) ? 1 : (H == 4) ? 2 : 3;
	__shared__ double2 cfac[LOG2H][H / 2];            // exp(+i pi beta / 2^s (1 + eps_s)), beta < 2^s
	if (threadIdx.x < LOG2H * (H / 2)) {
		const int sidx = threadIdx.x / (H / 2), beta = threadIdx.x % (H / 2);
		double sn = 0.0, cs = 1.0;
		if (beta < (1 << sidx)) sincospi(((double) beta / (double) (1 << sidx)) * (1.0 + A.eps[sidx]), &sn, &cs);
		cfac[sidx][beta] = make_double2(cs, sn);
	}
	__syncthreads();
	const unsigned n = A.n, per = n / H, v0 = (unsigned) A.rank * per;
	float *stream = reinterpret_cast<float *>(A.peers.win[A.root] + A.off_r);
	for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < per; j += gridDim.x * blockDim.x) {
		const unsigned v = v0 + j;
		float2 a[H];
		#pragma unroll
		for (int b = 0; b < H; b++) {                    // block b <- rank rev(b); H loads in flight
			const int t = (int) (__brev((unsigned) b) >> (32 - LOG2H));
			a[b] = ld_peer_f2(reinterpret_cast<const float2 *>(A.peers.win[t] + A.off_a) + v);
		}
		#pragma unroll
		for (int sidx = 0; sidx < LOG2H; sidx++) {
			double bs, bc;                                // exp(+i pi (v / N) / 2^s (1 + eps))
			sincospi((((double) v / (double) n) / (double) (1 << sidx)) * (1.0 + A.eps[sidx]), &bs, &bc);
			#pragma unroll
			for (int b = 0; b < H; b++) {
				if (b & (1 << sidx)) continue;
				const int beta = b & ((1 << sidx) - 1);
				const double2 cf = cfac[sidx][beta];
				const float wr = (float) (bc * cf.x - bs * cf.y), wi = (float) (bc * cf.y + bs * cf.x);
				const float2 hi = a[b | (1 << sidx)];
				const float2 th = make_float2(hi.x * wr - hi.y * wi, hi.x * wi + hi.y * wr);
				const float2 lo = a[b];
				a[b] = make_float2(lo.x + th.x, lo.y + th.y);
				a[b | (1 << sidx)] = make_float2(lo.x - th.x, lo.y - th.y);
			}
		}
		#pragma unroll
		for (int c = 0; c < H; c++) stream[(size_t) c * n + v] = mag_exact(a[c].x, a[c].y);      // peer stores, coalesced over v
	}
}

inline unsigned grid_for(unsigned long long n, int sm_count, int per_sm = 8) {
	const unsigned long long want = (n + 255) / 256, cap = (unsigned long long) sm_count * per_sm;
	return (unsigned) (want < cap ? (want ? want : 1) : cap);
}

}  // namespace

struct tsdrgpu_superb_mgpu {
	tsdrgpu_ctx_t *ctx;
	int H, log2H, rank, root;
	unsigned n_max;                                   // largest transform length the window was sized for
	DeviceBuf<unsigned char> win;
	size_t off_d, off_x, off_v, off_r;                // byte offsets in the window: D (difference spectrum), Xp (re-ordered spectrum), A (block transform), the root's stream
	Peers peers; int connected; int ipc_opened[SBM_MAX_RANKS];
	DeviceBuf<float2> d_work, d_p, d_x; DeviceBuf<unsigned char> d_part; DeviceBuf<int> d_lag;   // local temporaries (d_work, d_dd: 2 n_max complex -- the two difference signals / spectra side by side)
	DeviceBuf<float2> d_dd, d_side;                   // d_side: the side stream's transform scratch
	cudaStream_t s_side; cudaEvent_t ev_fork, ev_join; // the hop's own spectrum runs beside the lag search
	unsigned epoch; unsigned last_n;
	unsigned prep_n, prep_nd;                         // transform sizes whose kernels and twiddle tables are known to be resident
	long long timeout_cycles;
};

extern "C" {

// a group member whole or half built: the peers' windows are unmapped before its own window goes, then its stream and events
// (null ones are skipped) and the object; its buffers go with it
static void release(tsdrgpu_superb_mgpu *g) {
	for (int q = 0; q < g->H; q++) if (g->ipc_opened[q] && g->peers.win[q]) cudaIpcCloseMemHandle(g->peers.win[q]);
	if (g->s_side) cudaStreamDestroy(g->s_side);
	if (g->ev_fork) cudaEventDestroy(g->ev_fork);
	if (g->ev_join) cudaEventDestroy(g->ev_join);
	delete g;
}

static int create_handles(tsdrgpu_superb_mgpu *g) {
	tsdrgpu_ctx_t *ctx = g->ctx;
	const size_t n = g->n_max;
	CU_TRY(ctx, g->win.assign(g->off_r + sizeof(float) * n * (size_t) g->H));
	CU_TRY(ctx, cudaMemset(g->win.ptr, 0, sizeof(WinHeader)));
	CU_TRY(ctx, g->d_work.assign(2 * n));
	CU_TRY(ctx, g->d_dd.assign(2 * n));
	CU_TRY(ctx, g->d_side.assign(n));
	CU_TRY(ctx, g->d_p.assign(n));
	CU_TRY(ctx, g->d_x.assign(n));
	CU_TRY(ctx, cudaStreamCreateWithFlags(&g->s_side, cudaStreamNonBlocking));
	CU_TRY(ctx, cudaEventCreateWithFlags(&g->ev_fork, cudaEventDisableTiming));
	CU_TRY(ctx, cudaEventCreateWithFlags(&g->ev_join, cudaEventDisableTiming));
	CU_TRY(ctx, g->d_part.assign(8 * TSDRGPU_ARGMAX_PARTS));
	CU_TRY(ctx, g->d_lag.assign(64));
	CU_TRY(ctx, cudaMemset(g->d_lag.ptr, 0, 256));
	// The context's transform scratch, sized now for the largest a stitch runs (the two nd-point difference spectra, nd <= n_max):
	// growing it synchronises the device, and a rank that does so inside sbm_prepare while a peer on the same device already
	// spins on a flag of this stitch waits for that peer, which waits for it (found by a second stitch with a larger nd).
	void *scratch;
	const int rc = tsdrgpu_scratch(ctx, 0, sizeof(float2) * 2 * n, &scratch);
	if (rc) return rc;
	CU_TRY(ctx, cudaDeviceSynchronize());
	return TSDRGPU_OK;
}

int tsdrgpu_superb_mgpu_create(tsdrgpu_ctx_t *ctx, int nranks, int rank, int root, uint32_t max_pairs_per_hop, tsdrgpu_superb_mgpu_t **out) {
	BIND(ctx); ARG_TRY(ctx, out != NULL);
	ARG_TRY(ctx, (nranks == 2 || nranks == 4 || nranks == 8) && rank >= 0 && rank < nranks && root >= 0 && root < nranks && max_pairs_per_hop >= 64);
	tsdrgpu_superb_mgpu *g = new tsdrgpu_superb_mgpu();      // value-initialised: every field not set here starts at zero
	g->ctx = ctx; g->H = nranks; g->rank = rank; g->root = root;
	while ((1 << g->log2H) < nranks) g->log2H++;
	g->n_max = tsdrgpu_fft_getrealsize(max_pairs_per_hop);
	const size_t n = g->n_max;
	g->off_d = sizeof(WinHeader);
	g->off_x = g->off_d + sizeof(float2) * n;         // nd <= n
	g->off_v = g->off_x + sizeof(float2) * n;
	g->off_r = g->off_v + sizeof(float2) * n;
	const int rc = create_handles(g);
	if (rc) { release(g); return rc; }
	g->peers.win[rank] = g->win.ptr;
	const char *to = getenv("TSDRGPU_SBM_TIMEOUT_MS");
	g->timeout_cycles = (long long) ((to ? atof(to) : 15000.0) * 1.9e6);      // ~1.9 GHz SM clock
	*out = g;
	return TSDRGPU_OK;
}

// unmap the peers' windows (one process per GPU: every rank disconnects, THEN every rank destroys -- a barrier of the caller's
// choosing in between -- so that no window is freed while another process still has it mapped)
int tsdrgpu_superb_mgpu_disconnect(tsdrgpu_superb_mgpu_t *g) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL);
	BIND(g->ctx);
	CU_TRY(g->ctx, cudaDeviceSynchronize());
	for (int q = 0; q < g->H; q++) {
		if (g->ipc_opened[q] && g->peers.win[q]) { cudaIpcCloseMemHandle(g->peers.win[q]); g->ipc_opened[q] = 0; }
		if (q != g->rank) g->peers.win[q] = NULL;
	}
	g->connected = 0;
	return TSDRGPU_OK;
}

void tsdrgpu_superb_mgpu_destroy(tsdrgpu_superb_mgpu_t *g) {
	if (!g) return;
	cudaSetDevice(g->ctx->device);
	cudaDeviceSynchronize();
	release(g);
}

int tsdrgpu_superb_mgpu_export(tsdrgpu_superb_mgpu_t *g, uint8_t handle[64]) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL && handle != NULL);
	BIND(g->ctx);
	cudaIpcMemHandle_t h;
	CU_TRY(g->ctx, cudaIpcGetMemHandle(&h, g->win.ptr));
	memcpy(handle, &h, 64);
	return TSDRGPU_OK;
}

// one process per GPU: handles = nranks x 64 bytes, rank-major (entry `rank` is ignored)
int tsdrgpu_superb_mgpu_connect_ipc(tsdrgpu_superb_mgpu_t *g, const uint8_t *handles) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL && handles != NULL);
	tsdrgpu_ctx_t *ctx = g->ctx;
	BIND(ctx);
	for (int q = 0; q < g->H; q++) {
		if (q == g->rank) continue;
		cudaIpcMemHandle_t h;
		memcpy(&h, handles + 64 * q, 64);
		void *p = NULL;
		CU_TRY(ctx, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
		g->peers.win[q] = (unsigned char *) p; g->ipc_opened[q] = 1;
	}
	g->connected = 1;
	return TSDRGPU_OK;
}

// all ranks in this process (one device each): peer access both ways, windows cross-linked
int tsdrgpu_superb_mgpu_connect_local(tsdrgpu_superb_mgpu_t *const *all, int nranks) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, all != NULL && nranks >= 2 && nranks <= SBM_MAX_RANKS);
	for (int r = 0; r < nranks; r++) ARG_TRY((tsdrgpu_ctx_t *) NULL, all[r] != NULL && all[r]->H == nranks && all[r]->rank == r);
	for (int r = 0; r < nranks; r++) {
		tsdrgpu_ctx_t *ctx = all[r]->ctx;
		BIND(ctx);
		for (int q = 0; q < nranks; q++) {
			if (q == r) continue;
			if (all[q]->ctx->device != ctx->device) {
				int can = 0;
				CU_TRY(ctx, cudaDeviceCanAccessPeer(&can, ctx->device, all[q]->ctx->device));
				if (!can) return tsdrgpu_fail(ctx, TSDRGPU_ENODEVICE, "no peer access between the devices of the superbandwidth group", cudaSuccess, __FILE__, __LINE__);
				const cudaError_t e = cudaDeviceEnablePeerAccess(all[q]->ctx->device, 0);
				if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "cudaDeviceEnablePeerAccess", e, __FILE__, __LINE__);
				cudaGetLastError();
			}
			all[r]->peers.win[q] = all[q]->win.ptr;
		}
		all[r]->connected = 1;
	}
	return TSDRGPU_OK;
}

// Everything a stitch launches must already be loaded when the first flag-waiting kernel goes into the stream: with CUDA's lazy
// module loading the FIRST launch of a kernel may synchronise the whole context, and a context that holds a kernel spinning
// on a flag which only work not yet enqueued can raise would never drain (all ranks of one process on one device, or the
// host thread that drives every device in turn).  So the transforms of this size run once on dummy data -- which also builds
// the context's own twiddle tables for them (cudaMalloc + cudaMemcpy) and sizes the scratch -- and the small kernels are touched by name.
}  // extern "C"
template <typename K> static void preload(K kernel) { cudaFuncAttributes a; cudaFuncGetAttributes(&a, kernel); cudaGetLastError(); }
extern "C" {
static int sbm_prepare(tsdrgpu_superb_mgpu *g, cudaStream_t stream, unsigned N, unsigned nd) {
	if (g->prep_n == N && g->prep_nd == nd) return TSDRGPU_OK;
	tsdrgpu_ctx_t *ctx = g->ctx;
	int rc;
	CU_TRY(ctx, cudaMemsetAsync(g->d_work.ptr, 0, sizeof(float2) * N, stream));
	if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, g->d_x.ptr, N, 0))) return rc;
	if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, g->d_p.ptr, nd, 0))) return rc;
	if ((rc = tsdrgpu_fft_internal(ctx, stream, g->d_p.ptr, nd, 1))) return rc;
	if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, g->d_x.ptr, N, 1))) return rc;
	int *tmp_lag = g->d_lag.ptr + 8;
	if ((rc = tsdrgpu_argmax_mag_internal(ctx, stream, g->d_p.ptr, nd, g->d_part.ptr, tmp_lag))) return rc;
	if ((rc = tsdrgpu_fft_batch_internal(ctx, stream, g->d_work.ptr, (long long) nd, g->d_dd.ptr, (long long) nd, NULL, nd, 2, 0))) return rc;
	if ((rc = tsdrgpu_fft_batch_internal(ctx, g->s_side, g->d_work.ptr, 0, g->d_x.ptr, 0, g->d_side.ptr, N, 1, 0))) return rc;
	CU_TRY(ctx, cudaStreamSynchronize(g->s_side));
	preload(sbm_abs_diff2);
	preload(sbm_sync); preload(sbm_abs_diff); preload(sbm_xcorr_pull); preload(sbm_permute_ramp); preload(sbm_pull_blocks);
	switch (g->H) {
	case 2: preload(sbm_final<2>); break;
	case 4: preload(sbm_final<4>); break;
	default: preload(sbm_final<8>); break;
	}
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	g->prep_n = N; g->prep_nd = nd;
	return TSDRGPU_OK;
}

// Rank-local part of one stitch; every rank of the group calls it once per stitch with the same count_pairs / samples_in_frame,
// each on a stream of its own device.  Asynchronous.  The root's d_stream_out receives nranks * N magnitudes (N returned in
// *h_n), time-contiguous: sample H p + s is residue s, element p.  d_stream_out is ignored on the other ranks.
int tsdrgpu_superb_mgpu_stitch(tsdrgpu_superb_mgpu_t *g, void *stream_, const float *d_hop, const float *d_hop0, int count_pairs, int samples_in_frame,
                               float *d_stream_out, uint32_t *h_n) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL);
	tsdrgpu_ctx_t *ctx = g->ctx;
	BIND(ctx);
	ARG_TRY(ctx, g->connected && d_hop != NULL && count_pairs > 0 && samples_in_frame > 0);
	cudaStream_t stream = (cudaStream_t) stream_;
	const unsigned N = tsdrgpu_fft_getrealsize((uint32_t) count_pairs);
	int size = (int) ((2ull * N / (unsigned) samples_in_frame) * (unsigned) samples_in_frame);     // superbandwidth.c:84-86 with bufsize = 2N floats
	ARG_TRY(ctx, size >= 2);
	size = (int) tsdrgpu_fft_getrealsize((uint32_t) size);
	const unsigned nd = (unsigned) size / 2;
	ARG_TRY(ctx, N <= g->n_max && N >= 64 && nd >= 8 && (N % (unsigned) g->H) == 0);
	const int H = g->H, rank = g->rank;
	const unsigned all = (H >= 32) ? 0xffffffffu : ((1u << H) - 1u);
	int rc;
	if ((rc = sbm_prepare(g, stream, N, nd))) return rc;
	const unsigned epoch = ++g->epoch;
	g->last_n = N;
	float2 *D = reinterpret_cast<float2 *>(g->win.ptr + g->off_d), *Xp = reinterpret_cast<float2 *>(g->win.ptr + g->off_x), *Ablk = reinterpret_cast<float2 *>(g->win.ptr + g->off_v);
	// ---- phase 1: this hop's spectrum, this hop's alignment lag, the spectrum re-ordered + ramped into the own window
	// The hop's own spectrum (N points) and the search for its lag (three nd-point transforms) do not depend on each other, and a
	// single transform of this size fills the chip for little more than one wave of CTAs: on every rank but the first the spectrum
	// runs on the group's side stream (own scratch) beside the lag search; the two meet again in front of sbm_permute_ramp.
	const bool forked = rank != 0;
	if (forked) {
		CU_TRY(ctx, cudaEventRecord(g->ev_fork, stream));
		CU_TRY(ctx, cudaStreamWaitEvent(g->s_side, g->ev_fork, 0));
		if ((rc = tsdrgpu_fft_batch_internal(ctx, g->s_side, reinterpret_cast<const float2 *>(d_hop), 0, g->d_x.ptr, 0, g->d_side.ptr, N, 1, 0))) return rc;
		CU_TRY(ctx, cudaEventRecord(g->ev_join, g->s_side));
	} else if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, reinterpret_cast<const float2 *>(d_hop), g->d_x.ptr, N, 0))) return rc;
	if (rank != 0) {
		const float4 *d0;
		if (d_hop0) {                                         // the alignment reference is resident here: both difference spectra in one batched transform
			KL(ctx, "sbm_abs_diff", stream, sbm_abs_diff2<<<dim3(grid_for(nd, ctx->sm_count), 2), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hop), reinterpret_cast<const float2 *>(d_hop0), g->d_work.ptr, nd));
			if ((rc = tsdrgpu_fft_batch_internal(ctx, stream, g->d_work.ptr, (long long) nd, g->d_dd.ptr, (long long) nd, NULL, nd, 2, 0))) return rc;
			D = g->d_dd.ptr;
			d0 = reinterpret_cast<const float4 *>(g->d_dd.ptr + nd);
		} else {                                              // pull it from rank 0 once its spectra are in place
			KL(ctx, "sbm_abs_diff", stream, sbm_abs_diff<<<grid_for(nd, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hop), g->d_work.ptr, nd));
			if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, D, nd, 0))) return rc;
			KL(ctx, "sbm_sync", stream, sbm_sync<<<1, 32, 0, stream>>>(g->peers, H, rank, PH_SPEC, epoch, all, all, (const int *) NULL, g->timeout_cycles));
			d0 = reinterpret_cast<const float4 *>(g->peers.win[0] + g->off_d);
		}
		KL(ctx, "sbm_xcorr_pull", stream, sbm_xcorr_pull<<<grid_for(nd / 2, ctx->sm_count), 256, 0, stream>>>(d0, reinterpret_cast<const float4 *>(D), reinterpret_cast<float4 *>(g->d_p.ptr), nd / 2));
		if ((rc = tsdrgpu_fft_internal(ctx, stream, g->d_p.ptr, nd, 1))) return rc;
		if ((rc = tsdrgpu_argmax_mag_internal(ctx, stream, g->d_p.ptr, nd, g->d_part.ptr, g->d_lag.ptr))) return rc;
	} else if (!d_hop0) {                                     // rank 0 serves its difference spectrum; its own lag stays 0
		KL(ctx, "sbm_abs_diff", stream, sbm_abs_diff<<<grid_for(nd, ctx->sm_count), 256, 0, stream>>>(reinterpret_cast<const float2 *>(d_hop), g->d_work.ptr, nd));
		if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, D, nd, 0))) return rc;
		KL(ctx, "sbm_sync", stream, sbm_sync<<<1, 32, 0, stream>>>(g->peers, H, rank, PH_SPEC, epoch, all, all, (const int *) NULL, g->timeout_cycles));
	}
	if (forked) CU_TRY(ctx, cudaStreamWaitEvent(stream, g->ev_join, 0));
	KL(ctx, "sbm_permute_ramp", stream, sbm_permute_ramp<<<grid_for(N, ctx->sm_count, 16), 256, 0, stream>>>(g->d_x.ptr, Xp, N, g->log2H, g->d_lag.ptr));
	KL(ctx, "sbm_sync", stream, sbm_sync<<<1, 32, 0, stream>>>(g->peers, H, rank, PH_LAG, epoch, all, all, g->d_lag.ptr, g->timeout_cycles));
	// ---- phase 2: all-to-all #1 (pull this rank's run from everybody), the block transform with the reference's stage angles
	{
		PullArgs A; A.peers = g->peers; A.off_xp = g->off_x; A.H = H; A.rank = rank; A.per = N / (unsigned) H;
		KL(ctx, "sbm_pull_blocks", stream, sbm_pull_blocks<<<grid_for(N / 2, ctx->sm_count, 16), 256, 0, stream>>>(A, reinterpret_cast<float4 *>(g->d_work.ptr)));
	}
	if ((rc = tsdrgpu_fft_oop_internal(ctx, stream, g->d_work.ptr, Ablk, N, 1))) return rc;
	KL(ctx, "sbm_sync", stream, sbm_sync<<<1, 32, 0, stream>>>(g->peers, H, rank, PH_MIX, epoch, all, all, (const int *) NULL, g->timeout_cycles));
	// ---- phase 3: all-to-all #2 + the reference's last log2 H stages + |.| pushed into the root's (time-contiguous) stream
	{
		FinalArgs A; A.peers = g->peers; A.off_a = g->off_v; A.off_r = g->off_r; A.H = H; A.log2H = g->log2H; A.rank = rank; A.root = g->root; A.n = N;
		double eps_all[40];
		unsigned log2N = 0; while ((1u << log2N) < N) log2N++;
		tsdrgpu_fft_reference_eps((int) (log2N + (unsigned) g->log2H), 1, eps_all);
		for (int sidx = 0; sidx < 4; sidx++) A.eps[sidx] = (!tsdrgpu_fft_true_dft() && sidx < g->log2H) ? eps_all[log2N + sidx] : 0.0;
		const unsigned grid = grid_for(N / H, ctx->sm_count, 16);
		switch (H) {
		case 2: KL(ctx, "sbm_final", stream, sbm_final<2><<<grid, 256, 0, stream>>>(A)); break;
		case 4: KL(ctx, "sbm_final", stream, sbm_final<4><<<grid, 256, 0, stream>>>(A)); break;
		default: KL(ctx, "sbm_final", stream, sbm_final<8><<<grid, 256, 0, stream>>>(A)); break;
		}
	}
	KL(ctx, "sbm_sync", stream, sbm_sync<<<1, 32, 0, stream>>>(g->peers, H, rank, PH_RES, epoch, 1u << g->root, rank == g->root ? all : 0u, (const int *) NULL, g->timeout_cycles));
	// ---- phase 4 (root): the stream is complete and time-contiguous in the window; hand it to the caller
	// (d_stream_out == NULL: the caller reads it in place, tsdrgpu_superb_mgpu_stream_window -- on this stream, before its next stitch)
	if (rank == g->root && d_stream_out) CU_TRY(ctx, cudaMemcpyAsync(d_stream_out, g->win.ptr + g->off_r, sizeof(float) * (size_t) H * N, cudaMemcpyDeviceToDevice, stream));
	if (h_n) *h_n = N;
	return TSDRGPU_OK;
}

// Where the root's stream lands inside its window (nranks * N floats after a stitch).  A root that passes d_stream_out = NULL to
// tsdrgpu_superb_mgpu_stitch consumes the stream from here: on the stitch's stream and before its next stitch, whose last phase
// overwrites it (the peers cannot get there earlier: they wait for the root's flags of the next stitch).
int tsdrgpu_superb_mgpu_stream_window(tsdrgpu_superb_mgpu_t *g, float **d_stream) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL && d_stream != NULL);
	*d_stream = reinterpret_cast<float *>(g->win.ptr + g->off_r);
	return TSDRGPU_OK;
}

// the lags (complex samples) every rank published in the last stitch, and the group's status word; synchronises `stream`
int tsdrgpu_superb_mgpu_lags(tsdrgpu_superb_mgpu_t *g, void *stream_, int *h_lags, uint32_t *h_status) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, g != NULL);
	tsdrgpu_ctx_t *ctx = g->ctx;
	BIND(ctx);
	cudaStream_t stream = (cudaStream_t) stream_;
	WinHeader h;
	CU_TRY(ctx, cudaMemcpyAsync(&h, g->win.ptr, sizeof h, cudaMemcpyDeviceToHost, stream));
	CU_TRY(ctx, cudaStreamSynchronize(stream));
	if (h_lags) for (int q = 0; q < g->H; q++) h_lags[q] = h.lag[q];
	if (h_status) *h_status = h.status;
	if (h.status) {
		char msg[160];
		snprintf(msg, sizeof msg, "superbandwidth group: rank %d never finished phase %u of the stitch (timeout)", (int) (h.status >> 8), (h.status & 0xffu) - 1u);
		return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, msg, cudaSuccess, __FILE__, __LINE__);
	}
	return TSDRGPU_OK;
}

}  // extern "C"
