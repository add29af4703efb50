// ctx.cu -- context, memory and stream plumbing of libtsdrgpu (include/tsdrgpu.h, "context" section).
#include "common.cuh"
#include <string.h>
#include <stdlib.h>
#include <ctype.h>
#include <sched.h>
#include <unistd.h>
#include <sys/syscall.h>

thread_local char g_tsdrgpu_err[512] = "";

extern "C" {

int tsdrgpu_device_count(void) {
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
	return n;
}

int tsdrgpu_create(tsdrgpu_ctx_t **out, int device) {
	if (!out) return tsdrgpu_fail(NULL, TSDRGPU_EINVAL, "null out pointer", cudaSuccess, __FILE__, __LINE__);
	*out = NULL;
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n <= 0) {
		cudaGetLastError();
		return tsdrgpu_fail(NULL, TSDRGPU_ENODEVICE, "no CUDA device visible (this library has no CPU fallback)", e, __FILE__, __LINE__);
	}
	if (device < 0 || device >= n) return tsdrgpu_fail(NULL, TSDRGPU_EINVAL, "device index out of range", cudaSuccess, __FILE__, __LINE__);
	cudaDeviceProp prop;
	e = cudaGetDeviceProperties(&prop, device);
	if (e != cudaSuccess) return tsdrgpu_fail(NULL, TSDRGPU_ECUDA, "cudaGetDeviceProperties", e, __FILE__, __LINE__);
	if (prop.major != 9 || prop.minor != 0) {
		char msg[160];
		snprintf(msg, sizeof msg, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
		return tsdrgpu_fail(NULL, TSDRGPU_ENODEVICE, msg, cudaSuccess, __FILE__, __LINE__);
	}
	tsdrgpu_ctx_t *c = new tsdrgpu_ctx();
	c->device = device;
	c->sm_count = prop.multiProcessorCount;
	c->err[0] = 0;
	c->launches = 0;
	c->profiling = false; c->prof_nnames = 0;
	e = cudaSetDevice(device);
	if (e != cudaSuccess) { delete c; return tsdrgpu_fail(NULL, TSDRGPU_ECUDA, "cudaSetDevice", e, __FILE__, __LINE__); }
	*out = c;
	return TSDRGPU_OK;
}

void tsdrgpu_destroy(tsdrgpu_ctx_t *ctx) {
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	for (auto &r : ctx->prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
	for (auto e : ctx->prof_pool) cudaEventDestroy(e);
	delete ctx;
}

const char *tsdrgpu_last_error(tsdrgpu_ctx_t *ctx) { return ctx ? ctx->err : g_tsdrgpu_err; }
int tsdrgpu_sm_count(tsdrgpu_ctx_t *ctx) { return ctx ? ctx->sm_count : 0; }
uint64_t tsdrgpu_launch_count(tsdrgpu_ctx_t *ctx) { return ctx ? ctx->launches : 0; }

int tsdrgpu_malloc(tsdrgpu_ctx_t *ctx, size_t bytes, void **d_ptr) {
	BIND(ctx); ARG_TRY(ctx, d_ptr != NULL);
	CU_TRY(ctx, cudaMalloc(d_ptr, bytes ? bytes : 1));
	return TSDRGPU_OK;
}
int tsdrgpu_free(tsdrgpu_ctx_t *ctx, void *d_ptr) { BIND(ctx); CU_TRY(ctx, cudaFree(d_ptr)); return TSDRGPU_OK; }
// ---- host memory near the GPU -------------------------------------------------------------------------------------------
// On a two-socket box half of the GPUs hang off each socket; page-locked buffers on the far socket cross the inter-socket link
// on every DMA.  The NUMA node of the device comes from sysfs; allocations
// are steered with set_mempolicy(MPOL_PREFERRED) around cudaMallocHost (the driver faults the pages in inside that call),
// raw syscalls because libnuma is not a dependency.  Everything degrades to a no-op when sysfs or the syscall says no.
int tsdrgpu_device_numa_node(tsdrgpu_ctx_t *ctx) {
	if (!ctx) return -1;
	char bus[32] = {0}, path[128];
	if (cudaDeviceGetPCIBusId(bus, sizeof bus, ctx->device) != cudaSuccess) { cudaGetLastError(); return -1; }
	for (char *c = bus; *c; c++) *c = (char) tolower(*c);
	snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
	FILE *f = fopen(path, "r");
	if (!f) return -1;
	int node = -1;
	if (fscanf(f, "%d", &node) != 1) node = -1;
	fclose(f);
	return node;
}
static long mempolicy_prefer(int node, int *old_mode, unsigned long *old_mask) {
#if defined(SYS_set_mempolicy) && defined(SYS_get_mempolicy)
	if (node < 0 || node >= 64) return -1;
	if (syscall(SYS_get_mempolicy, old_mode, old_mask, 64ul, NULL, 0ul) != 0) return -1;
	unsigned long mask = 1ul << node;
	return syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, &mask, 64ul);
#else
	(void) node; (void) old_mode; (void) old_mask; return -1;
#endif
}
static void mempolicy_restore(int old_mode, unsigned long old_mask) {
#if defined(SYS_set_mempolicy)
	syscall(SYS_set_mempolicy, old_mode, old_mode == 0 ? NULL : &old_mask, old_mode == 0 ? 0ul : 64ul);
#endif
}
int tsdrgpu_malloc_host(tsdrgpu_ctx_t *ctx, size_t bytes, void **h_ptr) {
	BIND(ctx); ARG_TRY(ctx, h_ptr != NULL);
	int old_mode = 0; unsigned long old_mask = 0;
	const bool steer = !getenv("TSDRGPU_NO_NUMA") && mempolicy_prefer(tsdrgpu_device_numa_node(ctx), &old_mode, &old_mask) == 0;
	const cudaError_t e = cudaMallocHost(h_ptr, bytes ? bytes : 1);
	if (steer) mempolicy_restore(old_mode, old_mask);
	CU_TRY(ctx, e);
	return TSDRGPU_OK;
}
// pin the CALLING thread to the cores of the device's NUMA node (what a per-GPU worker process or thread wants); 0 = done
int tsdrgpu_bind_thread_near_device(tsdrgpu_ctx_t *ctx) {
	if (getenv("TSDRGPU_NO_NUMA")) return TSDRGPU_EINVAL;
	const int node = tsdrgpu_device_numa_node(ctx);
	if (node < 0) return TSDRGPU_EINVAL;
	char path[128], list[4096] = {0};
	snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
	FILE *f = fopen(path, "r");
	if (!f) return TSDRGPU_EINVAL;
	if (!fgets(list, sizeof list, f)) { fclose(f); return TSDRGPU_EINVAL; }
	fclose(f);
	cpu_set_t allowed, want;
	CPU_ZERO(&want);
	if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return TSDRGPU_EINVAL;
	int any = 0;
	for (char *tok = strtok(list, ",\n"); tok; tok = strtok(NULL, ",\n")) {
		int a = 0, b = 0;
		const int k = sscanf(tok, "%d-%d", &a, &b);
		if (k < 1) continue;
		if (k == 1) b = a;
		for (int c = a; c <= b && c < CPU_SETSIZE; c++) if (CPU_ISSET(c, &allowed)) { CPU_SET(c, &want); any = 1; }
	}
	if (!any) return TSDRGPU_EINVAL;                   // a cgroup / taskset already excludes that node: leave things alone
	return sched_setaffinity(0, sizeof want, &want) == 0 ? TSDRGPU_OK : TSDRGPU_EINVAL;
}
int tsdrgpu_free_host(tsdrgpu_ctx_t *ctx, void *h_ptr) { BIND(ctx); CU_TRY(ctx, cudaFreeHost(h_ptr)); return TSDRGPU_OK; }

int tsdrgpu_memcpy_h2d(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, const void *h_src, size_t bytes) {
	BIND(ctx);
	CU_TRY(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, (cudaStream_t) stream));
	return TSDRGPU_OK;
}
int tsdrgpu_memcpy_d2h(tsdrgpu_ctx_t *ctx, void *stream, void *h_dst, const void *d_src, size_t bytes) {
	BIND(ctx);
	CU_TRY(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t) stream));
	return TSDRGPU_OK;
}
int tsdrgpu_memcpy_d2d(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, const void *d_src, size_t bytes) {
	BIND(ctx);
	if (bytes) CU_TRY(ctx, cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t) stream));
	return TSDRGPU_OK;
}
int tsdrgpu_memset(tsdrgpu_ctx_t *ctx, void *stream, void *d_dst, int value, size_t bytes) {
	BIND(ctx);
	CU_TRY(ctx, cudaMemsetAsync(d_dst, value, bytes, (cudaStream_t) stream));
	return TSDRGPU_OK;
}
int tsdrgpu_stream_create(tsdrgpu_ctx_t *ctx, void **stream) {
	BIND(ctx); ARG_TRY(ctx, stream != NULL);
	cudaStream_t s;
	CU_TRY(ctx, cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
	*stream = (void *) s;
	return TSDRGPU_OK;
}
int tsdrgpu_stream_destroy(tsdrgpu_ctx_t *ctx, void *stream) { BIND(ctx); CU_TRY(ctx, cudaStreamDestroy((cudaStream_t) stream)); return TSDRGPU_OK; }
int tsdrgpu_stream_sync(tsdrgpu_ctx_t *ctx, void *stream) { BIND(ctx); CU_TRY(ctx, cudaStreamSynchronize((cudaStream_t) stream)); return TSDRGPU_OK; }

int tsdrgpu_profile_enable(tsdrgpu_ctx_t *ctx, int on) {
	BIND(ctx);
	ctx->profiling = on != 0;
	return TSDRGPU_OK;
}

int tsdrgpu_profile_collect(tsdrgpu_ctx_t *ctx, char *names, double *total_ms, uint64_t *counts, int cap, int *n) {
	BIND(ctx); ARG_TRY(ctx, names && total_ms && counts && n && cap > 0);
	CU_TRY(ctx, cudaDeviceSynchronize());
	std::lock_guard<std::mutex> lock(ctx->mu);
	const int m = ctx->prof_nnames < cap ? ctx->prof_nnames : cap;
	for (int i = 0; i < m; i++) { strncpy(names + 48 * i, ctx->prof_names[i], 48); total_ms[i] = 0.0; counts[i] = 0; }
	for (auto &r : ctx->prof_recs) {
		float ms = 0.0f;
		if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess && r.id < m) { total_ms[r.id] += ms; counts[r.id]++; }
		ctx->prof_pool.push_back(r.a); ctx->prof_pool.push_back(r.b);
	}
	ctx->prof_recs.clear();
	*n = m;
	return TSDRGPU_OK;
}

}  // extern "C"

static cudaEvent_t prof_event(tsdrgpu_ctx_t *ctx) {
	if (!ctx->prof_pool.empty()) { cudaEvent_t e = ctx->prof_pool.back(); ctx->prof_pool.pop_back(); return e; }
	cudaEvent_t e; cudaEventCreate(&e); return e;
}
void tsdrgpu_prof_begin(tsdrgpu_ctx_t *ctx, const char *name, cudaStream_t stream) {
	std::lock_guard<std::mutex> lock(ctx->mu);
	int id = -1;
	for (int i = 0; i < ctx->prof_nnames; i++) if (!strcmp(ctx->prof_names[i], name)) { id = i; break; }
	if (id < 0) { if (ctx->prof_nnames >= 48) return; id = ctx->prof_nnames++; strncpy(ctx->prof_names[id], name, 47); ctx->prof_names[id][47] = 0; }
	tsdrgpu_ctx::ProfRec r; r.id = id; r.a = prof_event(ctx); r.b = prof_event(ctx);
	cudaEventRecord(r.a, stream);
	ctx->prof_recs.push_back(r);
}
void tsdrgpu_prof_end(tsdrgpu_ctx_t *ctx, cudaStream_t stream) {
	std::lock_guard<std::mutex> lock(ctx->mu);
	if (!ctx->prof_recs.empty()) cudaEventRecord(ctx->prof_recs.back().b, stream);
}

int tsdrgpu_scratch(tsdrgpu_ctx_t *ctx, int slot, size_t bytes, void **out) {
	DeviceBuf<unsigned char> &b = ctx->scratch[slot];
	if (b.cap < bytes) {
		if (b.ptr) CU_TRY(ctx, cudaDeviceSynchronize());
		CU_TRY(ctx, b.assign(bytes + (bytes >> 2) + 256));
	}
	*out = b.ptr;
	return TSDRGPU_OK;
}

int tsdrgpu_pinned(tsdrgpu_ctx_t *ctx, size_t bytes, void **out) {
	PinnedBuf<unsigned char> &b = ctx->pinned;
	if (b.cap < bytes) {
		if (b.ptr) CU_TRY(ctx, cudaDeviceSynchronize());
		const int rc = b.assign(ctx, bytes * 2 + 4096);
		if (rc) return rc;
	}
	*out = b.ptr;
	return TSDRGPU_OK;
}
