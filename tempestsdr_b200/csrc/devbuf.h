// devbuf.h -- owning buffers of libtsdrgpu: device and page-locked host memory that frees itself with its owner.  Host code
// only (no kernel, no device function), so that it also builds with a plain C++ compiler.
#pragma once
#include <cuda_runtime.h>

#include "../../include/tsdrgpu.h"

// Device memory owned by an object: a pointer and its capacity in elements, freed with the owner.  Neither call leaves a
// freed pointer behind: a failed assign leaves the buffer empty, a failed reserve leaves the old one in place.
template <class T> struct DeviceBuf {
	T *ptr = nullptr; size_t cap = 0;
	DeviceBuf() = default; DeviceBuf(const DeviceBuf &) = delete; DeviceBuf &operator=(const DeviceBuf &) = delete;
	~DeviceBuf() { if (ptr) cudaFree(ptr); }
	// at least `need` elements (need + need/2 + 1024 when it grows); the first `keep` are copied on stream s, which is then
	// synchronised before the old buffer is freed
	cudaError_t reserve(cudaStream_t s, size_t need, size_t keep = 0) {
		if (cap >= need) return cudaSuccess;
		const size_t ncap = need + need / 2 + 1024;
		T *nb;
		cudaError_t e = cudaMalloc(&nb, sizeof(T) * ncap);
		if (e != cudaSuccess) return e;
		if (ptr && keep) e = cudaMemcpyAsync(nb, ptr, sizeof(T) * keep, cudaMemcpyDeviceToDevice, s);
		if (e == cudaSuccess) e = cudaStreamSynchronize(s);
		if (e != cudaSuccess) { cudaFree(nb); return e; }
		T *old = ptr; ptr = nb; cap = ncap;
		return old ? cudaFree(old) : cudaSuccess;
	}
	// exactly n elements, contents not kept: the old buffer is freed first
	cudaError_t assign(size_t n) {
		cudaError_t e = ptr ? cudaFree(ptr) : cudaSuccess;
		ptr = nullptr; cap = 0;
		if (e == cudaSuccess) e = cudaMalloc(&ptr, sizeof(T) * n);
		if (e == cudaSuccess) cap = n; else ptr = nullptr;
		return e;
	}
};

// Page-locked host memory owned by an object (tsdrgpu_malloc_host: on the device's NUMA node), a pointer and its capacity in
// elements, freed with the owner.
template <class T> struct PinnedBuf {
	T *ptr = nullptr; size_t cap = 0;
	PinnedBuf() = default; PinnedBuf(const PinnedBuf &) = delete; PinnedBuf &operator=(const PinnedBuf &) = delete;
	~PinnedBuf() { if (ptr) cudaFreeHost(ptr); }
	// exactly n elements, contents not kept: the old buffer is freed first, so peak pinned memory is the larger of the two; a
	// failure leaves the buffer empty
	int assign(tsdrgpu_ctx_t *ctx, size_t n) {
		if (ptr) cudaFreeHost(ptr);
		ptr = nullptr; cap = 0;
		const int rc = tsdrgpu_malloc_host(ctx, sizeof(T) * n, (void **) &ptr);
		if (rc == TSDRGPU_OK) cap = n; else ptr = nullptr;
		return rc;
	}
};
