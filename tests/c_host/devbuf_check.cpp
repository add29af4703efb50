// devbuf_check.cpp -- DeviceBuf / PinnedBuf (tempestsdr_b200/csrc/devbuf.h) under allocation failures, without a GPU.
//
// The six runtime calls the header uses are stubbed here on top of malloc, and no CUDA library is linked.  The stub fails the
// k-th allocation (device or pinned) and keeps a table of live allocations.  For every k, a fixed sequence of assign / reserve
// calls runs and, after each call, every buffer must be either what it was before the call, or (nullptr, 0), or the new
// allocation the call asked for; a successful reserve must have kept its first `keep` elements.  When the buffers go out of
// scope, every live allocation must have been freed exactly once, with the matching call, and nothing else freed.
// Prints "ok <runs>" and exits 0, or prints what went wrong and exits 1.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "../../tempestsdr_b200/csrc/devbuf.h"

namespace {

struct Alloc { size_t bytes; bool pinned; };
std::map<void *, Alloc> g_live;
long g_allocs = 0, g_fail_at = -1;                 // allocations so far; the one (0-based) that fails, -1: none
std::vector<std::string> g_errors;

void error(const std::string &what) { if (g_errors.size() < 20) g_errors.push_back(what); }

bool take(void **p, size_t bytes, bool pinned) {
	if (g_allocs++ == g_fail_at) { *p = (void *) 0x1; return false; }      // a failed call leaves garbage behind
	*p = malloc(bytes ? bytes : 1);
	g_live[*p] = Alloc{bytes, pinned};
	return true;
}

void give(void *p, bool pinned) {
	if (!p) return;                                // cudaFree(NULL) is legal and does nothing
	auto it = g_live.find(p);
	if (it == g_live.end()) { error("free of a pointer that is not a live allocation"); return; }
	if (it->second.pinned != pinned) error(pinned ? "cudaFreeHost of device memory" : "cudaFree of pinned memory");
	free(p);
	g_live.erase(it);
}

// [p, p + bytes) lies inside one live allocation
bool inside(const void *p, size_t bytes) {
	auto it = g_live.upper_bound(const_cast<void *>(p));
	if (it == g_live.begin()) return false;
	--it;
	const char *a = (const char *) it->first, *q = (const char *) p;
	return q >= a && q + bytes <= a + it->second.bytes;
}

}  // namespace

extern "C" {
cudaError_t cudaMalloc(void **p, size_t bytes) { return take(p, bytes, false) ? cudaSuccess : cudaErrorMemoryAllocation; }
cudaError_t cudaFree(void *p) { give(p, false); return cudaSuccess; }
cudaError_t cudaFreeHost(void *p) { give(p, true); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *dst, const void *src, size_t bytes, enum cudaMemcpyKind, cudaStream_t) {
	if (!inside(dst, bytes) || !inside(src, bytes)) { error("copy outside a live allocation"); return cudaErrorInvalidValue; }
	memcpy(dst, src, bytes);
	return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
int tsdrgpu_malloc_host(tsdrgpu_ctx_t *, size_t bytes, void **p) { return take(p, bytes, true) ? TSDRGPU_OK : TSDRGPU_ECUDA; }
}

namespace {

// one buffer under test and what it must hold: `valid` elements of the pattern `tag`
template <class B> struct Watched {
	const char *name; B buf; int tag = 0; size_t valid = 0;
	Watched(const char *n) : name(n) {}
	void fill() {                                  // a fresh pattern over the whole allocation
		tag++;
		for (size_t i = 0; i < buf.cap; i++) buf.ptr[i] = (decltype(+buf.ptr[0])) (tag * 100000 + i);
		valid = buf.cap;
	}
	bool holds(size_t n) const {
		for (size_t i = 0; i < n; i++) if (buf.ptr[i] != (decltype(+buf.ptr[0])) (tag * 100000 + i)) return false;
		return true;
	}
};

template <class W> void check_state(W &w, const char *op, void *old_ptr, size_t old_cap, bool ok, size_t want_cap, size_t keep) {
	char what[200];
	const bool same = w.buf.ptr == old_ptr && w.buf.cap == old_cap;
	const bool empty = w.buf.ptr == nullptr && w.buf.cap == 0;
	if (ok) {
		if (w.buf.cap != want_cap || (want_cap && !w.buf.ptr)) { snprintf(what, sizeof what, "%s %s: capacity %zu, expected %zu", w.name, op, w.buf.cap, want_cap); error(what); }
	} else if (!same && !empty) {
		snprintf(what, sizeof what, "%s %s failed and left neither the old buffer nor an empty one", w.name, op); error(what);
	}
	if (w.buf.ptr && !inside(w.buf.ptr, sizeof(*w.buf.ptr) * w.buf.cap)) { snprintf(what, sizeof what, "%s %s: buffer is not a live allocation", w.name, op); error(what); }
	if (!w.buf.ptr && w.buf.cap) { snprintf(what, sizeof what, "%s %s: null buffer with a capacity", w.name, op); error(what); }
	if (same) return;                              // unchanged: its contents stay as they were
	if (ok && keep && !w.holds(keep)) { snprintf(what, sizeof what, "%s %s did not keep its first %zu elements", w.name, op, keep); error(what); }
	if (w.buf.ptr) w.fill(); else w.valid = 0;
}

template <class W> bool assign(W &w, size_t n) {
	void *p = w.buf.ptr; const size_t c = w.buf.cap;
	const bool ok = w.buf.assign(n) == cudaSuccess;
	check_state(w, "assign", p, c, ok, n, 0);
	return ok;
}
template <class W> bool assign_pinned(W &w, size_t n) {
	void *p = w.buf.ptr; const size_t c = w.buf.cap;
	const bool ok = w.buf.assign(nullptr, n) == TSDRGPU_OK;
	check_state(w, "assign", p, c, ok, n, 0);
	return ok;
}
template <class W> bool reserve(W &w, size_t need, size_t keep) {
	void *p = w.buf.ptr; const size_t c = w.buf.cap;
	const bool ok = w.buf.reserve(nullptr, need, keep) == cudaSuccess;
	const size_t want = c >= need ? c : need + need / 2 + 1024;
	check_state(w, "reserve", p, c, ok, want, p && c < need && keep <= w.valid ? keep : 0);
	return ok;
}

// the fixed sequence: both kinds of buffer, growth and no-op reserves, assigns that shrink and grow, reserves from empty
void sequence() {
	Watched<DeviceBuf<int>> a("a");
	Watched<DeviceBuf<double>> b("b");
	Watched<PinnedBuf<float>> h("h");
	assign(a, 10);
	reserve(a, 20, 10);
	reserve(a, 30, 10);                            // fits: nothing happens
	reserve(b, 5, 0);
	assign_pinned(h, 8);
	assign(b, 3);
	reserve(a, 5000, 10);
	assign_pinned(h, 100);
	reserve(b, 2000, 3);
	assign(a, 7);
	reserve(a, 7, 7);
	assign_pinned(h, 4);
	reserve(a, 9000, 7);
}

}  // namespace

int main() {
	sequence();                                    // no failure: how many allocations the sequence makes
	const long total = g_allocs;
	if (total < 10) error("the sequence made too few allocations");
	long runs = 0;
	for (long k = -1; k <= total; k++) {           // -1: no failure; total: one past the last allocation
		g_allocs = 0; g_fail_at = k; g_live.clear();
		sequence();
		runs++;
		if (!g_live.empty()) { char what[120]; snprintf(what, sizeof what, "failing allocation %ld: %zu allocations never freed", k, g_live.size()); error(what); }
	}
	if (!g_errors.empty()) {
		for (const std::string &e : g_errors) fprintf(stderr, "%s\n", e.c_str());
		return 1;
	}
	printf("ok %ld\n", runs);
	return 0;
}
