// pipeline.cu -- a1, a3, a5, a16, a17: the streaming glue between the plugin callback and the frame callback.
//
// Replaces the body of process() (TSDRLibrary.c:264-298), decimatingthread / postprocessingthread /
// videodecodingthread (TSDRLibrary.c:300-418), the three CircBuff rings between them (circbuff.c) and the
// frame-rate detector thread's capture loop (frameratedetector.c:128-187, 215-230).  Host buffers in, host frame
// and plot buffers out: this is the object the C host library (tempestsdr_b200/host/TSDRLibrary.c) drives from
// the reference's own process() callback, and the one bench.py times end to end.
//
// Data movement per IQ block: one H2D copy of the plugin's buffer (float32, or the front end's 8/16-bit wire format
// converted on the device: tsdrgpu_pipeline_process_raw),
// everything else stays in HBM: IQ -> (fused demod+resample) -> pixel stream -> (frame stage, batches of frames)
// -> one D2H copy of the finished frames into page-locked slots -> frame callback on the delivery thread.
// The reference's rings, which copy every sample 2x per stage under a mutex, do not exist here; what is kept
// is their observable behaviour: whole-block dropping with frame-aligned resynchronisation (dsp.c:313-368),
// purge of the autocorrelation capture on any drop (frameratedetector.c:221-224).
//
// Ordering differences to the (timing-dependent, SURVEY.md F9) threaded reference, both deterministic here:
//   * geometry changes made by the PLL take effect at the next batch boundary;
//   * tsdr_sync offsets are applied between batches of decimator blocks rather than between single blocks.
#include "common.cuh"
#include "host_plan.h"
#include <math.h>
#include <condition_variable>
#include <deque>
#include <memory>
#include <thread>
#include <vector>

struct tsdrgpu_frd;
struct tsdrgpu_resampler;
struct tsdrgpu_framestage;

namespace {

constexpr int PL_SLOTS = 4;
using Stats = tsdrgpu_pipeline_stats_t;

// The busy flags of one kind of delivery slot, under tsdrgpu_pipeline::mu.  The worker takes a slot before it queues a copy into
// the slot's page-locked buffers; the delivery thread releases it once the job's callbacks have returned.
struct SlotPool {
	tsdrgpu_pipeline *p; int n;                       // n <= PL_SLOTS slots
	uint64_t Stats::*delivered, Stats::*skipped;      // count what release delivers / what acquire finds no slot for (null: nothing)
	int busy[PL_SLOTS];
	int free_slot() const { for (int k = 0; k < n; k++) if (!busy[k]) return k; return -1; }
	template <class F> bool any(F f) const { for (int k = 0; k < n; k++) if (f(k)) return true; return false; }   // f(k) for some slot k
	int acquire(bool wait, uint64_t count);           // a free slot, or -1; wait: until the delivery thread frees one
	void release(int slot, uint64_t count);           // also counts the job delivered and wakes whoever waits for that
};

enum JobKind { JOB_FRAMES, JOB_PLOTS, JOB_REPORT };

struct FrameJob {
	JobKind kind;
	SlotPool *pool;           // the slot's pool, released after delivery
	int slot; uint32_t samplerate;   // samplerate: plots and reports
	int nframes, w, h;
	int plot_id, report_n;    // a report: TSDRGPU_PLOT_ID_SPECTRUM or _COHERENCE, and N
	double *report;           // a report: its values in the slot
	cudaEvent_t ev;
	int foff, flen, loff, llen; uint64_t calls; int reset_announce, dump_announce;
	int detect_mode;          // plots: announce the video mode detected from them
	int snr_valid;            // frames: results carry an SNR to announce
	int pll_valid;            // frames: h_pll_rr holds the refresh rates the PLL set
	int stack_valid;          // frames: h_stack holds the stack's records
};

// Everything the public setters write, under tsdrgpu_pipeline::set_mu.  The worker reads copies taken under the lock (per
// process() call and per group of decimator blocks), so a batch never sees half of a setting; the one-shot requests (pending
// sync offset, PLOTS_RESET, DUMP) are taken and cleared under the lock where they are consumed.
struct Settings {
	uint32_t samplerate = 0, samplerate_real = 0;     // the decimator's rate (superbandwidth: hops x the front end's) / the front end's
	int height = 0; double refreshrate = 0;
	int width = 0; double ptos = 0;                    // derived from the three above: geometry()
	float motionblur = 0;
	uint32_t params[9] = {};
	int syncoffset = 0;                                // tsdr_sync pixels not yet applied
	int report_snr = 0, detect_mode = 0;               // 8f-4 / 8f-3, both off by default (the reference announces neither)
	int argb_mode = 0, argb_inverted = 0;              // 8f-2: final pixels instead of floats
	int rs_kernel = TSDRGPU_RS_BOX;                    // applied per group of blocks
	int ag_mode = TSDRGPU_AG_MINMAX, ag_ppm = 0;       // applied per frame-stage batch, as are contrast and denoise
	int ct_mode = TSDRGPU_CONTRAST_OFF, ct_clip = 200, ct_tx = 8, ct_ty = 8;
	int nl_mode = TSDRGPU_DENOISE_OFF, nl_h = 100, nl_r = 5, nl_p = 1;
	int st_mode = TSDRGPU_STACK_OFF, st_depth = 32, st_rx = 8, st_ry = 2;
	int db_mode = TSDRGPU_DEBLUR_OFF, db_sigma = 100, db_iters = 20;
	int stack_restart = 0;                             // tsdr_sync: the stack restarts at the next frame-stage batch
	tsdrgpu_channel_t cf_spec = {};                    // taps == 0: off; applied per process()
	tsdrgpu_welch_t sp_spec = {};                      // n == 0: off; applied per process()
	tsdrgpu_coherence_t ch_spec = {};                  // rate == 0: off; applied per process()
	tsdrgpu_superband_t sbd_spec = {};                 // mode 0: the reference's stitch; latched at the start of each superbandwidth round
	int host_register = 0;                             // opt-in: tsdrgpu_pipeline_set_host_registration
	tsdrgpu_retune_cb retune_cb = nullptr;
};

// block-aligned dropping, dsp.c:313-368 (integer bookkeeping, host side)
struct DropComp {
	int64_t difference = 0;
	static uint64_t debt(int block, int dropped) { const uint64_t whole = (uint64_t) (dropped / block); return ((whole + 1) * block - dropped) % block; }
	void shift_with(uint32_t block, int64_t syncoffset) {
		if (syncoffset >= 0) difference -= syncoffset % block; else difference -= block + syncoffset % block;
		if (difference < 0) difference = (int64_t) debt((int) block, (int) -difference);
	}
	bool will_drop_all(uint32_t size) const { return size <= difference; }
	// returns elements forwarded; *skip = leading elements discarded.  accepted = downstream took the block
	uint32_t add(uint32_t size, uint32_t block, bool accepted, uint32_t *skip) {
		*skip = 0;
		if (size <= difference) { difference -= size; *skip = size; return 0; }
		if (accepted) { const uint32_t lead = (uint32_t) difference; difference = 0; *skip = lead; return size - lead; }
		difference -= size % block;
		if (difference < 0) difference = (int64_t) debt((int) block, (int) -difference);
		return 0;
	}
};

__global__ void pl_copy_f32(const float *__restrict__ src, float *__restrict__ dst, size_t n) {
	for (size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t) gridDim.x * blockDim.x) dst[i] = src[i];
}

// Raw sample formats of the RawFile front end converted on the device (SURVEY section 8f-1): the same values as the plugin's
// host loop (TSDRPlugin_RawFile.c:241-261) -- int8 v/128.0, uint8 (v-128)/128.0 (exact in float), int16 v/32767.0 and
// uint16 (v-32767)/32767.0 (double quotient rounded to float, exactly as the C expression).
__device__ __forceinline__ float raw_to_float(int v, int fmt) {
	switch (fmt) {
	case TSDRGPU_FMT_INT8:   return (float) v * 0.0078125f;
	case TSDRGPU_FMT_UINT8:  return (float) (v - 128) * 0.0078125f;
	case TSDRGPU_FMT_INT16:  return __double2float_rn(__ddiv_rn((double) v, 32767.0));
	default:                 return __double2float_rn(__ddiv_rn((double) (v - 32767), 32767.0));
	}
}
__global__ void __launch_bounds__(256) pl_convert(const void *__restrict__ raw, float *__restrict__ dst, size_t items, int fmt) {
	const size_t stride = (size_t) gridDim.x * blockDim.x, t0 = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	if (fmt == TSDRGPU_FMT_INT8 || fmt == TSDRGPU_FMT_UINT8) {
		// 4 samples per thread only where both sides allow it (the superbandwidth gather appends at odd pair counts: dst is then
		// only 8-byte aligned); otherwise everything goes through the scalar tail loop
		const bool vec = ((reinterpret_cast<unsigned long long>(dst) & 15ull) == 0) && ((reinterpret_cast<unsigned long long>(raw) & 3ull) == 0);
		const size_t n4 = vec ? (items >> 2) : 0;
		for (size_t i = t0; i < n4; i += stride) {           // 4 samples per thread
			const uchar4 q = __ldg(reinterpret_cast<const uchar4 *>(raw) + i);
			float4 o;
			if (fmt == TSDRGPU_FMT_INT8) { o.x = raw_to_float((signed char) q.x, fmt); o.y = raw_to_float((signed char) q.y, fmt); o.z = raw_to_float((signed char) q.z, fmt); o.w = raw_to_float((signed char) q.w, fmt); }
			else { o.x = raw_to_float(q.x, fmt); o.y = raw_to_float(q.y, fmt); o.z = raw_to_float(q.z, fmt); o.w = raw_to_float(q.w, fmt); }
			reinterpret_cast<float4 *>(dst)[i] = o;
		}
		for (size_t i = (n4 << 2) + t0; i < items; i += stride) {
			const unsigned char b = reinterpret_cast<const unsigned char *>(raw)[i];
			dst[i] = raw_to_float(fmt == TSDRGPU_FMT_INT8 ? (int) (signed char) b : (int) b, fmt);
		}
		return;
	}
	for (size_t i = t0; i < items; i += stride) {                 // 16-bit formats: scalar (2-byte alignment is the format's own)
		const unsigned short u = __ldg(reinterpret_cast<const unsigned short *>(raw) + i);
		dst[i] = raw_to_float(fmt == TSDRGPU_FMT_INT16 ? (int) (short) u : (int) u, fmt);
	}
}
static inline size_t fmt_bytes(int fmt) { return fmt == TSDRGPU_FMT_FLOAT ? 4 : ((fmt == TSDRGPU_FMT_INT8 || fmt == TSDRGPU_FMT_UINT8) ? 1 : 2); }

}  // namespace

// One hop of a superbandwidth round on device `dev`.  Ranks >= 1 of the sharded mode own a context, streams and an event; rank 0
// and the one-GPU mode's hops borrow the pipeline's.  Destroyed after the group with `dev` current: streams and event, buffers, context.
struct SbRank {
	int dev = 0; tsdrgpu_ctx_t *ctx = nullptr; cudaStream_t stream = nullptr, copy = nullptr; cudaEvent_t ev = nullptr;
	struct OwnCtx { tsdrgpu_ctx_t *c = nullptr; ~OwnCtx() { tsdrgpu_destroy(c); } } own;      // null: everything is borrowed
	DeviceBuf<float> hop, hop0;                       // the hop; an owned rank's copy of hop 0, the alignment reference
	DeviceBuf<unsigned char> raw;                     // an owned rank's raw-format staging (the others use the pipeline's d_raw[0])
	~SbRank() { cudaSetDevice(dev); if (own.c) { if (stream) cudaStreamDestroy(stream); if (copy) cudaStreamDestroy(copy); if (ev) cudaEventDestroy(ev); } }
};

// A report side path (the Welch spectrum, the coherence): its object runs over every converted block on s_spec, and its reports go
// out through slots of their own, so one path's reports waiting for delivery never take the other path's slots.
template <class Obj> struct ReportPath {
	int plot_id; SlotPool pool;
	Obj *obj;                                          // created on first use
	DeviceBuf<double> d_out; PinnedBuf<double> h[PL_SLOTS];
	int fresh;                                         // blocks went by without this path: the next one starts a new report
};

struct tsdrgpu_pipeline {
	tsdrgpu_ctx_t *ctx;
	tsdrgpu_pipeline_config_t cfg;
	tsdrgpu_frame_cb frame_cb; tsdrgpu_value_cb value_cb; tsdrgpu_plot_cb plot_cb; void *user;
	cudaStream_t s_main, s_copy, s_out, s_ingest;      // heavy kernels | H2D | D2H | light per-block kernels
	cudaEvent_t ev_ingest, ev_decim, ev_cap_used[2];
	cudaEvent_t ev_out[2], ev_main; int out_phase;
	cudaEvent_t ev_h2d[4], ev_used[4]; int stage_slot;

	std::mutex set_mu; Settings set;                   // see Settings

	// stage 0: H2D staging of the plugin's buffer
	DeviceBuf<float> d_stage[4];                       // 4 slots so H2D runs ahead of the kernels
	DeviceBuf<unsigned char> d_raw[4];                 // raw-format blocks land here and are converted into d_stage
	// plugin buffers seen on process(): page-locked in place (cudaHostRegister) once the same buffer keeps coming back, so that
	// an unmodified plugin's malloc'd block crosses PCIe by direct DMA instead of through the driver's staging copy
	struct HostBuf { const void *base; size_t bytes; int seen; int state; };      // state: 0 candidate, 1 registered here, 2 pinned by its owner, 3 refused
	std::vector<HostBuf> hostbufs;
	// stage 1: decimator input (IQ pairs waiting for whole blocks)
	// samples waiting for whole decimator blocks: [decim_read, decim_read + decim_fill) samples of decim_elem floats each
	// (2 = interleaved I,Q, demodulated inside rs_main; 1 = magnitudes, what the multi-GPU superbandwidth stitch delivers).
	// Consumed from the front by moving decim_read; compacted only when the hole in front is at least as large as what is
	// left, so source and destination of the move never overlap.
	DeviceBuf<float> d_decim; size_t decim_fill, decim_read; int decim_elem = 2;
	DropComp dev_drop;
	// stage 2: pixels waiting for whole frames
	tsdrgpu_resampler *rs;
	// channel filter (tsdrgpu_pipeline_set_channel): created on first use
	tsdrgpu_chanfilt *cf; DeviceBuf<float> d_cf_out;
	int cf_stale;                                      // a block with samples went by unfiltered: zero the history before the next
	// Welch spectrum and coherence (tsdrgpu_pipeline_set_spectrum, _set_coherence): their work runs on s_spec (low priority)
	ReportPath<tsdrgpu_spectrum> spec{TSDRGPU_PLOT_ID_SPECTRUM, {this, PL_SLOTS, &Stats::spectra_delivered, &Stats::spectra_skipped}};
	ReportPath<tsdrgpu_coherence> coh{TSDRGPU_PLOT_ID_COHERENCE, {this, PL_SLOTS, &Stats::coherence_delivered, &Stats::coherence_skipped}};
	cudaStream_t s_spec;
	cudaEvent_t ev_conv, ev_sp_used[4];                // the block is converted / s_spec (spectrum, coherence) has read staging slot i
	DeviceBuf<float> d_pix; size_t pix_read, pix_fill;
	DropComp pix_drop;
	// stage 3: frames
	tsdrgpu_framestage *fs;
	DeviceBuf<float> d_frames[2];                      // double-buffered: D2H of batch k overlaps the kernels of batch k+1
	DeviceBuf<int32_t> d_argb_last;                    // 8f-2: the host's persistent pixels, carried across frames (transparent samples)
	PinnedBuf<float> h_frames[PL_SLOTS]; PinnedBuf<tsdrgpu_frame_result_t> h_results[PL_SLOTS]; PinnedBuf<int32_t> h_report[PL_SLOTS];
	PinnedBuf<tsdrgpu_stack_record_t> h_stack[PL_SLOTS];
	// the stack's drift report (delivery thread only): the offset at the last report or restart and the frames taken since
	double stack_ref; int stack_frames;
	std::vector<double> h_pll_rr[PL_SLOTS];            // refresh rate after frame f when the PLL moved it there (NaN: it did not)
	cudaEvent_t ev_res;                                // the batch's sync results have reached the host (PLL write-back needs them)
	SlotPool frame_slots{this, PL_SLOTS, &Stats::frames_delivered, &Stats::frames_dropped};
	// autocorrelation side path
	tsdrgpu_frd *frd; DeviceBuf<float> d_capture[2]; size_t cap_fill; int cap_phase; uint32_t cap_rate;
	PinnedBuf<double> h_plot_frame[2], h_plot_line[2];
	SlotPool plot_slots{this, 2, &Stats::plots_delivered, nullptr};
	PinnedBuf<int32_t> h_peaks[2];                     // where the two plots peak, picked on the device (8f-3)
	// superbandwidth (superb_run's state machine, superbandwidth.c:179-264)
	struct {
		int state; int buffid; long long to_gather, gathered, in_frame, to_pause; uint32_t rate;
		int nhops;                                    // SUPER_HOPS_TO_MAKE (superbandwidth.c:22): 4, or the number of devices when the hops are sharded
		DeviceBuf<float> d_out; cudaEvent_t ev;
		// hop i is recorded by rank i; ndev ranks of one hop per GPU (tsdrgpu_pipeline_set_superb_devices), or 0 in the one-GPU mode
		int ndev; std::unique_ptr<SbRank> rank[16];
		tsdrgpu_superb_mgpu_t *grp[16];               // the sharded mode's group, one member per rank, once the hop size is known
		// the round's stitch (Settings::sbd_spec at its start); coherent: the spacing D, the retune offsets, the joins' records
		tsdrgpu_superband_t spec; uint32_t d; int32_t offsets[TSDRGPU_SUPERBAND_MAX_HOPS];
		DeviceBuf<tsdrgpu_superband_est_t> d_est; int est_n;
	} sb;
	// delivery
	std::thread thread; std::mutex mu; std::condition_variable cv_job, cv_done;
	std::deque<FrameJob> jobs; int stop; uint64_t submitted, delivered;
	tsdrgpu_pipeline_stats_t stats;
};

enum { SB_STOPPED = 0, SB_STARTING, SB_GATHERING, SB_PAUSE };

int SlotPool::acquire(bool wait, uint64_t count) {
	std::unique_lock<std::mutex> g(p->mu);
	int slot;
	while ((slot = free_slot()) < 0 && wait) p->cv_done.wait(g);
	if (slot >= 0) busy[slot] = 1; else if (skipped) p->stats.*skipped += count;
	return slot;
}
void SlotPool::release(int slot, uint64_t count) {
	std::lock_guard<std::mutex> g(p->mu);
	busy[slot] = 0; p->stats.*delivered += count; p->delivered++;
	p->cv_done.notify_all();
}
// every job submitted so far has been delivered: before a pool's page-locked buffers are regrown, and by flush
static void wait_delivered(tsdrgpu_pipeline *p) {
	std::unique_lock<std::mutex> g(p->mu);
	while (p->delivered < p->submitted) p->cv_done.wait(g);
}

static void geometry(Settings &s) {                    // set_internal_samplerate, TSDRLibrary.c:540-550
	double pr, pt; int w;
	tsdrgpu_geometry(s.samplerate, s.height, s.refreshrate, &w, &pr, &pt);
	s.width = w;
	if (s.samplerate != 0 && pr != 0) s.ptos = pt;
}
static Settings settings(tsdrgpu_pipeline *p) { std::lock_guard<std::mutex> g(p->set_mu); return p->set; }
// a one-shot request (pending sync offset, PLOTS_RESET, DUMP) of the live settings: taken and cleared under the lock
template <class T> static T take_request(tsdrgpu_pipeline *p, T &field) { std::lock_guard<std::mutex> g(p->set_mu); return std::exchange(field, T(0)); }
// a change to the live settings (every setter's): with a pipeline and valid arguments, `write` runs under the lock
template <class F> static int update(tsdrgpu_pipeline *p, bool valid, F write) {
	if (!p || !valid) return TSDRGPU_EINVAL;
	std::lock_guard<std::mutex> g(p->set_mu);
	write(p->set);
	return TSDRGPU_OK;
}

static void delivery_main(tsdrgpu_pipeline *p) {
	cudaSetDevice(p->ctx->device);
	tsdrgpu_bind_thread_near_device(p->ctx);          // the frames it hands out live in page-locked memory on the device's node
	for (;;) {
		std::unique_lock<std::mutex> g(p->mu);
		while (p->jobs.empty() && !p->stop) p->cv_job.wait(g);
		if (p->jobs.empty()) break;                     // stopped, and every job delivered
		FrameJob j = p->jobs.front(); p->jobs.pop_front();
		g.unlock();
		cudaEventSynchronize(j.ev);
		if (j.kind == JOB_FRAMES) {
			const size_t n = (size_t) j.w * j.h;
			for (int f = 0; f < j.nframes; f++) {
				const tsdrgpu_frame_result_t &r = p->h_results[j.slot].ptr[f];
				// frameratepll's announce (syncdetector.c:151): the write-back itself happened in drain_frames, in stream order
				if (j.pll_valid && p->h_pll_rr[j.slot][f] == p->h_pll_rr[j.slot][f] && p->value_cb)
					p->value_cb(0 /* VALUE_ID_PLL_FRAMERATE */, p->h_pll_rr[j.slot][f], 0, p->user);
				if (p->h_report[j.slot].ptr[f] && p->value_cb) p->value_cb(3 /* VALUE_ID_AUTOGAIN_VALUES */, r.lastmin, r.lastmax, p->user);
				if (p->h_report[j.slot].ptr[f] && p->value_cb && j.snr_valid) p->value_cb(4 /* VALUE_ID_SNR: the announce dsp.c:234 leaves commented out */, r.snr, 0, p->user);
				if (j.stack_valid) {                     // the stack's drift, with the auto-gain report's cadence
					const tsdrgpu_stack_record_t &sr = p->h_stack[j.slot].ptr[f];
					if (sr.restarted) { p->stack_ref = 0.0; p->stack_frames = 0; } else p->stack_frames++;
					if (p->h_report[j.slot].ptr[f]) {
						const double drift = p->stack_frames ? (sr.offset - p->stack_ref) / p->stack_frames : 0.0;
						double at = fmod(sr.offset, (double) n);
						if (at < 0) at += (double) n;
						if (p->value_cb) p->value_cb(TSDRGPU_VALUE_ID_STACK_DRIFT, drift, at, p->user);
						p->stack_ref = sr.offset; p->stack_frames = 0;
					}
				}
				if (p->frame_cb) p->frame_cb(p->h_frames[j.slot].ptr + f * n, j.w, j.h, p->user);
			}
		} else if (j.kind == JOB_PLOTS) {
			if (j.reset_announce && p->value_cb) p->value_cb(1 /* VALUE_ID_AUTOCORRECT_RESET */, 0, 0, p->user);
			if (j.dump_announce && p->value_cb) p->value_cb(5 /* VALUE_ID_AUTOCORRECT_DUMPED, frameratedetector.c:115 */, 0, 0, p->user);
			if (p->plot_cb) {
				p->plot_cb(0 /* PLOT_ID_FRAME */, j.foff, p->h_plot_frame[j.slot].ptr, j.flen, j.samplerate, p->user);
				p->plot_cb(1 /* PLOT_ID_LINE */, j.loff, p->h_plot_line[j.slot].ptr, j.llen, j.samplerate, p->user);
			}
			if (p->value_cb) p->value_cb(2 /* VALUE_ID_AUTOCORRECT_FRAMES_COUNT */, 0, (double) j.calls, p->user);
			if (j.detect_mode && p->value_cb && j.flen > 0 && j.llen > 0) {
				double fps = 0; int height = 0;
				tsdrgpu_detect_videomode(p->h_plot_frame[j.slot].ptr, j.foff, j.flen, p->h_plot_line[j.slot].ptr, j.loff, j.llen, j.samplerate, &fps, &height, NULL, NULL);
				p->value_cb(TSDRGPU_VALUE_ID_DETECTED_MODE, fps, (double) height, p->user);
			}
		} else if (p->plot_cb) p->plot_cb(j.plot_id, -j.report_n / 2, j.report, j.report_n, j.samplerate, p->user);
		cudaEventDestroy(j.ev);
		j.pool->release(j.slot, j.kind == JOB_FRAMES ? (uint64_t) j.nframes : 1);
	}
}

static int submit(tsdrgpu_pipeline *p, FrameJob &j, cudaStream_t on) {
	CU_TRY(p->ctx, cudaEventCreateWithFlags(&j.ev, cudaEventDisableTiming));
	CU_TRY(p->ctx, cudaEventRecord(j.ev, on));
	std::lock_guard<std::mutex> g(p->mu);
	p->jobs.push_back(j); p->submitted++;
	p->cv_job.notify_one();
	return TSDRGPU_OK;
}

// room for `more` samples behind the ones waiting in the decimator input (contents kept); returns where they go
static int decim_reserve(tsdrgpu_pipeline *p, size_t more, float **where) {
	const size_t E = (size_t) p->decim_elem, used = E * (p->decim_read + p->decim_fill);
	CU_TRY(p->ctx, p->d_decim.reserve(p->s_main, used + E * more, used));
	*where = p->d_decim.ptr + used;
	return TSDRGPU_OK;
}
// the decimator input switches between I,Q pairs and magnitudes: what is still waiting is converted (rare: at most a few
// blocks, when superbandwidth mode with one hop per GPU starts or ends)
static int decim_set_elem(tsdrgpu_pipeline *p, int elem) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	if (p->decim_elem == elem) return TSDRGPU_OK;
	CU_TRY(ctx, cudaStreamSynchronize(p->s_ingest));
	const size_t n = p->decim_fill;
	int rc;
	if (n) {
		void *tmp;
		float *src = p->d_decim.ptr + (size_t) p->decim_elem * p->decim_read;
		if ((rc = tsdrgpu_scratch(ctx, 3, sizeof(float) * 2 * n, &tmp))) return rc;
		if (elem == 1) {                                  // pairs -> magnitudes (am_demod, TSDRLibrary.c:244-262)
			if ((rc = tsdrgpu_am_demod(ctx, p->s_main, src, n, (float *) tmp))) return rc;
			CU_TRY(ctx, cudaMemcpyAsync(p->d_decim.ptr, tmp, sizeof(float) * n, cudaMemcpyDeviceToDevice, p->s_main));
		} else {                                          // magnitudes -> pairs (m, 0): |(m, 0)| == m
			CU_TRY(ctx, cudaMemsetAsync(tmp, 0, sizeof(float) * 2 * n, p->s_main));
			CU_TRY(ctx, cudaMemcpy2DAsync(tmp, 2 * sizeof(float), src, sizeof(float), sizeof(float), n, cudaMemcpyDeviceToDevice, p->s_main));
			CU_TRY(ctx, p->d_decim.reserve(p->s_main, 2 * n));
			CU_TRY(ctx, cudaMemcpyAsync(p->d_decim.ptr, tmp, sizeof(float) * 2 * n, cudaMemcpyDeviceToDevice, p->s_main));
		}
		CU_TRY(ctx, cudaEventRecord(p->ev_decim, p->s_main));
	}
	p->decim_read = 0; p->decim_elem = elem;
	return TSDRGPU_OK;
}

// A plugin hands over the same malloc'd buffer call after call (TSDRPlugin_RawFile.c:212, Mirics, SDRplay).  From pageable memory
// cudaMemcpyAsync goes through the driver's staging buffer at a fraction of the link rate; once a buffer has come back
// REG_AFTER times it is page-locked in place.  Buffers are released again when the run ends (tsdrgpu_pipeline_destroy).
// OPT-IN (tsdrgpu_pipeline_set_host_registration): a registration pins the PHYSICAL pages behind an address range, so it is
// only safe for a caller that keeps its buffer mapped for the whole run, as the reference's plugins do (one malloc per
// tsdrplugin_readasync).  A caller that frees and re-allocates a buffer per call (numpy temporaries land on the same address
// again and again) would be read through the stale mapping -- measured: wrong frames, then cudaErrorInvalidValue.  The C host
// library switches it on for the plugins it loads (TSDR_NO_HOST_REGISTER=1 keeps it off).
static const void *host_source(tsdrgpu_pipeline *p, bool host_register, const void *h, size_t bytes) {
	constexpr int REG_AFTER = 3;
	if (!host_register || bytes < 65536 || h == NULL) return h;
	for (auto &b : p->hostbufs) {
		if (b.base != h) continue;
		if (b.state == 1 && bytes > b.bytes) { cudaHostUnregister(const_cast<void *>(b.base)); cudaGetLastError(); b.state = 0; b.seen = REG_AFTER - 1; }
		if (b.state != 0) return h;
		if (++b.seen < REG_AFTER) return h;
		cudaPointerAttributes a;
		if (cudaPointerGetAttributes(&a, h) == cudaSuccess && a.type != cudaMemoryTypeUnregistered) { b.state = 2; return h; }
		cudaGetLastError();
		if (cudaHostRegister(const_cast<void *>(h), bytes, cudaHostRegisterDefault) == cudaSuccess) { b.state = 1; b.bytes = bytes; p->stats.host_buffers_registered++; }
		else { cudaGetLastError(); b.state = 3; }
		return h;
	}
	if (p->hostbufs.size() >= 8) {
		if (p->hostbufs.front().state == 1) { cudaHostUnregister(const_cast<void *>(p->hostbufs.front().base)); cudaGetLastError(); }
		p->hostbufs.erase(p->hostbufs.begin());
	}
	p->hostbufs.push_back({h, bytes, 1, 0});
	return h;
}

// ---- autocorrelation side path: append demodulated samples, fire a capture when full (frameratedetector.c:128-230)
static int feed_capture(tsdrgpu_pipeline *p, const Settings &s, const float *d_iq, uint64_t pairs, bool dropped) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	if (s.params[TSDRGPU_PARAM_AUTOCORR_PLOTS_OFF]) return TSDRGPU_OK;
	if (dropped) { p->cap_fill = 0; return TSDRGPU_OK; }              // cb_purge on any drop
	if (p->cap_rate != s.samplerate) { p->cap_rate = s.samplerate; p->cap_fill = 0; }
	const size_t want = tsdrgpu_frd_capture_size(s.samplerate);
	if (want == 0) return TSDRGPU_OK;
	int rc;
	for (int i = 0; i < 2; i++) if (p->d_capture[i].cap < want) {
		CU_TRY(ctx, cudaStreamSynchronize(p->s_ingest));
		CU_TRY(ctx, p->d_capture[i].reserve(p->s_main, want, (i == p->cap_phase) ? p->cap_fill : 0));
	}
	uint64_t done = 0;
	while (done < pairs) {
		const uint64_t take = (want - p->cap_fill) < (pairs - done) ? (want - p->cap_fill) : (pairs - done);
		float *cap = p->d_capture[p->cap_phase].ptr;
		if (p->cap_fill == 0) CU_TRY(ctx, cudaStreamWaitEvent(p->s_ingest, p->ev_cap_used[p->cap_phase], 0));   // the FFT that last read it is done
		if ((rc = tsdrgpu_am_demod(ctx, p->s_ingest, d_iq + 2 * done, take, cap + p->cap_fill))) return rc;
		p->cap_fill += take; done += take;
		if (p->cap_fill == want) {
			p->cap_fill = 0;
			const int cph = p->cap_phase; p->cap_phase ^= 1;
			CU_TRY(ctx, cudaEventRecord(p->ev_ingest, p->s_ingest));
			CU_TRY(ctx, cudaStreamWaitEvent(p->s_main, p->ev_ingest, 0));
			int reset_announce = 0;
			if (const uint32_t reset = take_request(p, p->set.params[TSDRGPU_PARAM_AUTOCORR_PLOTS_RESET])) {  // frameratedetector.c:97-104
				reset_announce = (reset == 1);
				tsdrgpu_frd_reset(p->frd);
			}
			int fmin, fmax, lmin, lmax;
			tsdrgpu_frd_windows(s.samplerate, &fmin, &fmax, &lmin, &lmax);
			const size_t need = (size_t) (fmax - fmin) + 8;
			// a free plot slot; when the host is slower than the GPU the capture is still accumulated on
			// the device, only this particular plot delivery is skipped
			const int slot = p->plot_slots.acquire(false, 1);
			// too small, or left empty by a failed re-allocation
			if (p->plot_slots.any([&](int k) { return p->h_plot_frame[k].cap < need || p->h_plot_line[k].cap < need || !p->h_peaks[k].ptr; })) {
				CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
				wait_delivered(p);
				for (int k = 0; k < 2; k++) {
					if ((rc = p->h_peaks[k].assign(ctx, 16))) return rc;
					if ((rc = p->h_plot_frame[k].assign(ctx, need))) return rc;
					if ((rc = p->h_plot_line[k].assign(ctx, need))) return rc;
				}
			}
			int dump_announce = 0;
			if (take_request(p, p->set.params[TSDRGPU_PARAM_AUTOCORR_DUMP])) {        // frameratedetector.c:110-116: "autocorr.csv" in the working directory
				if ((rc = tsdrgpu_frd_dump_csv(p->frd, p->s_main, s.samplerate, cap, (uint32_t) want, "autocorr.csv"))) return rc;
				dump_announce = 1;
			}
			uint64_t calls = 0;
			if ((rc = tsdrgpu_frd_run_async(p->frd, p->s_main, s.samplerate, cap, (uint32_t) want,
			                                slot >= 0 ? p->h_plot_frame[slot].ptr : NULL, fmax - fmin,
			                                slot >= 0 ? p->h_plot_line[slot].ptr : NULL, lmax - lmin, &calls))) return rc;
			if (slot >= 0 && (rc = tsdrgpu_frd_peaks_async(p->frd, p->s_main, p->h_peaks[slot].ptr))) return rc;
			CU_TRY(ctx, cudaEventRecord(p->ev_cap_used[cph], p->s_main));
			p->stats.captures++;
			if (slot >= 0) {
				FrameJob j{JOB_PLOTS, &p->plot_slots, slot, s.samplerate};
				j.foff = fmin; j.flen = fmax - fmin; j.loff = lmin; j.llen = lmax - lmin;
				j.calls = calls; j.reset_announce = reset_announce; j.dump_announce = dump_announce; j.detect_mode = s.detect_mode;
				if ((rc = submit(p, j, p->s_main))) return rc;
			}
		}
	}
	return TSDRGPU_OK;
}

// ---- pixels -> frames (postprocessingthread + videodecodingthread), with the settings of the group of blocks that made them
static int drain_frames(tsdrgpu_pipeline *p, const Settings &s) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	const int w = s.width, h = s.height;
	const size_t n = (size_t) w * h;
	int rc;
	const int batch = p->cfg.batch_frames > 0 ? p->cfg.batch_frames : 1;
	while (p->pix_fill - p->pix_read >= n * (size_t) batch) {
		const int nf = batch;
		// a free delivery slot, or the batch is dropped whole (frames stay aligned), as a full ring would (circbuff.c:95-104)
		const int slot = p->frame_slots.acquire(p->cfg.block_when_busy, (uint64_t) nf);
		if (slot < 0) { p->pix_read += n * nf; continue; }
		// too small, or left empty by a failed re-allocation
		if (p->frame_slots.any([&](int k) { return p->h_frames[k].cap < n * nf || !p->h_results[k].ptr || !p->h_report[k].ptr || !p->h_stack[k].ptr; })) {
			CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
			wait_delivered(p);
			for (int k = 0; k < PL_SLOTS; k++) {
				p->h_pll_rr[k] = std::vector<double>(nf);
				if ((rc = p->h_frames[k].assign(ctx, n * nf))) return rc;
				if ((rc = p->h_results[k].assign(ctx, nf))) return rc;
				if ((rc = p->h_report[k].assign(ctx, nf))) return rc;
				if ((rc = p->h_stack[k].assign(ctx, nf))) return rc;
			}
		}
		const int op = p->out_phase; p->out_phase ^= 1;
		CU_TRY(ctx, p->d_frames[op].reserve(p->s_main, n * nf));
		CU_TRY(ctx, cudaStreamWaitEvent(p->s_main, p->ev_out[op], 0));       // the D2H that last read this buffer is done
		unsigned flags = 0;
		if (s.params[TSDRGPU_PARAM_INT_AUTOSHIFT]) flags |= TSDRGPU_FS_AUTOSHIFT;
		if (s.params[TSDRGPU_PARAM_LOW_PASS_BEFORE_SYNC]) flags |= TSDRGPU_FS_LOWPASS_BEFORE_SYNC;
		if (s.params[TSDRGPU_PARAM_AUTOGAIN_AFTER_PROCESSING]) flags |= TSDRGPU_FS_AUTOGAIN_AFTER_PROC;
		if (s.params[TSDRGPU_PARAM_AUTOCORR_SUPERRESOLUTION]) flags |= TSDRGPU_FS_SUPERRESOLUTION;
		if (s.report_snr) flags |= TSDRGPU_FS_COMPUTE_SNR;
		if ((rc = tsdrgpu_framestage_set_autogain(p->fs, s.ag_mode, s.ag_ppm))) return rc;
		if ((rc = tsdrgpu_framestage_set_contrast(p->fs, s.ct_mode, s.ct_clip, s.ct_tx, s.ct_ty))) return rc;
		if ((rc = tsdrgpu_framestage_set_denoise(p->fs, s.nl_mode, s.nl_h, s.nl_r, s.nl_p))) return rc;
		if ((rc = tsdrgpu_framestage_set_stack(p->fs, s.st_mode, s.st_depth, s.st_rx, s.st_ry))) return rc;
		if ((rc = tsdrgpu_framestage_set_deblur(p->fs, s.db_mode, s.db_sigma, s.db_iters))) return rc;
		const bool stack_on = s.st_mode != TSDRGPU_STACK_OFF;
		if ((rc = framestage_stack_next(p->fs, take_request(p, p->set.stack_restart), stack_on ? p->h_stack[slot].ptr : NULL))) return rc;
		if ((rc = tsdrgpu_framestage_run_async(p->fs, p->s_main, p->d_pix.ptr + p->pix_read, nf, w, h, s.motionblur,
		                                       0.1f /* NORMALISATION_LOWPASS_COEFF, TSDRLibrary.c:37 */, flags, p->d_frames[op].ptr,
		                                       p->h_results[slot].ptr, p->h_report[slot].ptr))) return rc;
		// the frames become valid on the frame stage's side stream: copy them out on the output stream behind it
		CU_TRY(ctx, cudaEventRecord(p->ev_main, p->s_main));
		CU_TRY(ctx, cudaStreamWaitEvent(p->s_out, p->ev_main, 0));             // serial stage orders finish on the main stream
		if ((rc = tsdrgpu_framestage_join(p->fs, p->s_out))) return rc;        // the overlapped order finishes on the side stream
		const bool pll_on = s.params[TSDRGPU_PARAM_INT_FRAMERATE_PLL] != 0;
		if (pll_on) CU_TRY(ctx, cudaEventRecord(p->ev_res, p->s_out));          // the batch's results are on the host behind this
		if (s.argb_mode) {                                                     // float frames -> the host's int32 pixels, in place
			if (p->d_argb_last.cap != n) {
				CU_TRY(ctx, p->d_argb_last.assign(n));
				CU_TRY(ctx, cudaMemsetAsync(p->d_argb_last.ptr, 0, sizeof(int32_t) * n, p->s_out));
			}
			if ((rc = tsdrgpu_pixels_argb_batch(ctx, p->s_out, p->d_frames[op].ptr, n, nf, s.argb_inverted, p->d_argb_last.ptr))) return rc;
		}
		CU_TRY(ctx, cudaMemcpyAsync(p->h_frames[slot].ptr, p->d_frames[op].ptr, sizeof(float) * n * nf, cudaMemcpyDeviceToHost, p->s_out));
		CU_TRY(ctx, cudaEventRecord(p->ev_out[op], p->s_out));
		p->stats.d2h_bytes += sizeof(float) * n * nf;
		p->pix_read += n * nf;
		p->stats.frames_processed += nf;
		FrameJob j{JOB_FRAMES, &p->frame_slots, slot, 0, nf, w, h};
		j.snr_valid = s.report_snr; j.pll_valid = pll_on; j.stack_valid = stack_on;
		if (pll_on) {
			// frameratepll's write-back (syncdetector.c:141-152).  The reference does it from its post-processing thread while the
			// decimating thread reads refreshrate unlocked (SURVEY F9); here it is applied in stream order: the results of this
			// batch move the refresh rate before the decimator plans its next group of blocks, frame by frame in order.  The
			// price is one host wait per batch, paid only while the PLL is switched on (the frames' D2H is already queued).
			CU_TRY(ctx, cudaEventSynchronize(p->ev_res));
			for (int f = 0; f < nf; f++) {
				const tsdrgpu_frame_result_t &r = p->h_results[slot].ptr[f];
				std::lock_guard<std::mutex> g(p->set_mu);
				double rr = p->set.refreshrate;
				const int moved = tsdrgpu_pll_step(&rr, r.x_vx, r.pll_state, r.avg_speed);
				if (moved) { p->set.refreshrate = rr; geometry(p->set); }
				p->h_pll_rr[slot][f] = moved ? rr : nan("");
			}
		}
		if ((rc = submit(p, j, p->s_out))) return rc;
	}
	// compact the pixel buffer when the consumed prefix is large
	if (p->pix_read > 0 && p->pix_read >= (p->pix_fill - p->pix_read)) {
		const size_t left = p->pix_fill - p->pix_read;
		if (left) {
			pl_copy_f32<<<(unsigned) ((left + 255) / 256 < 1024 ? (left + 255) / 256 : 1024), 256, 0, p->s_main>>>(p->d_pix.ptr + p->pix_read, p->d_pix.ptr, left);
			LAUNCH_CHECK(ctx);
		}
		p->pix_read = 0; p->pix_fill = left;
	}
	return TSDRGPU_OK;
}

// ---- samples -> pixels (decimatingthread)
static int drain_blocks(tsdrgpu_pipeline *p) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	int rc;
	for (;;) {
		// the settings, read again for every group of blocks: the PLL (drain_frames) or the host may have moved the geometry
		const Settings s = settings(p);
		const int w = s.width, h = s.height; const double fv = s.refreshrate; const uint32_t fs_ = s.samplerate;
		if (w <= 0 || h <= 0) return TSDRGPU_OK;
		const uint32_t block = (uint32_t) (0.1 * fs_ / fv);                 // FRAMES_TO_POLL, TSDRLibrary.c:41,335
		if (block == 0) return TSDRGPU_OK;
		const uint32_t min_blocks = p->cfg.batch_blocks > 0 ? (uint32_t) p->cfg.batch_blocks : 10;
		if (p->decim_fill / block < min_blocks) return TSDRGPU_OK;
		// whole multiples of the batch size, so the grouping (and with it every result) does not depend on how the
		// plugin happened to cut the stream into process() calls; with the PLL on exactly one group at a time, because the
		// frames it completes may move the refresh rate the next group is resampled with
		uint32_t nb = (uint32_t) ((p->decim_fill / block / min_blocks) * min_blocks);
		if (nb > 4000) nb = (4000 / min_blocks) * min_blocks;
		if (nb == 0 || s.params[TSDRGPU_PARAM_INT_FRAMERATE_PLL]) nb = min_blocks;
		const double up = (double) (w * h) * fv;        // width*height*refreshrate, TSDRLibrary.c:340
		const uint64_t npix = tsdrgpu_resampler_plan(p->rs, NULL, block, nb, up, (double) fs_);
		if (npix == 0) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "resampler plan produced no pixels", cudaSuccess, __FILE__, __LINE__);
		CU_TRY(ctx, p->d_pix.reserve(p->s_main, p->pix_fill + npix + 64, p->pix_fill));
		uint64_t n_out = 0;
		if ((rc = tsdrgpu_resampler_set_kernel(p->rs, s.rs_kernel))) return rc;
		if ((rc = tsdrgpu_resampler_run(p->rs, p->s_main, p->d_decim.ptr + (size_t) p->decim_elem * p->decim_read, p->decim_elem == 2, NULL, block, nb, up, (double) fs_,
		                                (int) s.params[TSDRGPU_PARAM_NEAREST_NEIGHBOUR_RESAMPLING], p->d_pix.ptr + p->pix_fill,
		                                p->d_pix.cap - p->pix_fill, &n_out))) return rc;
		// pixel-level alignment (dsp.c:326-346 on the pixel ring) and manual sync (TSDRLibrary.c:344-346)
		const uint32_t totalpixels = (uint32_t) (w * h);
		uint32_t skip = 0;
		const uint32_t fwd = p->pix_drop.add((uint32_t) n_out, totalpixels, true, &skip);
		if (skip && fwd) {                               // rare (after drops / manual sync): shift through scratch, ranges overlap
			void *tmp;
			if ((rc = tsdrgpu_scratch(ctx, 3, sizeof(float) * fwd, &tmp))) return rc;
			const unsigned g = (unsigned) ((fwd + 255) / 256 < 1024 ? (fwd + 255) / 256 : 1024);
			pl_copy_f32<<<g, 256, 0, p->s_main>>>(p->d_pix.ptr + p->pix_fill + skip, (float *) tmp, fwd); LAUNCH_CHECK(ctx);
			pl_copy_f32<<<g, 256, 0, p->s_main>>>((const float *) tmp, p->d_pix.ptr + p->pix_fill, fwd); LAUNCH_CHECK(ctx);
		}
		p->pix_fill += fwd;
		p->pix_drop.shift_with(totalpixels, -(int64_t) take_request(p, p->set.syncoffset));
		// consume the blocks; move what is left to the front once the hole there is big enough for a non-overlapping move
		const size_t used = (size_t) nb * block, left = p->decim_fill - used, E = (size_t) p->decim_elem;
		p->decim_read += used; p->decim_fill = left;
		if (left == 0) p->decim_read = 0;
		else if (p->decim_read >= left) {
			pl_copy_f32<<<(unsigned) ((E * left + 255) / 256 < 1024 ? (E * left + 255) / 256 : 1024), 256, 0, p->s_main>>>(p->d_decim.ptr + E * p->decim_read, p->d_decim.ptr, E * left); LAUNCH_CHECK(ctx);
			p->decim_read = 0;
		}
		CU_TRY(ctx, cudaEventRecord(p->ev_decim, p->s_main));                // later appends (ingest stream) must come after this
		p->stats.samples_resampled += used;
		if ((rc = drain_frames(p, s))) return rc;
	}
}

// One report path over a whole converted block on s_spec (after ev_conv), its reports queued for delivery in free slots of its pool.
// N == 0 (a geometry the path cannot resolve): no reports, and a new one once it can.  set(obj): this block's settings.
template <class Obj, class Create, class Reset, class Plan, class Run, class Set>
static int report_block(tsdrgpu_pipeline *p, ReportPath<Obj> &r, size_t N, Create create, Reset reset, Plan plan, Run run, Set set,
                        uint32_t samplerate, const float *stage, uint64_t pairs, bool dropped) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	int rc;
	if (N == 0) { r.fresh = 1; return TSDRGPU_OK; }
	if (!r.obj && (rc = create(ctx, &r.obj))) return rc;
	if ((rc = set(r.obj)) || (r.fresh && (rc = reset(r.obj)))) return rc;
	r.fresh = 0;
	uint32_t nrep = 0;
	if ((rc = plan(r.obj, pairs, dropped, &nrep))) return rc;
	CU_TRY(ctx, r.d_out.reserve(p->s_spec, nrep * N));              // grows behind s_spec's last use of the old buffer
	if (nrep && r.pool.any([&](int k) { return r.h[k].cap < N; })) {        // too small, or left empty by a failed re-allocation
		wait_delivered(p);
		for (int k = 0; k < PL_SLOTS; k++) if ((rc = r.h[k].assign(ctx, N))) return rc;
	}
	if ((rc = run(r.obj, p->s_spec, stage, pairs, dropped, r.d_out.ptr, nrep, &nrep))) return rc;
	for (uint32_t i = 0; i < nrep; i++) {
		const int slot = r.pool.acquire(false, 1);
		if (slot < 0) continue;
		CU_TRY(ctx, cudaMemcpyAsync(r.h[slot].ptr, r.d_out.ptr + i * N, sizeof(double) * N, cudaMemcpyDeviceToHost, p->s_spec));
		p->stats.d2h_bytes += sizeof(double) * N;
		FrameJob j{JOB_REPORT, &r.pool, slot, samplerate, 0, 0, 0, r.plot_id, (int) N, r.h[slot].ptr};
		if ((rc = submit(p, j, p->s_spec))) return rc;
	}
	return TSDRGPU_OK;
}

extern "C" {

// the error a superbandwidth rank's own context holds (NULL: the thread's, where tsdrgpu_create leaves it), in the pipeline's
static int rank_error(tsdrgpu_pipeline *p, tsdrgpu_ctx_t *from, int rc) { if (from != p->ctx) snprintf(p->ctx->err, sizeof p->ctx->err, "%s", tsdrgpu_last_error(from)); return rc; }
// the sharded mode's ranks >= 1: a context of its own on devices[i], and streams and an event there (rank 0 is made with the hops)
static int superb_ranks(tsdrgpu_pipeline *p, const int *devices, int n) {
	for (int i = 1; i < n; i++) {
		SbRank &r = *(p->sb.rank[i] = std::make_unique<SbRank>());
		if (const int rc = tsdrgpu_create(&r.own.c, devices[i])) return rank_error(p, NULL, rc);
		r.dev = devices[i]; r.ctx = r.own.c; CU_TRY(p->ctx, cudaSetDevice(r.dev));
		CU_TRY(p->ctx, cudaStreamCreateWithFlags(&r.stream, cudaStreamNonBlocking)); CU_TRY(p->ctx, cudaStreamCreateWithFlags(&r.copy, cudaStreamNonBlocking));
		CU_TRY(p->ctx, cudaEventCreateWithFlags(&r.ev, cudaEventDisableTiming));
	}
	CU_TRY(p->ctx, cudaSetDevice(p->ctx->device));
	return TSDRGPU_OK;
}
// back to the one-GPU mode, stopped: the group first (its windows are cross-linked), then the ranks; ends on the pipeline's device
static void superb_release(tsdrgpu_pipeline *p) {
	for (auto &g : p->sb.grp) { tsdrgpu_superb_mgpu_destroy(g); g = NULL; }
	for (auto &r : p->sb.rank) r.reset();
	p->sb.ndev = 0; p->sb.rate = 0; p->sb.state = SB_STOPPED;
	cudaSetDevice(p->ctx->device);
}

// the pipeline's own streams and events, for create and release alike
static std::vector<cudaStream_t *> own_streams(tsdrgpu_pipeline *p) { return {&p->s_main, &p->s_copy, &p->s_out, &p->s_ingest}; }
static std::vector<cudaEvent_t *> own_events(tsdrgpu_pipeline *p) {
	return {&p->ev_ingest, &p->ev_decim, &p->ev_cap_used[0], &p->ev_cap_used[1], &p->ev_out[0], &p->ev_out[1], &p->ev_main, &p->ev_res, &p->sb.ev,
	        &p->ev_h2d[0], &p->ev_h2d[1], &p->ev_h2d[2], &p->ev_h2d[3], &p->ev_used[0], &p->ev_used[1], &p->ev_used[2], &p->ev_used[3],
	        &p->ev_conv, &p->ev_sp_used[0], &p->ev_sp_used[1], &p->ev_sp_used[2], &p->ev_sp_used[3]};
}

static int create_handles(tsdrgpu_pipeline *p) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	for (cudaStream_t *s : own_streams(p)) CU_TRY(ctx, cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
	for (cudaEvent_t *e : own_events(p)) CU_TRY(ctx, cudaEventCreateWithFlags(e, cudaEventDisableTiming));
	// the spectrum is background work (a report every 100 ms of stream): the block scheduler serves the pixel path first
	int lo = 0, hi = 0;
	CU_TRY(ctx, cudaDeviceGetStreamPriorityRange(&lo, &hi));
	CU_TRY(ctx, cudaStreamCreateWithPriority(&p->s_spec, cudaStreamNonBlocking, lo));
	int rc;
	if ((rc = tsdrgpu_resampler_create(ctx, &p->rs))) return rc;
	if ((rc = tsdrgpu_framestage_create(ctx, &p->fs))) return rc;
	tsdrgpu_framestage_set_overlap(p->fs, 1);
	return tsdrgpu_frd_create(ctx, &p->frd);
}

// everything a pipeline holds, whole or half built (null handles are skipped); its buffers go with the object.  The delivery
// thread must not be running and the pipeline's device must be current.
static void release(tsdrgpu_pipeline *p) {
	tsdrgpu_resampler_destroy(p->rs); tsdrgpu_framestage_destroy(p->fs); tsdrgpu_frd_destroy(p->frd); tsdrgpu_chanfilt_destroy(p->cf);
	tsdrgpu_spectrum_destroy(p->spec.obj); tsdrgpu_coherence_destroy(p->coh.obj);
	for (auto &b : p->hostbufs) if (b.state == 1) { cudaHostUnregister(const_cast<void *>(b.base)); cudaGetLastError(); }
	superb_release(p);
	for (cudaStream_t *s : own_streams(p)) if (*s) cudaStreamDestroy(*s);
	if (p->s_spec) cudaStreamDestroy(p->s_spec);
	for (cudaEvent_t *e : own_events(p)) if (*e) cudaEventDestroy(*e);
	delete p;
}

int tsdrgpu_pipeline_create(tsdrgpu_ctx_t *ctx, const tsdrgpu_pipeline_config_t *cfg, tsdrgpu_frame_cb frame_cb,
                            tsdrgpu_value_cb value_cb, tsdrgpu_plot_cb plot_cb, void *user, tsdrgpu_pipeline_t **out) {
	BIND(ctx); ARG_TRY(ctx, cfg != NULL && out != NULL);
	ARG_TRY(ctx, cfg->samplerate > 0 && cfg->height > 0 && cfg->refreshrate > 0);
	tsdrgpu_pipeline *p = new tsdrgpu_pipeline();      // value-initialised: every field not set here starts at zero
	p->ctx = ctx; p->cfg = *cfg; p->frame_cb = frame_cb; p->value_cb = value_cb; p->plot_cb = plot_cb; p->user = user;
	Settings &s = p->set;
	s.samplerate = s.samplerate_real = cfg->samplerate; s.height = cfg->height; s.refreshrate = cfg->refreshrate; s.motionblur = cfg->motionblur;
	memcpy(s.params, cfg->params_int, sizeof s.params);
	geometry(s);
	const int rc = create_handles(p);
	if (rc) { release(p); return rc; }
	p->thread = std::thread(delivery_main, p);
	*out = p;
	return TSDRGPU_OK;
}

int tsdrgpu_pipeline_flush(tsdrgpu_pipeline_t *p) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, p != NULL);
	BIND(p->ctx);
	for (cudaStream_t st : {p->s_copy, p->s_ingest, p->s_main, p->s_out, p->s_spec}) CU_TRY(p->ctx, cudaStreamSynchronize(st));
	wait_delivered(p);
	return TSDRGPU_OK;
}

void tsdrgpu_pipeline_destroy(tsdrgpu_pipeline_t *p) {
	if (!p) return;
	tsdrgpu_pipeline_flush(p);
	{ std::lock_guard<std::mutex> g(p->mu); p->stop = 1; p->cv_job.notify_all(); }
	p->thread.join();
	cudaSetDevice(p->ctx->device);
	release(p);
}

int tsdrgpu_pipeline_set_param_int(tsdrgpu_pipeline_t *p, int id, uint32_t value) {
	return update(p, id >= 0 && id < 9, [&](Settings &s) { s.params[id] = value; });
}
int tsdrgpu_pipeline_set_resolution(tsdrgpu_pipeline_t *p, int height, double refreshrate) {
	return update(p, height > 0 && refreshrate > 0, [&](Settings &s) { s.height = height; s.refreshrate = refreshrate; geometry(s); });
}
int tsdrgpu_pipeline_set_samplerate(tsdrgpu_pipeline_t *p, uint32_t samplerate) {
	return update(p, samplerate != 0, [&](Settings &s) { s.samplerate = samplerate; s.samplerate_real = samplerate; geometry(s); });
}
// superbandwidth with one hop per GPU: devices[0] must be the pipeline's own device; n in {2, 4, 8} = number of hops.  n <= 1
// returns to the one-GPU mode (4 hops).  Call while no superbandwidth round is in flight (before PARAM_AUTOCORR_SUPERRESOLUTION
// is switched on).  The same device may be listed more than once (test set-ups on a single GPU).
int tsdrgpu_pipeline_set_superb_devices(tsdrgpu_pipeline_t *p, const int *devices, int n) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, p != NULL);
	tsdrgpu_ctx_t *ctx = p->ctx;
	BIND(ctx);
	if (n > 1 && settings(p).sbd_spec.mode == TSDRGPU_SUPERBAND_COHERENT)
		return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "the coherent superbandwidth stitch runs on one GPU: set the reference stitch before sharding the hops", cudaSuccess, __FILE__, __LINE__);
	CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
	superb_release(p);
	if (n <= 1) return TSDRGPU_OK;
	ARG_TRY(ctx, devices != NULL && (n == 2 || n == 4 || n == 8) && devices[0] == ctx->device);
	const int rc = superb_ranks(p, devices, n);
	if (rc) superb_release(p); else p->sb.ndev = n;     // a failure leaves the one-GPU mode, its error text in ctx
	return rc;
}
int tsdrgpu_pipeline_set_superband(tsdrgpu_pipeline_t *p, const tsdrgpu_superband_t *spec) {
	if (!p) return TSDRGPU_EINVAL;
	tsdrgpu_superband_t b = {TSDRGPU_SUPERBAND_REFERENCE, 0, 0};
	if (spec && spec->mode != TSDRGPU_SUPERBAND_REFERENCE) {
		if (!superband_ok(spec)) return tsdrgpu_fail(p->ctx, TSDRGPU_EINVAL, "invalid superband spec (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
		if (p->sb.ndev > 1)
			return tsdrgpu_fail(p->ctx, TSDRGPU_EINVAL, "the coherent superbandwidth stitch runs on one GPU: return to one device (set_superb_devices with n <= 1) first", cudaSuccess, __FILE__, __LINE__);
		b = *spec;
	}
	return update(p, true, [&](Settings &s) { s.sbd_spec = b; });
}
int tsdrgpu_pipeline_superband_estimates(tsdrgpu_pipeline_t *p, tsdrgpu_superband_est_t *out, int cap, int *n) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, p != NULL && n != NULL);
	tsdrgpu_ctx_t *ctx = p->ctx;
	BIND(ctx);
	ARG_TRY(ctx, p->sb.est_n == 0 || (out != NULL && cap >= p->sb.est_n));
	CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
	if (p->sb.est_n) CU_TRY(ctx, cudaMemcpy(out, p->sb.d_est.ptr, sizeof(tsdrgpu_superband_est_t) * p->sb.est_n, cudaMemcpyDeviceToHost));
	*n = p->sb.est_n;
	return TSDRGPU_OK;
}
int tsdrgpu_pipeline_set_host_registration(tsdrgpu_pipeline_t *p, int on) { return update(p, true, [&](Settings &s) { s.host_register = on != 0; }); }
int tsdrgpu_pipeline_set_retune(tsdrgpu_pipeline_t *p, tsdrgpu_retune_cb cb) { return update(p, true, [&](Settings &s) { s.retune_cb = cb; }); }
int tsdrgpu_pipeline_set_motionblur(tsdrgpu_pipeline_t *p, float coeff) { return update(p, true, [&](Settings &s) { s.motionblur = coeff; }); }
int tsdrgpu_pipeline_set_output_argb(tsdrgpu_pipeline_t *p, int mode, int inverted) {
	return update(p, true, [&](Settings &s) { s.argb_mode = mode != 0; s.argb_inverted = inverted != 0; });
}
int tsdrgpu_pipeline_set_reports(tsdrgpu_pipeline_t *p, int report_snr, int detect_mode) {
	return update(p, true, [&](Settings &s) { s.report_snr = report_snr != 0; s.detect_mode = detect_mode != 0; });
}
int tsdrgpu_pipeline_set_resampler(tsdrgpu_pipeline_t *p, int kernel) {
	return update(p, kernel == TSDRGPU_RS_BOX || kernel == TSDRGPU_RS_SINC, [&](Settings &s) { s.rs_kernel = kernel; });
}
int tsdrgpu_pipeline_set_autogain(tsdrgpu_pipeline_t *p, int mode, int ppm) {
	return update(p, autogain_ok(mode, ppm), [&](Settings &s) { s.ag_ppm = ppm; s.ag_mode = mode; });
}
int tsdrgpu_pipeline_set_contrast(tsdrgpu_pipeline_t *p, int mode, int clip_centi, int tx, int ty) {
	return update(p, contrast_ok(mode, clip_centi, tx, ty), [&](Settings &s) {
		if (mode == TSDRGPU_CONTRAST_CLAHE) { s.ct_clip = clip_centi; s.ct_tx = tx; s.ct_ty = ty; }
		s.ct_mode = mode;
	});
}
int tsdrgpu_pipeline_set_channel(tsdrgpu_pipeline_t *p, const tsdrgpu_channel_t *spec) {
	if (!p) return TSDRGPU_EINVAL;
	tsdrgpu_channel_t c = {};
	if (spec && spec->taps != 0) {
		if (tsdrgpu_channel_taps(spec, 1, NULL, NULL) != TSDRGPU_OK)
			return tsdrgpu_fail(p->ctx, TSDRGPU_EINVAL, "invalid channel filter spec (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
		c = *spec;
	}
	return update(p, true, [&](Settings &s) { s.cf_spec = c; });
}
int tsdrgpu_pipeline_set_spectrum(tsdrgpu_pipeline_t *p, const tsdrgpu_welch_t *spec) {
	if (!p) return TSDRGPU_EINVAL;
	tsdrgpu_welch_t w = {0, 0};
	if (spec && spec->n != 0) {
		if (tsdrgpu_spectrum_k(spec, 1) == 0) return tsdrgpu_fail(p->ctx, TSDRGPU_EINVAL, "invalid spectrum spec (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
		w = *spec;
	}
	return update(p, true, [&](Settings &s) { s.sp_spec = w; });
}
int tsdrgpu_pipeline_set_coherence(tsdrgpu_pipeline_t *p, const tsdrgpu_coherence_t *spec) {
	if (!p) return TSDRGPU_EINVAL;
	tsdrgpu_coherence_t c = {0};
	if (spec && spec->rate != 0) {
		if (spec->rate < 1 || spec->rate > TSDRGPU_COHERENCE_MAX_RATE)
			return tsdrgpu_fail(p->ctx, TSDRGPU_EINVAL, "invalid coherence spec (tsdrgpu.h)", cudaSuccess, __FILE__, __LINE__);
		c = *spec;
	}
	return update(p, true, [&](Settings &s) { s.ch_spec = c; });
}
int tsdrgpu_pipeline_set_denoise(tsdrgpu_pipeline_t *p, int mode, int h_milli, int r, int p_radius) {
	return update(p, denoise_ok(mode, h_milli, r, p_radius), [&](Settings &s) {
		if (mode == TSDRGPU_DENOISE_NLM) { s.nl_h = h_milli; s.nl_r = r; s.nl_p = p_radius; }
		s.nl_mode = mode;
	});
}
int tsdrgpu_pipeline_set_stack(tsdrgpu_pipeline_t *p, int mode, int depth, int rx, int ry) {
	return update(p, stack_ok(mode, depth, rx, ry), [&](Settings &s) {
		if (mode != TSDRGPU_STACK_OFF) { s.st_depth = depth; s.st_rx = rx; s.st_ry = ry; }
		s.st_mode = mode;
	});
}
int tsdrgpu_pipeline_set_deblur(tsdrgpu_pipeline_t *p, int mode, int sigma_centi, int iterations) {
	return update(p, deblur_ok(mode, sigma_centi, iterations), [&](Settings &s) {
		if (mode == TSDRGPU_DEBLUR_RL) { s.db_sigma = sigma_centi; s.db_iters = iterations; }
		s.db_mode = mode;
	});
}
int tsdrgpu_pipeline_sync(tsdrgpu_pipeline_t *p, int pixels) { return update(p, true, [&](Settings &s) { s.syncoffset += pixels; s.stack_restart = 1; }); }
int tsdrgpu_pipeline_get_geometry(tsdrgpu_pipeline_t *p, int *width, int *height, double *refreshrate) {
	if (!p) return TSDRGPU_EINVAL;
	const Settings s = settings(p);
	if (width) *width = s.width; if (height) *height = s.height; if (refreshrate) *refreshrate = s.refreshrate;
	return TSDRGPU_OK;
}
int tsdrgpu_pipeline_stats(tsdrgpu_pipeline_t *p, tsdrgpu_pipeline_stats_t *out) {
	if (!p || !out) return TSDRGPU_EINVAL;
	{ std::lock_guard<std::mutex> g(p->mu); *out = p->stats; }
	out->gpu_launches = p->ctx->launches;
	return TSDRGPU_OK;
}

// ---- superbandwidth mode: superb_run (superbandwidth.c:179-254) + superb_ondataready (:121-152) -------------------
// Four hops of 10 frames each are recorded at centre frequencies fc + (hop-2)*fs (0.5 s settling pause after every
// retune), aligned, and stitched into one 4x-rate signal that then flows through the normal decimator / frame stages.
// The reference does the stitch on a helper thread (~3 s of CPU FFTs); here it runs on the GPU inside the call that
// completes the last hop (a few ms), so its output appears one process() call earlier.  Everything else is the same.
// back to the front end's own rate, in the live settings and in the caller's copy s
static void superb_stop(tsdrgpu_pipeline *p, Settings &s) {     // superbandwidth.c:256-264
	if (p->sb.state == SB_STOPPED) return;
	p->sb.state = SB_STOPPED;
	if (s.retune_cb) s.retune_cb(0, p->user);
	update(p, true, [](Settings &live) { live.samplerate = live.samplerate_real; geometry(live); });
	s.samplerate = s.samplerate_real; geometry(s);
}
// make room for `bytes` of raw samples in slot ss (contents are not preserved)
static int raw_reserve(tsdrgpu_pipeline *p, int ss, size_t bytes) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	if (p->d_raw[ss].cap >= bytes) return TSDRGPU_OK;
	CU_TRY(ctx, cudaStreamSynchronize(p->s_ingest)); CU_TRY(ctx, cudaStreamSynchronize(p->s_copy));
	CU_TRY(ctx, p->d_raw[ss].assign(bytes + bytes / 2));
	return TSDRGPU_OK;
}

// H ranks' hop buffers (the borrowing ranks are made here) and, sharded, their group; the hop size is recorded once all of it exists
static int superb_build(tsdrgpu_pipeline *p, const Settings &s, int H, bool sharded) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	const long long in_frame = (long long) (s.samplerate_real / s.refreshrate), pairs = 10 * in_frame;     // SUPER_SAMPLES_TO_RECORD
	CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
	for (int i = 0; i < H; i++) {
		if (!p->sb.rank[i]) p->sb.rank[i].reset(new SbRank{p->ctx->device, p->ctx, p->s_main, p->s_copy, p->sb.ev});
		SbRank &r = *p->sb.rank[i];
		CU_TRY(ctx, cudaSetDevice(r.dev)); CU_TRY(ctx, r.hop.assign(2 * (size_t) pairs));
		if (r.own.c) CU_TRY(ctx, r.hop0.assign(2 * (size_t) pairs));
	}
	if (sharded) {
		for (int i = 0; i < H; i++) { tsdrgpu_superb_mgpu_destroy(p->sb.grp[i]); p->sb.grp[i] = NULL; }
		for (int i = 0; i < H; i++)
			if (const int rc = tsdrgpu_superb_mgpu_create(p->sb.rank[i]->ctx, H, i, 0, (uint32_t) pairs, &p->sb.grp[i])) return rank_error(p, p->sb.rank[i]->ctx, rc);
		if (const int rc = tsdrgpu_superb_mgpu_connect_local(p->sb.grp, H)) return rc;
	}
	CU_TRY(ctx, cudaSetDevice(ctx->device));
	p->sb.rate = s.samplerate_real; p->sb.nhops = H; p->sb.in_frame = in_frame; p->sb.to_gather = pairs;
	p->sb.to_pause = (long long) (0.5 * s.samplerate_real);   // SUPER_SECS_TO_PAUSE
	return TSDRGPU_OK;
}

static int superb_step(tsdrgpu_pipeline *p, const Settings &s, const void *h_iq, int fmt, uint64_t items_count, int64_t dropped) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	int rc;
	const bool sharded = p->sb.ndev > 1;
	if (p->sb.state == SB_STOPPED) p->sb.state = SB_STARTING;
	if (p->sb.state == SB_STARTING) p->sb.spec = s.sbd_spec;                   // a new stitch takes effect at the next round
	const bool coherent = p->sb.spec.mode == TSDRGPU_SUPERBAND_COHERENT;
	const int H = coherent ? p->sb.spec.hops : (sharded ? p->sb.ndev : 4);       // SUPER_HOPS_TO_MAKE
	if (p->sb.state == SB_STARTING) {
		p->sb.buffid = 0; p->sb.gathered = 0;
		if (coherent && sharded) return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "the coherent superbandwidth stitch runs on one GPU", cudaSuccess, __FILE__, __LINE__);
		// the coherent mode also follows the hop size when the refresh rate moves it (the reference mode keeps its first one)
		const bool resize = coherent && (long long) (s.samplerate_real / s.refreshrate) != p->sb.in_frame;
		if ((s.samplerate_real != p->sb.rate || p->sb.nhops != H || resize) && (rc = superb_build(p, s, H, sharded))) { cudaSetDevice(ctx->device); return rc; }
		if (coherent) {
			// every hop, hop 0 included, is recorded after a retune and the pause
			uint32_t n = 0;
			if (tsdrgpu_superband_schedule(&p->sb.spec, p->sb.rate, s.refreshrate, &n, &p->sb.d, p->sb.offsets) != TSDRGPU_OK ||
			    n != tsdrgpu_fft_getrealsize((uint32_t) p->sb.to_gather))
				return tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "no coherent superbandwidth schedule for this sample rate and refresh rate", cudaSuccess, __FILE__, __LINE__);
			if (s.retune_cb) s.retune_cb(p->sb.offsets[0], p->user);
			p->sb.state = SB_PAUSE;
		} else p->sb.state = SB_GATHERING;
	}
	if (p->sb.state == SB_PAUSE) {
		p->sb.gathered += (long long) (items_count / 2);
		if (p->sb.gathered > p->sb.to_pause) { p->sb.gathered = 0; p->sb.state = SB_GATHERING; }
	}
	if (p->sb.state != SB_GATHERING) return TSDRGPU_OK;
	if (dropped) { p->sb.gathered = 0; return TSDRGPU_OK; }
	const long long now = (long long) (items_count / 2);
	const long long take = (p->sb.gathered + now < p->sb.to_gather) ? now : (p->sb.to_gather - p->sb.gathered);
	if (take > 0) {
		SbRank &r = *p->sb.rank[p->sb.buffid];
		float *hop = r.hop.ptr + 2 * p->sb.gathered;
		const size_t bytes = fmt_bytes(fmt) * 2 * (size_t) take;
		// the hop lives on the device that will transform it: the block goes there straight from the host
		CU_TRY(ctx, cudaSetDevice(r.dev));
		cudaError_t e = cudaStreamWaitEvent(r.copy, r.ev, 0);     // the last stitch has finished reading the hop buffer
		if (e == cudaSuccess) {
			if (fmt == TSDRGPU_FMT_FLOAT) e = cudaMemcpyAsync(hop, h_iq, bytes, cudaMemcpyHostToDevice, r.copy);
			else {
				DeviceBuf<unsigned char> &raw = r.own.c ? r.raw : p->d_raw[0];
				if (raw.cap < bytes) { cudaStreamSynchronize(r.copy); e = raw.assign(bytes + bytes / 2); }
				if (e == cudaSuccess) e = cudaMemcpyAsync(raw.ptr, h_iq, bytes, cudaMemcpyHostToDevice, r.copy);
				if (e == cudaSuccess) { pl_convert<<<1024, 256, 0, r.copy>>>(raw.ptr, hop, 2 * (size_t) take, fmt); ctx->launches++; e = cudaGetLastError(); }
			}
		}
		const cudaError_t e2 = cudaStreamSynchronize(r.copy);            // the plugin's buffer has been read, whatever happened
		cudaSetDevice(ctx->device);
		if (e != cudaSuccess || e2 != cudaSuccess) return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "H2D of a superbandwidth hop block", e != cudaSuccess ? e : e2, __FILE__, __LINE__);
		p->stats.h2d_bytes += bytes;
	}
	p->sb.gathered += take;
	if (p->sb.gathered < p->sb.to_gather) return TSDRGPU_OK;
	const long long count_pairs = p->sb.gathered;
	p->sb.buffid++; p->sb.gathered = 0;
	if (sharded && p->sb.buffid == 1) {
		// hop 0 is complete: every other device gets its copy now (NVLink peer copy, seconds before the stitch needs it), so that
		// each rank derives its alignment lag from local data (superb_mgpu.cu phase 2)
		for (int i = 1; i < H; i++) {
			SbRank &r = *p->sb.rank[i], &r0 = *p->sb.rank[0];
			cudaSetDevice(r.dev);
			cudaError_t e = cudaStreamWaitEvent(r.copy, r.ev, 0);
			if (e == cudaSuccess) e = cudaMemcpyPeerAsync(r.hop0.ptr, r.dev, r0.hop.ptr, r0.dev, sizeof(float) * 2 * (size_t) count_pairs, r.copy);
			if (e == cudaSuccess) e = cudaStreamSynchronize(r.copy);
			if (e != cudaSuccess) { cudaSetDevice(ctx->device); return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "peer copy of the alignment reference (hop 0)", e, __FILE__, __LINE__); }
		}
		cudaSetDevice(ctx->device);
	}
	if (p->sb.buffid < H) {
		if (coherent) { if (s.retune_cb) s.retune_cb(p->sb.offsets[p->sb.buffid], p->user); }
		else if (s.retune_cb) s.retune_cb((int32_t) ((p->sb.buffid - H / 2) * (long long) p->sb.rate), p->user);    // shiftfreq, superbandwidth.c:241
		p->sb.state = SB_PAUSE;
		return TSDRGPU_OK;
	}
	// all hops recorded: align + stitch (superb_ondataready) and hand the H-times-rate signal to the decimator
	const unsigned long long N = tsdrgpu_fft_getrealsize((uint32_t) count_pairs);
	size_t total_samples = 0;
	CU_TRY(ctx, cudaStreamSynchronize(p->s_ingest));
	if (coherent) {
		// the coherent stitch: L = H N pairs at H fs, handed to the decimator as the one-GPU reference path hands its output
		const size_t L = (size_t) H * N;
		if (p->sb.d_out.cap < 2 * L || p->sb.d_est.cap < (size_t) H) {
			CU_TRY(ctx, cudaStreamSynchronize(p->s_main));
			CU_TRY(ctx, p->sb.d_out.reserve(p->s_main, 2 * L, 0)); CU_TRY(ctx, p->sb.d_est.reserve(p->s_main, (size_t) H, 0));
		}
		float *hops[TSDRGPU_SUPERBAND_MAX_HOPS];
		for (int i = 0; i < H; i++) hops[i] = p->sb.rank[i]->hop.ptr;
		if ((rc = tsdrgpu_superb_stitch_coherent(ctx, p->s_main, hops, H, (int) count_pairs, (int) p->sb.d, p->sb.d_out.ptr, p->sb.d_est.ptr))) return rc;
		p->sb.est_n = H - 1;
		CU_TRY(ctx, cudaEventRecord(p->sb.ev, p->s_main));
		float *where;
		if ((rc = decim_set_elem(p, 2))) return rc;
		if ((rc = decim_reserve(p, L, &where))) return rc;
		pl_copy_f32<<<2048, 256, 0, p->s_main>>>(p->sb.d_out.ptr, where, 2 * L);
		LAUNCH_CHECK(ctx);
		total_samples = L;
	} else if (!sharded) {
		if (p->sb.d_out.cap < 2 * (size_t) H * N) { CU_TRY(ctx, cudaStreamSynchronize(p->s_main)); CU_TRY(ctx, p->sb.d_out.assign(2 * (size_t) H * N)); }
		int offs[16], total = 0;
		float *hops[16];
		for (int i = 0; i < H; i++) hops[i] = p->sb.rank[i]->hop.ptr;
		if ((rc = tsdrgpu_superb_stitch(ctx, p->s_main, hops, H, (int) count_pairs, (int) p->sb.in_frame, p->sb.d_out.ptr, offs, &total))) return rc;
		CU_TRY(ctx, cudaEventRecord(p->sb.ev, p->s_main));
		float *where;
		if ((rc = decim_set_elem(p, 2))) return rc;
		if ((rc = decim_reserve(p, (size_t) total, &where))) return rc;
		pl_copy_f32<<<2048, 256, 0, p->s_main>>>(p->sb.d_out.ptr, where, 2ull * (size_t) total);
		LAUNCH_CHECK(ctx);
		total_samples = (size_t) total;
	} else {
		// one hop per GPU: every rank runs its share on its own device; rank 0 (this pipeline's device, the main stream) receives
		// the time-contiguous MAGNITUDE stream straight into the decimator input (superb_mgpu.cu)
		float *where;
		if ((rc = decim_set_elem(p, 1))) return rc;
		if ((rc = decim_reserve(p, (size_t) H * N, &where))) return rc;
		for (int i = 0; i < H; i++) {
			SbRank &r = *p->sb.rank[i];
			rc = tsdrgpu_superb_mgpu_stitch(p->sb.grp[i], r.stream, r.hop.ptr, i == 0 ? r.hop.ptr : r.hop0.ptr, (int) count_pairs, (int) p->sb.in_frame, i == 0 ? where : NULL, NULL);
			if (rc) { cudaSetDevice(ctx->device); return rank_error(p, r.ctx, rc); }
			if (i > 0) { cudaSetDevice(r.dev); cudaEventRecord(r.ev, r.stream); }
		}
		CU_TRY(ctx, cudaSetDevice(ctx->device));
		CU_TRY(ctx, cudaEventRecord(p->sb.ev, p->s_main));
		total_samples = (size_t) H * N;
	}
	p->stats.stitches++;
	update(p, true, [&](Settings &live) { live.samplerate = (uint32_t) H * p->sb.rate; geometry(live); });    // set_internal_samplerate(tsdr, buffscount*samplerate)
	p->decim_fill += total_samples;
	p->sb.state = SB_STARTING;
	return drain_blocks(p);
}

// the body of the reference's process() (TSDRLibrary.c:264-298)
int tsdrgpu_convert_samples(tsdrgpu_ctx_t *ctx, void *stream, const void *d_raw, int fmt, uint64_t items_count, float *d_out) {
	BIND(ctx);
	ARG_TRY(ctx, fmt >= TSDRGPU_FMT_FLOAT && fmt <= TSDRGPU_FMT_UINT16);
	if (items_count == 0) return TSDRGPU_OK;
	ARG_TRY(ctx, d_raw != NULL && d_out != NULL);
	if (fmt == TSDRGPU_FMT_FLOAT) { CU_TRY(ctx, cudaMemcpyAsync(d_out, d_raw, sizeof(float) * items_count, cudaMemcpyDeviceToDevice, (cudaStream_t) stream)); return TSDRGPU_OK; }
	const size_t want = (items_count / 4 + 255) / 256;
	KL(ctx, "pl_convert", (cudaStream_t) stream, pl_convert<<<(unsigned) (want < 2048 ? (want ? want : 1) : 2048), 256, 0, (cudaStream_t) stream>>>(d_raw, d_out, items_count, fmt));
	return TSDRGPU_OK;
}

static int process_impl(tsdrgpu_pipeline_t *p, const void *h_iq, int fmt, uint64_t items_count, int64_t samples_dropped, bool wait_for_copy);

// the channel filter over one whole block on the ingest stream, into d_cf_out (one buffer: s_ingest orders all its readers).  The
// history restarts from zero after a drop and after a block with samples that was not filtered.
static int channel_filter(tsdrgpu_pipeline *p, const tsdrgpu_channel_t *spec, uint32_t fs, const float *stage, uint64_t pairs, bool dropped) {
	tsdrgpu_ctx_t *ctx = p->ctx;
	int rc;
	if (!p->cf && (rc = tsdrgpu_chanfilt_create(ctx, &p->cf))) return rc;
	if ((rc = tsdrgpu_chanfilt_set(p->cf, spec, fs))) return rc;          // new taps (spec or samplerate) zero the history
	if ((dropped || p->cf_stale) && (rc = tsdrgpu_chanfilt_reset(p->cf, p->s_ingest))) return rc;
	p->cf_stale = 0;
	if (p->d_cf_out.cap < 2 * pairs) {
		CU_TRY(ctx, cudaStreamSynchronize(p->s_ingest));
		CU_TRY(ctx, p->d_cf_out.reserve(p->s_main, 2 * pairs));
	}
	return tsdrgpu_chanfilt_run(p->cf, p->s_ingest, stage, pairs, p->d_cf_out.ptr);
}

int tsdrgpu_pipeline_process(tsdrgpu_pipeline_t *p, const float *h_iq, uint64_t items_count, int64_t samples_dropped) {
	return process_impl(p, h_iq, TSDRGPU_FMT_FLOAT, items_count, samples_dropped, true);
}
int tsdrgpu_pipeline_process_raw(tsdrgpu_pipeline_t *p, const void *h_iq, int fmt, uint64_t items_count, int64_t samples_dropped) {
	return process_impl(p, h_iq, fmt, items_count, samples_dropped, true);
}
// For a front end that owns a ring of PAGE-LOCKED buffers: the call returns as soon as everything is enqueued, the buffer must
// stay untouched until tsdrgpu_pipeline_sync_input() has returned (or the buffer three calls later has been accepted: there are
// four staging slots).  Copies of consecutive blocks then run back to back on the link instead of waiting for the host's
// enqueue work in between.  Not for pageable memory (a pageable cudaMemcpyAsync is synchronous anyway).
int tsdrgpu_pipeline_process_raw_async(tsdrgpu_pipeline_t *p, const void *h_pinned, int fmt, uint64_t items_count, int64_t samples_dropped) {
	return process_impl(p, h_pinned, fmt, items_count, samples_dropped, false);
}
int tsdrgpu_pipeline_sync_input(tsdrgpu_pipeline_t *p) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, p != NULL);
	BIND(p->ctx);
	CU_TRY(p->ctx, cudaStreamSynchronize(p->s_copy));
	return TSDRGPU_OK;
}

static int process_impl(tsdrgpu_pipeline_t *p, const void *h_iq, int fmt, uint64_t items_count, int64_t samples_dropped, bool wait_for_copy) {
	ARG_TRY((tsdrgpu_ctx_t *) NULL, p != NULL);
	tsdrgpu_ctx_t *ctx = p->ctx;
	BIND(ctx);
	ARG_TRY(ctx, fmt >= TSDRGPU_FMT_FLOAT && fmt <= TSDRGPU_FMT_UINT16);
	ARG_TRY(ctx, (items_count & 1) == 0);                     // assert at TSDRLibrary.c:265
	const uint64_t size2 = items_count >> 1;
	Settings s = settings(p);
	const int w = s.width, h = s.height; const double ptos = s.ptos;     // the geometry at the call's start plans its blocks
	p->stats.samples_in += size2;
	if (samples_dropped > 0) p->stats.samples_dropped_upstream += (uint64_t) samples_dropped;
	const bool sp_on = s.sp_spec.n != 0, ch_on = s.ch_spec.rate != 0, superres = s.params[TSDRGPU_PARAM_AUTOCORR_SUPERRESOLUTION] != 0;
	p->spec.fresh |= superres || !sp_on;                                  // hops at other tunings, or the path is off
	p->coh.fresh |= superres || !ch_on;
	if (superres) {
		if (size2 > 0) p->cf_stale = 1;                        // the hops are recorded unfiltered: the bands refer to one tuning
		return superb_step(p, s, h_iq, fmt, items_count, samples_dropped);
	}
	superb_stop(p, s);
	const bool cf_on = s.cf_spec.taps != 0;
	const int block = (int) round((double) ((w * h) << 1) * ptos);           // TSDRLibrary.c:284
	if (block <= 0) return TSDRGPU_OK;
	p->dev_drop.shift_with((uint32_t) block, samples_dropped);
	const bool drop_all = p->dev_drop.will_drop_all((uint32_t) size2);
	const bool plots_on = !s.params[TSDRGPU_PARAM_AUTOCORR_PLOTS_OFF];
	int rc = TSDRGPU_OK;
	// the block is needed by the decimator or the capture (need_main), or by the spectrum or the coherence alone: they see every
	// pair delivered
	const bool need_main = size2 > 0 && (!drop_all || (plots_on && samples_dropped != 0));
	const bool need_data = need_main || ((sp_on || ch_on) && size2 > 0);
	const int ss = p->stage_slot;
	float *stage = NULL;
	bool copy_issued = false;
	// Every path out of this block -- success or failure -- passes the synchronisation of the copy stream below: the header's
	// contract is that the caller's buffer is read during the call only.
	do {
		if (need_data) {
			if (h_iq == NULL) { rc = tsdrgpu_fail(ctx, TSDRGPU_EINVAL, "invalid argument: h_iq != NULL", cudaSuccess, __FILE__, __LINE__); break; }
			p->stage_slot = (p->stage_slot + 1) & 3;
			if (p->d_stage[ss].cap < items_count) { cudaStreamSynchronize(p->s_ingest); cudaStreamSynchronize(p->s_copy); cudaStreamSynchronize(p->s_spec); }
			cudaError_t e = p->d_stage[ss].reserve(p->s_main, items_count);
			if (e != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "staging buffer", e, __FILE__, __LINE__); break; }
			stage = p->d_stage[ss].ptr;
			// The plugin's buffer is only valid during this call: copy it on the copy stream into one of four staging slots
			// (after the ingest kernels that read the slot four calls ago) and return once the host buffer has been read.
			// The light per-block kernels (capture demod, append to the decimator input) run on their own stream, so the
			// copy of block k+1..k+3 never waits behind the heavy resample / frame / FFT kernels of earlier blocks.
			const size_t bytes = fmt_bytes(fmt) * items_count;
			if (fmt != TSDRGPU_FMT_FLOAT && (rc = raw_reserve(p, ss, bytes))) break;
			const void *src = host_source(p, s.host_register, h_iq, bytes);
			e = cudaStreamWaitEvent(p->s_copy, p->ev_used[ss], 0);
			if (e == cudaSuccess && (p->spec.obj || p->coh.obj)) e = cudaStreamWaitEvent(p->s_copy, p->ev_sp_used[ss], 0);   // and s_spec's reads of it
			if (e == cudaSuccess) { e = cudaMemcpyAsync(fmt == TSDRGPU_FMT_FLOAT ? (void *) stage : p->d_raw[ss].ptr, src, bytes, cudaMemcpyHostToDevice, p->s_copy); copy_issued = true; }
			if (e == cudaSuccess) e = cudaEventRecord(p->ev_h2d[ss], p->s_copy);
			if (e == cudaSuccess) e = cudaStreamWaitEvent(p->s_ingest, p->ev_h2d[ss], 0);
			if (e != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "H2D of the plugin's block", e, __FILE__, __LINE__); break; }
			if (fmt != TSDRGPU_FMT_FLOAT) {                                    // raw samples -> float IQ, on the device
				const size_t want = (items_count / 4 + 255) / 256;
				pl_convert<<<(unsigned) (want < 2048 ? (want ? want : 1) : 2048), 256, 0, p->s_ingest>>>(p->d_raw[ss].ptr, stage, items_count, fmt);
				ctx->launches++;
				if ((e = cudaGetLastError()) != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "kernel launch", e, __FILE__, __LINE__); break; }
			}
			p->stats.h2d_bytes += bytes;
			if (sp_on || ch_on) {                                              // the converted block, before the channel filter
				e = cudaEventRecord(p->ev_conv, fmt == TSDRGPU_FMT_FLOAT ? p->s_copy : p->s_ingest);
				if (e == cudaSuccess) e = cudaStreamWaitEvent(p->s_spec, p->ev_conv, 0);
				if (e != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "stream ordering", e, __FILE__, __LINE__); break; }
				if (sp_on && (rc = report_block(p, p->spec, (size_t) s.sp_spec.n, tsdrgpu_spectrum_create, tsdrgpu_spectrum_reset, tsdrgpu_spectrum_plan,
				                                tsdrgpu_spectrum_run, [&](tsdrgpu_spectrum *o) { return tsdrgpu_spectrum_set(o, &s.sp_spec, s.samplerate); },
				                                s.samplerate, stage, size2, samples_dropped != 0))) break;
				const double alpha = (double) s.height * s.refreshrate;
				if (ch_on && (rc = report_block(p, p->coh, (size_t) tsdrgpu_coherence_n(s.samplerate, alpha), tsdrgpu_coherence_create, tsdrgpu_coherence_reset,
				                                tsdrgpu_coherence_plan, tsdrgpu_coherence_run, [&](tsdrgpu_coherence *o) { return tsdrgpu_coherence_set(o, &s.ch_spec, s.samplerate, alpha); },
				                                s.samplerate, stage, size2, samples_dropped != 0))) break;
				// ev_sp_used[ss] keeps the copy four calls later from overwriting the slot before s_spec has read it
				if ((e = cudaEventRecord(p->ev_sp_used[ss], p->s_spec)) != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "stream ordering", e, __FILE__, __LINE__); break; }
			}
			if (need_main) {
				if (cf_on) {                                                   // the capture and the decimator read the filtered block
					if ((rc = channel_filter(p, &s.cf_spec, s.samplerate, stage, size2, samples_dropped != 0))) break;
					stage = p->d_cf_out.ptr;
				}
				if ((rc = feed_capture(p, s, stage, size2, samples_dropped != 0))) break;
			}
		} else if (plots_on && samples_dropped != 0) p->cap_fill = 0;
		if (size2 > 0 && !(need_main && cf_on)) p->cf_stale = 1;
		uint32_t skip = 0;
		const uint32_t fwd = p->dev_drop.add((uint32_t) size2, (uint32_t) block, true, &skip);
		if (fwd) {
			float *where;
			if ((rc = decim_set_elem(p, 2))) break;
			if (p->d_decim.cap < 2 * (p->decim_read + p->decim_fill + fwd)) cudaStreamSynchronize(p->s_ingest);
			if ((rc = decim_reserve(p, fwd, &where))) break;
			cudaError_t e = cudaStreamWaitEvent(p->s_ingest, p->ev_decim, 0);  // the last compaction of the decimator input is done
			if (e == cudaSuccess) {
				pl_copy_f32<<<(unsigned) ((2ull * fwd + 255) / 256 < 2048 ? (2ull * fwd + 255) / 256 : 2048), 256, 0, p->s_ingest>>>(stage + 2ull * skip, where, 2ull * fwd);
				ctx->launches++;
				e = cudaGetLastError();
			}
			if (e != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "append to the decimator input", e, __FILE__, __LINE__); break; }
			p->decim_fill += fwd;
		}
		{
			cudaError_t e = cudaSuccess;
			if (need_data) e = cudaEventRecord(p->ev_used[ss], p->s_ingest);  // the slot may be overwritten after this point
			if (e == cudaSuccess) e = cudaEventRecord(p->ev_ingest, p->s_ingest);
			if (e == cudaSuccess) e = cudaStreamWaitEvent(p->s_main, p->ev_ingest, 0);      // the resampler may read what was appended
			if (e != cudaSuccess) { rc = tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "stream ordering", e, __FILE__, __LINE__); break; }
		}
		// Everything above and the launches below are only ENQUEUED (ordered on the device by events), so the host's launch
		// work for the heavy kernels runs while this block's H2D copy is still in flight; the copy is waited for last.
		rc = drain_blocks(p);
	} while (0);
	if (copy_issued && (wait_for_copy || rc != TSDRGPU_OK)) {
		const cudaError_t e = cudaStreamSynchronize(p->s_copy);             // the host buffer has been read
		if (e != cudaSuccess && rc == TSDRGPU_OK) return tsdrgpu_fail(ctx, TSDRGPU_ECUDA, "cudaStreamSynchronize(s_copy)", e, __FILE__, __LINE__);
	}
	return rc;
}

}  // extern "C"
