"""GPU parity: the CUDA path (through the C-ABI of include/tsdrgpu.h) against the oracle, on a real H100.

The oracle is the real reference binary (oracle/_ref) when it travelled with the snapshot, else the pinned C
restatement.  Integer/index results and every float produced by the sample->pixel->frame path must be BIT-EXACT;
the FFT family is tolerance-based (float32 Stockham vs the reference's float-storage radix-2): the tolerance is
written next to each check, relative to the peak magnitude of the reference result.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from tempestsdr_b200 import synth
from tests.test_golden import load, superb_hops

pytestmark = pytest.mark.gpu

CFGS = {
    "cfg1": (8_000_000, 525, 60.0),
    "cfg2": (25_000_000, 1125, 60.0),
    "cfg5": (50_000_000, 1125, 60.0),
    "exact2": (1_000_000, 100, 50.0),
    "odd": (2_400_000, 313, 59.94),
}


@pytest.fixture(scope="module")
def gpu():
    from tempestsdr_b200 import api
    return api.Context(0)


@pytest.fixture(scope="module")
def O():
    return orc.best()


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def assert_same_bits(a, b, what=""):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    assert a.shape == b.shape, f"{what}: shape {a.shape} vs {b.shape}"
    bad = np.flatnonzero(bits(a) != bits(b))
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} differ, first at {bad[:5]}: {a[bad[:5]]} vs {b[bad[:5]]}"


# ------------------------------------------------------------------------------------------------ a2
def test_am_demod(gpu, O):
    iq = synth.noise_iq(1_000_003, seed=1)
    iq[:8] = [0, 0, 1e-30, 1e-30, 3e38, 1e38, -0.0, 0.0]
    assert_same_bits(gpu.am_demod(dev(iq)), O.am_demod(iq), "am_demod")
    assert gpu.am_demod(torch.empty(0, device="cuda")).numel() == 0


# ------------------------------------------------------------------------------------------------ a6
def _oracle_stream(O, x, sizes, up, down, nearest, P=None):
    rs = O.resampler()
    out, pos, stale = [], 0, []
    base = 0
    for n in sizes:
        o = rs.run(x[pos:pos + n], up, down, nearest)
        if P is not None and not nearest:   # slots the reference leaves stale (we write 0.0f there)
            pr = P["rs"]
            pr.run(x[pos:pos + n], up, down, nearest)
            for s in range(pr.last_emitted, o.size):
                stale.append(base + s)
        out.append(o); pos += n; base += o.size
    return np.concatenate(out), rs.state, stale


@pytest.mark.parametrize("name", list(CFGS))
@pytest.mark.parametrize("nearest", [False, True])
@pytest.mark.parametrize("fused", [False, True])
def test_resample_stream(gpu, O, name, nearest, fused):
    fs, h, fv = CFGS[name]
    w, _, _ = O.geometry(fs, h, fv)
    up = w * h * fv
    block = int(0.1 * fs / fv)
    sizes = [block] * 7 + [max(3, block // 3), block, 5, block + 17, block]
    rng = np.random.default_rng(7)
    iq = rng.standard_normal(2 * sum(sizes)).astype(np.float32)
    mag = O.am_demod(iq)
    P = {"rs": orc.port().resampler()}
    want, state, stale = _oracle_stream(O, mag, sizes, up, fs, nearest, P)
    r = gpu.resampler()
    x = dev(iq) if fused else dev(mag)
    # two calls: state (contrib on device, offset on host) must carry across calls exactly
    want_mag = fused and not nearest                        # the fused pass can also leave am_demod's output (one demodulation, two consumers)
    mag_a = torch.full((sum(sizes[:5]) + 3,), -1.0, device="cuda") if want_mag else None
    a = r.process(x[: (2 if fused else 1) * sum(sizes[:5])], sizes[:5], up, fs, nearest, in_is_iq=fused, mag_out=mag_a).clone()
    b = r.process(x[(2 if fused else 1) * sum(sizes[:5]):], sizes[5:], up, fs, nearest, in_is_iq=fused)
    got = torch.cat([a, b]).cpu().numpy()
    if want_mag:
        m = mag_a.cpu().numpy()
        assert_same_bits(m[:-3], mag[: sum(sizes[:5])], "magnitudes from the fused pass")
        assert np.all(m[-3:] == -1.0)                      # nothing written past the input
    if stale:
        assert np.all(got[stale] == 0.0)
        want = want.copy(); want[stale] = 0.0
    assert_same_bits(got, want, f"resample {name} nearest={nearest} fused={fused}")
    if not nearest:
        assert r.state == state
    else:
        assert r.state[1] == state[1]


@pytest.mark.parametrize("ratio", [0.37, 0.9999, 1.0, 1.5, 2.0, 3.25, 7.5])
def test_resample_general_ratio(gpu, O, ratio):
    rng = np.random.default_rng(11)
    sizes = [1000 + 37 * k for k in range(9)] + [7, 11, 4100]     # every block must yield >= 1 pixel (the reference asserts)
    x = rng.standard_normal(sum(sizes)).astype(np.float32)
    P = {"rs": orc.port().resampler()}
    want, state, stale = _oracle_stream(O, x, sizes, ratio * 1e6, 1e6, False, P)
    r = gpu.resampler()
    got = r.process(dev(x), sizes, ratio * 1e6, 1e6).cpu().numpy()
    want = want.copy(); want[stale] = 0.0
    assert_same_bits(got, want, f"ratio {ratio}")
    assert r.state == state


def test_resample_state_roundtrip_and_errors(gpu):
    from tempestsdr_b200.api import TsdrGpuError
    r = gpu.resampler()
    r.state = (0.125, -0.25)
    assert r.state == (0.125, -0.25)
    r.reset()
    assert r.state == (0.0, 0.0)
    with pytest.raises(TsdrGpuError):      # a block that yields no pixel: the reference asserts
        r.process(torch.zeros(1, device="cuda"), [1], 0.1, 1.0)
    with pytest.raises(TsdrGpuError):      # output buffer too small
        r.process(torch.zeros(100, device="cuda"), [100], 2.0, 1.0, out=torch.zeros(10, device="cuda"))


# ------------------------------------------------------------------------------------------------ a8-a10, a14
def test_frame_stage_pieces(gpu, O):
    w, h = 507, 525
    f = synth.video_like_frame(w, h, seed=5, shift_x=100, shift_y=40)
    f[1234] = 512.0; f[99] = -300.0
    so = orc.Autogain(0, 0, 1); sg = [0.0, 0.0, 1.0]
    for _ in range(3):
        want = O.autogain(so, f, 0.1)
        got = gpu.dsp_autogain_run(sg, dev(f), 0.1)
        assert_same_bits(got, want, "autogain")
        assert (sg[0], sg[1]) == (so.lastmax, so.lastmin)
        assert abs(sg[2] - so.snr) <= 1e-5 * abs(so.snr)        # tolerance: 1e-5 relative (parallel double sums)
    f2 = f.copy(); f2[0] = 1024.0                                 # a marker in slot 0 seeds min AND max (dsp.c:50)
    so = orc.Autogain(0.3, 0.1, 1); sg = [so.lastmax, so.lastmin, 1.0]
    assert_same_bits(gpu.dsp_autogain_run(sg, dev(f2), 0.1), O.autogain(so, f2, 0.1), "autogain marker at 0")
    s_ref = np.zeros(w * h, np.float32); s_gpu = torch.zeros(w * h, device="cuda")
    for c in (0.0, 0.3, 0.97):
        O.timelowpass(c, f, s_ref); gpu.dsp_timelowpass_run(c, dev(f), s_gpu)
        assert_same_bits(s_gpu, s_ref, f"timelowpass {c}")
    for (ww, hh) in ((507, 525), (740, 1125), (1, 7), (130, 3), (64, 64)):
        g = synth.video_like_frame(ww, hh, seed=ww) if ww > 8 and hh > 8 else np.random.default_rng(1).uniform(0, 1, ww * hh).astype(np.float32)
        wb, hb = gpu.dsp_average_v_h(dev(g), ww, hh)
        wr, hr = O.average_v_h(g, ww, hh)
        assert_same_bits(wb, wr, f"colsum {ww}x{hh}"); assert_same_bits(hb, hr, f"rowsum {ww}x{hh}")
    for n in (1, 2, 3, 4, 5, 6, 17, 507, 4000):
        s = np.random.default_rng(n).uniform(0, 5, n).astype(np.float32)
        assert_same_bits(gpu.gaussianblur(dev(s)), O.gaussianblur(s), f"gauss n={n}")


def _results_tuple(r):
    return (r.x_dx, r.x_vx, r.x_absvx, r.x_stripsize, r.y_dx, r.y_vx, r.y_absvx, r.y_stripsize)


@pytest.mark.parametrize("lpbs,aap,autoshift,mb", [
    (1, 0, 1, 0.0), (1, 1, 1, 0.4), (0, 0, 1, 0.3), (0, 1, 0, 0.0), (0, 0, 0, 0.5), (1, 0, 0, 0.0), (0, 1, 1, 0.2), (1, 1, 0, 0.0),
])
@pytest.mark.parametrize("batches", [(9,), (1, 3, 5), (4, 5)])
def test_post_process_sequence(gpu, O, lpbs, aap, autoshift, mb, batches):
    from tempestsdr_b200.api import PostProcessFlags
    fs, hgt, fv = CFGS["cfg1"]
    w, _, _ = O.geometry(fs, hgt, fv)
    po = O.postprocessor(fs, hgt, fv, autoshift, 0)
    frames = [synth.video_like_frame(w, hgt, seed=k, shift_x=60 + 9 * k, shift_y=20 + 3 * k) for k in range(9)]
    want = [po.run(f, w, hgt, mb, 0.1, lpbs, aap) for f in frames]
    pg = gpu.post_processor()
    flags = PostProcessFlags(autoshift=bool(autoshift), lowpass_before_sync=bool(lpbs), autogain_after_proc=bool(aap), compute_snr=True)
    k = 0
    for nb in batches:
        x = dev(np.concatenate(frames[k:k + nb]))
        out, res = pg.process(x, w, hgt, mb, 0.1, flags)
        out = out.cpu().numpy().reshape(nb, -1)
        for i in range(nb):
            wf, wr = want[k + i]
            assert_same_bits(out[i], wf, f"frame {k + i}")
            assert _results_tuple(res[i]) == wr.x.astuple() + wr.y.astuple(), f"sync state frame {k + i}"
            assert res[i].avg_speed == wr.avg_speed and res[i].pll_state == wr.pll_state
            assert (res[i].lastmax, res[i].lastmin) == (wr.lastmax, wr.lastmin)
            assert res[i].autogain_report == wr.autogain_callback_fired
            if np.isfinite(wr.snr):
                assert abs(res[i].snr - wr.snr) <= 1e-5 * abs(wr.snr)     # tolerance 1e-5 relative
        k += nb


@pytest.mark.parametrize("batches", [(12,), (1, 4, 7)])
def test_post_process_pll_writeback_arithmetic(gpu, O, batches):
    """PLL on (syncdetector.c:133-153): the frame stage leaves vx / avg_speed / pll_state per frame, tsdrgpu_pll_step applies
    the reference's write-back to the refresh rate.  Against the oracle built with PLL = 1: same frames, same sync state, and
    the refresh rate after every frame EXACTLY equal (drifting frames, so the rate moves on most of them and the lock toggles)."""
    import ctypes as C
    from tempestsdr_b200 import _native
    from tempestsdr_b200.api import PostProcessFlags
    fs, hgt, fv = CFGS["cfg1"]
    w, _, _ = O.geometry(fs, hgt, fv)
    po = O.postprocessor(fs, hgt, fv, 1, 1)
    shifts = [60, 63, 66, 69, 72, 72, 72, 73, 73, 74, 90, 110]
    frames = [synth.video_like_frame(w, hgt, seed=k, shift_x=sx, shift_y=20) for k, sx in enumerate(shifts)]
    want = [po.run(f, w, hgt, 0.0, 0.1, 1, 0) for f in frames]
    assert sum(r.pll_callback_fired for _, r in want) >= 4
    pg = gpu.post_processor()
    rr = C.c_double(fv)
    k = 0
    for nb in batches:
        out, res = pg.process(dev(np.concatenate(frames[k:k + nb])), w, hgt, 0.0, 0.1, PostProcessFlags())
        out = out.cpu().numpy().reshape(nb, -1)
        for i in range(nb):
            wf, wr = want[k + i]
            assert_same_bits(out[i], wf, f"frame {k + i}")
            assert _results_tuple(res[i]) == wr.x.astuple() + wr.y.astuple()
            assert res[i].avg_speed == wr.avg_speed and res[i].pll_state == wr.pll_state
            moved = _native.lib().tsdrgpu_pll_step(C.byref(rr), res[i].x_vx, res[i].pll_state, res[i].avg_speed)
            assert moved == wr.pll_callback_fired and rr.value == wr.refreshrate_after, f"refresh rate after frame {k + i}"
        k += nb


@pytest.mark.parametrize("name", ["cfg2", "cfg5", "odd"])
@pytest.mark.parametrize("overlap", [False, True, "tma"])
def test_post_process_full_size_frames(gpu, O, name, overlap, monkeypatch):
    """The frame stage at BASELINE's real frame sizes (740x1125, 1481x1125) and at an odd width (no 16-byte rows: the
    scalar collapse path), default GUI stage order, two batches, with and without the side-stream overlap."""
    from tempestsdr_b200.api import PostProcessFlags
    fs, hgt, fv = CFGS[name]
    w, _, _ = O.geometry(fs, hgt, fv)
    po = O.postprocessor(fs, hgt, fv, 1, 0)
    frames = [synth.video_like_frame(w, hgt, seed=40 + k, shift_x=(70 + 31 * k) % w, shift_y=(25 + 11 * k) % hgt) for k in range(5)]
    want = [po.run(f, w, hgt, 0.0, 0.1, 1, 0) for f in frames]
    if overlap == "tma":                                   # the opt-in TMA (cp.async.bulk + mbarrier) variant of the collapse kernel
        monkeypatch.setenv("TSDRGPU_COLLAPSE_TMA", "1")
    pg = gpu.post_processor()
    pg.set_overlap(bool(overlap))
    flags = PostProcessFlags(autoshift=True, lowpass_before_sync=True)
    k = 0
    outs = []
    for nb in (2, 3):
        x = dev(np.concatenate(frames[k:k + nb]))
        out = torch.empty(nb * w * hgt, dtype=torch.float32, device="cuda")
        pg.process(x, w, hgt, 0.0, 0.1, flags, out=out, want_results=False)
        outs.append(out); k += nb
    pg.join(); torch.cuda.synchronize()
    got = torch.cat(outs).cpu().numpy().reshape(5, -1)
    for i in range(5):
        assert_same_bits(got[i], want[i][0], f"{name} frame {i}")


@pytest.mark.parametrize("mode", ["forced_serial", "wide_dynamic_range", "denormals"])
def test_sync_search_serial_fallback(gpu, O, mode, monkeypatch):
    """The sync search replaces the reference's serial sliding sums by exact prefix sums when a per-strip exactness
    certificate holds; these inputs make it fail (or force the serial chains) -- results must still be bit-identical."""
    from tempestsdr_b200.api import PostProcessFlags
    w, h = 253, 105
    po = O.postprocessor(800_000, h, 60.0, 1, 0)
    pg = gpu.post_processor()
    if mode == "forced_serial":
        monkeypatch.setenv("TSDRGPU_SYNC_SERIAL", "1")
    frames = []
    for k in range(5):
        f = synth.video_like_frame(w, h, seed=70 + k, shift_x=20 + 7 * k, shift_y=5 + k).reshape(h, w)
        if mode == "wide_dynamic_range":
            f[:, ::7] *= 1e-9; f[::5, :] *= 3e4                # column/row sums now span > 2^17
        if mode == "denormals":
            f[:, 3] = 0.0; f[0, 3] = 1e-44                      # a denormal column sum
        frames.append(np.ascontiguousarray(f.reshape(-1)))
    # auto-gain after processing so the (extreme) raw values reach the collapse unchanged
    fl = PostProcessFlags(lowpass_before_sync=True, autogain_after_proc=True)
    out, res = pg.process(dev(np.concatenate(frames)), w, h, 0.0, 0.1, fl)
    out = out.cpu().numpy().reshape(5, -1)
    for k in range(5):
        wf, wr = po.run(frames[k], w, h, 0.0, 0.1, 1, 1)
        assert _results_tuple(res[k]) == wr.x.astuple() + wr.y.astuple(), f"{mode} frame {k}"
        assert_same_bits(out[k], wf, f"{mode} frame {k}")


def test_post_process_resize_and_flag_flip(gpu, O):
    from tempestsdr_b200.api import PostProcessFlags
    po = O.postprocessor(8_000_000, 525, 60.0)
    pg = gpu.post_processor()
    shapes = [(200, 100, 1), (200, 100, 1), (150, 120, 1), (150, 120, 0), (300, 200, 0), (200, 100, 1)]
    for k, (w, h, lpbs) in enumerate(shapes):
        f = synth.video_like_frame(w, h, seed=40 + k, shift_x=11, shift_y=7)
        want, _ = po.run(f, w, h, 0.25, 0.1, lpbs, 0)
        got, _ = pg.process(dev(f), w, h, 0.25, 0.1, PostProcessFlags(lowpass_before_sync=bool(lpbs)))
        assert_same_bits(got, want, f"resize step {k}")


def test_pixels_argb(gpu):
    P = orc.port()
    f = np.array([-1, 0, 1e-9, 0.5, 1.0, 1.0001, 256, 512, 1024, 2048, 7], dtype=np.float32)
    f = np.concatenate([f, np.random.default_rng(0).uniform(-0.1, 1.1, 5000).astype(np.float32)])
    for inv in (False, True):
        assert np.array_equal(gpu.pixels_argb(dev(f), inv).cpu().numpy(), P.pixels_argb(f, inv))


# ------------------------------------------------------------------------------------------------ a19, a20
def _close(got, want, tol, what):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    peak = float(np.max(np.abs(want))) or 1.0
    err = float(np.max(np.abs(got - want))) / peak
    rel_l2 = float(np.linalg.norm(got - want) / (np.linalg.norm(want) or 1.0))
    assert err <= tol, f"{what}: max|err|/peak = {err:.3g} > {tol} (rel L2 {rel_l2:.3g})"
    return err, rel_l2


@pytest.mark.parametrize("logn", range(25))        # every size: one-pass 2^0..2^13, two passes 2^14..2^21, three above
def test_fft(gpu, O, logn):
    n = 1 << logn
    x = synth.noise_iq(n, seed=logn)
    for inv in (False, True):
        want = O.fft(x, inv)
        d = dev(x)
        gpu.fft_perform(d, n, inv)
        # tolerance: 1e-6 of the peak bin up to 2^22, 2e-6 at 2^23 (the worst of 16.7 M outputs after 23 float32 stages
        # lands at 1.0e-6); the project bound for float intermediates is 1e-5 (BASELINE.json north_star).  Both sides keep
        # float32 between stages (~1e-7*sqrt(log2 N) noise each).  Above 2^19 the reference itself drifts from the true DFT by up to 5e-5 (its stage twiddles come
        # from the half-angle recurrence c2 = sqrt((1-c1)/2), fft.c:161, which cancels for small angles); the CUDA FFT
        # uses the same perturbed stage angles (tsdrgpu_fft_reference_eps), so it tracks the reference, not the true DFT.
        # 2^24 (the top of BASELINE configs[2]'s sweep): the last stage's angle error is 1e-4 relative there and the float32
        # rounding of 24 stages adds up; measured 2.1e-6 worst case, bound 4e-6
        err, _ = _close(d, want, 1e-6 if logn <= 22 else (2e-6 if logn == 23 else 4e-6), f"fft 2^{logn} inv={inv}")
        print(f"fft 2^{logn} inv={inv}: max|err|/peak = {err:.3g}")


def test_reference_stage_angle_model():
    """The perturbed-angle model behind the large-N parity: eps from the host replay of the recurrence explains the
    reference's deviation from the true DFT (CPU-side check of the model, on the GPU box for its float64 FFT speed)."""
    import ctypes as C
    from tempestsdr_b200 import _native
    eps = (C.c_double * 24)()
    _native.lib().tsdrgpu_fft_reference_eps(24, 0, eps)
    assert eps[0] == 0.0 and abs(eps[1]) < 1e-15 and abs(eps[10]) < 1e-9
    assert 1e-7 < abs(eps[20]) < 1e-5 and abs(eps[23]) > abs(eps[18])


@pytest.mark.parametrize("size", [1, 5, 1000, 4096, 70_001, 450_909, 450_910, 1_409_090, 2_818_181])
def test_autocorrelation_and_xcorr(gpu, O, size):
    """The default path: even sizes take the half-size transforms, odd sizes the N-point ones (cfg1 / cfg2 / cfg5 capture sizes
    450 909, 1 409 090 and 2 818 181 included)."""
    x = np.abs(synth.noise_iq(size, seed=size)[:size]).astype(np.float32)
    want = O.autocorrelation(x)
    got = gpu.fft_autocorrelation(dev(x))
    _close(got, want, 2e-6, f"autocorrelation {size}")        # tolerance 2e-6 of the zero-lag peak
    n = gpu.fft_getrealsize(size)
    assert n == O.fft_getrealsize(size)
    if size > n:                                              # the untransformed tail is exact: (|x|, 0)
        assert_same_bits(got[2 * n:], want[2 * n:], "autocorr tail")
    if size >= 4:
        a = synth.noise_iq(size, seed=1); b = synth.noise_iq(size, seed=2)
        da, db = dev(a), dev(b)
        gpu.fft_crosscorrelation(da, db, size)
        _close(da[: 2 * n], O.crosscorrelation(a, b)[: 2 * n], 4e-6, f"xcorr {size}")


@pytest.mark.parametrize("size", [4096, 70_001 + 1, 450_910, 1_409_090])
def test_autocorrelation_full_size_path(gpu, O, size, monkeypatch):
    """TSDRGPU_AUTOCORR_FULL=1: the N-point transforms (fft.c:49-64 literally) instead of the default half-size ones (real input
    packed as complex pairs + the reference's last radix-2 stage; profiles/studies/real_input_autocorr_study.py bounds that
    approximation).  Same tolerance either way, and the two paths agree with each other far inside it."""
    x = np.abs(synth.noise_iq(size, seed=size)[:size]).astype(np.float32)
    want = O.autocorrelation(x)
    half = gpu.fft_autocorrelation(dev(x)).cpu().numpy()
    monkeypatch.setenv("TSDRGPU_AUTOCORR_FULL", "1")
    got = gpu.fft_autocorrelation(dev(x))
    _close(got, want, 2e-6, f"full-size autocorrelation {size}")
    n = gpu.fft_getrealsize(size)
    _close(half[: 2 * n], got.cpu().numpy()[: 2 * n], 1e-6, f"half-size vs full-size path {size}")


def test_accumulate_exact_and_framerate_plots(gpu, O):
    fs = 2_000_000
    size = O.framerate_capture_size(fs) if O.kind == "port" else orc.port().framerate_capture_size(fs)
    from tempestsdr_b200.api import FrameRateDetector
    assert FrameRateDetector.capture_size(fs) == size
    assert FrameRateDetector.windows(fs) == orc.port().framerate_windows(fs)
    # accumulate alone is exact when fed the same autocorrelation
    ac = O.autocorrelation(np.abs(synth.noise_iq(30_000, seed=4)[:30_000]).astype(np.float32))
    want = np.zeros(5000); got = torch.zeros(5000, dtype=torch.float64, device="cuda")
    for calls in (1, 2, 3):
        O.accumulate(want, calls, ac, 1000, 5000); gpu.accummulate(got, calls, dev(ac), 1000, 5000)
        assert_same_bits(got, want, f"accumulate calls={calls}")
    do, dg = O.framerate_detector(), gpu.framerate_detector()
    for k in range(3):
        x = O.am_demod(synth.video_like_iq(size, fs, 400, 200, 50.0, seed=k))
        (fo, fp), (lo, lp), c = do.run(fs, x)
        (go, gp), (glo, glp), gc = dg.run(fs, dev(x))
        assert (fo, lo, c) == (go, glo, gc)
        _close(gp, fp, 1e-5, "frame plot"); _close(glp, lp, 1e-5, "line plot")   # tolerance 1e-5 of the plot's peak
        assert int(np.argmax(gp)) == int(np.argmax(fp))       # the lag the GUI would pick is the same


def test_autocorrelation_dump_csv(gpu, O, tmp_path):
    """PARAM_AUTOCORR_DUMP (frameratedetector.c:64-85, 110-116): the CSV of one capture's autocorrelation -- same header, same
    lags (the first fft_getrealsize(2 size) / 4 of them), same time column; the dB column against the reference's autocorrelation
    within the FFT tolerance (2e-6 of the peak on |r|) plus the six printed decimals."""
    fs, size = 2_000_000, 112_727                          # the detector's own (odd) capture size at 2 MS/s
    x = np.abs(synth.video_like_iq(size, fs, 400, 200, 50.0, seed=77).view(np.complex64)).astype(np.float32)
    path = str(tmp_path / "autocorr.csv")
    gpu.framerate_detector().dump_csv(fs, dev(x), path)
    lines = open(path).read().splitlines()
    assert lines[0] == "ms, dB"
    rows = np.array([[float(v) for v in ln.split(",")] for ln in lines[1:]])
    want = O.autocorrelation(x).astype(np.float64)
    nreal = 1 << (int(2 * size).bit_length() - 1)
    maxels = nreal // 2
    assert rows.shape == (maxels // 2, 2)
    k = np.arange(maxels // 2)
    assert np.allclose(rows[:, 0], np.round(1000.0 * k / fs, 6), atol=1e-6)
    mag = np.sqrt(want[0:maxels:2] ** 2 + want[1:maxels:2] ** 2)
    got = 10.0 ** (rows[:, 1] / 10.0)
    assert np.max(np.abs(got - mag)) <= 2e-6 * mag.max() + 3e-7 * mag.max()


def test_framerate_detector_overlapped_mode_gives_the_same_plots(gpu):
    """tsdrgpu_frd_set_overlap: the same kernels on the detector's own stream with its own work buffers -- plots, peaks and call
    counts must be bit-identical to the in-stream mode, also when the caller keeps its stream busy and reuses the capture
    memory right after tsdrgpu_frd_join."""
    fs = 2_000_000
    from tempestsdr_b200.api import FrameRateDetector
    size = FrameRateDetector.capture_size(fs)
    caps = [torch.from_numpy(np.abs(synth.video_like_iq(3 * size, fs, 400, 200, 50.0, seed=40 + k).view(np.complex64)).astype(np.float32)).cuda() for k in range(3)]
    plain, over = gpu.framerate_detector(), gpu.framerate_detector()
    over.set_overlap(True)
    busy = torch.empty(8 << 20, device="cuda")
    for k, c in enumerate(caps):
        work = c.clone()
        plain.run_batch(fs, c, size, 3, size)
        over.run_batch(fs, work, size, 3, size)
        busy.normal_()                                     # the caller's stream has other things to do meanwhile
        over.join()
        work.zero_()                                       # after the join the capture memory may be reused
        (fo, fp), (lo, lp) = plain.plots(fs)
        (go, gp), (glo, glp) = over.plots(fs)
        assert (fo, lo) == (go, glo)
        assert np.array_equal(fp.view(np.uint64), gp.view(np.uint64)) and np.array_equal(lp.view(np.uint64), glp.view(np.uint64)), f"plots after batch {k}"
    over.set_overlap(False)
    plain.run_batch(fs, caps[0], size, 2, size); over.run_batch(fs, caps[0], size, 2, size)
    assert np.array_equal(plain.plots(fs)[0][1].view(np.uint64), over.plots(fs)[0][1].view(np.uint64))


def test_plot_peaks_on_the_device_match_the_gui_pick(gpu):
    """SURVEY 8f-3: the first strict maximum of the two autocorrelation plots, reduced on the GPU (k_plot_peaks), against the
    GUI's pick restated on the host (tsdrgpu_detect_videomode <- PlotVisualizer.java:203-236): 120 seeded plots with ties,
    plateaus, infinities, NaNs (in element 0 and elsewhere) and degenerate lengths; and the detector's own plots after a run."""
    import ctypes as C
    from tempestsdr_b200 import _native
    lib = _native.lib()
    rng = np.random.default_rng(2024)

    def host_pick(fp, lp):
        fi, li = C.c_int(-1), C.c_int(-1)
        rc = lib.tsdrgpu_detect_videomode(fp.ctypes.data_as(C.POINTER(C.c_double)), 1, fp.size, lp.ctypes.data_as(C.POINTER(C.c_double)), 1, lp.size,
                                          1000, None, None, C.byref(fi), C.byref(li))
        assert rc == 0
        return fi.value, li.value
    for case in range(120):
        n0 = int(rng.integers(1, 200_000)) if case % 5 else int(rng.integers(1, 40))
        n1 = int(rng.integers(1, 900))
        fp, lp = rng.standard_normal(n0), rng.uniform(0, 1, n1)
        if case % 4 == 1:                                  # plateaus and exact ties: the first one must win
            fp = np.round(fp * 3) / 3; lp = np.round(lp * 5) / 5
        if case % 7 == 2:
            fp[rng.integers(0, n0)] = np.inf; lp[rng.integers(0, n1)] = -np.inf
        if case % 9 == 3:
            fp[rng.integers(0, n0)] = np.nan                # a NaN elsewhere never wins
        if case % 11 == 4:
            lp[0] = np.nan                                  # a NaN in element 0 is never beaten
        if case % 13 == 5:
            fp[:] = fp[0]
        got = (C.c_int32 * 2)()
        d_fp, d_lp = dev(fp), dev(lp)                        # kept alive across the call (a temporary's memory would be reused)
        gpu.chk(lib.tsdrgpu_plot_peaks(gpu._h, gpu.stream, d_fp.data_ptr(), n0, d_lp.data_ptr(), n1, got))
        assert (got[0], got[1]) == host_pick(fp, lp), f"case {case}"
    det = gpu.framerate_detector()
    fs = 2_000_000
    size = det.capture_size(fs)
    x = orc.port().am_demod(synth.video_like_iq(size, fs, 400, 200, 50.0, seed=8))
    (fo, fp), (lo, lp), _ = det.run(fs, dev(x))
    got = (C.c_int32 * 2)()
    gpu.chk(lib.tsdrgpu_frd_peaks(det._h, gpu.stream, got))
    assert (got[0], got[1]) == host_pick(fp, lp)


# ------------------------------------------------------------------------------------------------ a22
def test_superbandwidth(gpu, O):
    fs, fv = 400_000, 50.0
    sif = int(fs / fv)
    pairs = 10 * sif
    base = synth.video_like_iq(pairs + 5000, fs, 200, 160, fv, seed=9, snr_db=25)
    hops = [base[2 * l: 2 * (l + pairs)].copy() + synth.noise_iq(pairs, seed=100 + i, scale=0.01)
            for i, l in enumerate((0, 1234, 77, 3999))]
    d = hops[1][:4096].copy()
    dd = dev(d); gpu.complex_to_abs_diff(dd)
    assert_same_bits(dd, O.complex_to_abs_diff(d), "abs diff")
    want, offs = O.superb_ondataready(hops, sif)
    got, goffs = gpu.superb_stitch([dev(h) for h in hops], sif)
    assert list(goffs) == list(offs)                          # integer alignment lags: exact
    _close(got, want, 4e-6, "stitched")
    # the one-exchange dataflow (raw spectra + difference spectra gathered once, lags applied as phase ramps)
    from tempestsdr_b200 import superband
    sim, sim_offs = superband.stitch_simulated(gpu, [dev(h) for h in hops], sif)
    assert list(sim_offs) == list(offs)
    _close(sim, want, 8e-6, "one-exchange stitch")


# The sharded path (csrc/superb_mgpu.cu) with all ranks on this GPU, and configs[3]'s 4 x 2^21, are in tests/test_superb_sweep.py.


# ------------------------------------------------------------------------------------------------ golden vectors
def test_golden_vectors_gpu(gpu):
    from tempestsdr_b200.api import PostProcessFlags
    g = load("demod_resample.npz")
    fs, h, fv, w, block = int(g["fs"]), int(g["h"]), float(g["fv"]), int(g["w"]), int(g["block"])
    iq = synth.video_like_iq(6 * block, fs, 2 * w // 2, h, fv, seed=int(g["seed"]))
    assert_same_bits(gpu.am_demod(dev(iq)), g["mag"], "golden demod")
    r = gpu.resampler()
    assert_same_bits(r.process(dev(iq), (block, 6), w * h * fv, fs, in_is_iq=True), g["pixels"], "golden pixels")
    assert r.state == tuple(g["states"][-1])
    assert_same_bits(gpu.resampler().process(dev(iq), (block, 6), w * h * fv, fs, True, in_is_iq=True), g["pixels_nn"], "golden nn")
    for name, mb, lpbs, aap, sx, sy in (("frame_stage_default.npz", 0.0, 1, 0, (31, 5), (11, 1)),
                                        ("frame_stage_blur.npz", 0.35, 0, 1, (40, 0), (9, 0))):
        g = load(name)
        w, h = int(g["w"]), int(g["h"])
        fr = np.concatenate([synth.video_like_frame(w, h, seed=int(s), shift_x=sx[0] + sx[1] * k, shift_y=sy[0] + sy[1] * k)
                             for k, s in enumerate(g["seeds"])])
        out, res = gpu.post_processor().process(dev(fr), w, h, mb, 0.1, PostProcessFlags(lowpass_before_sync=bool(lpbs), autogain_after_proc=bool(aap)))
        assert_same_bits(out.reshape(len(g["seeds"]), -1), g["out"], name)
        got_meta = [[r_.x_dx, r_.x_vx, r_.x_stripsize, r_.y_dx, r_.y_vx, r_.y_stripsize] for r_ in res]
        assert got_meta == g["meta"].tolist()
    g = load("fft_4096.npz")
    d = dev(g["x"]); gpu.fft_perform(d, 4096, False); _close(d, g["fwd"], 2e-6, "golden fft fwd")
    d = dev(g["x"]); gpu.fft_perform(d, 4096, True); _close(d, g["inv"], 2e-6, "golden fft inv")
    g = load("autocorr_20000.npz")
    _close(gpu.fft_autocorrelation(dev(g["x"])), g["ac"], 2e-6, "golden autocorr")
    g = load("superb_4x16384.npz")
    hops, sif = superb_hops(g)
    got, offs = gpu.superb_stitch([dev(h) for h in hops], sif)
    assert list(offs) == list(g["offsets"])
    _close(got, g["out"], 4e-6, "golden superb")


# ------------------------------------------------------------------------------------------------ full-size properties
def test_full_size_properties(gpu):
    """BASELINE cfg2 at full size (64 frames of 25 MS/s, 1125 lines): properties that need no CPU oracle."""
    from tempestsdr_b200.api import PostProcessFlags
    fs, h, fv = CFGS["cfg2"]
    O = orc.port()
    w, _, _ = O.geometry(fs, h, fv)
    nframes, block = 16, int(0.1 * fs / fv)
    nblocks = nframes * 10 + 2
    torch.manual_seed(0)
    iq = torch.randn(2 * block * nblocks, device="cuda")
    r1, r2 = gpu.resampler(), gpu.resampler()
    one = r1.process(iq, (block, nblocks), w * h * fv, fs, in_is_iq=True)
    # (1) chunk invariance: the same stream cut into different call boundaries gives identical pixels and state
    cut = 2 * block * 37
    two = torch.cat([r2.process(iq[:cut], (block, 37), w * h * fv, fs, in_is_iq=True).clone(),
                     r2.process(iq[cut:], (block, nblocks - 37), w * h * fv, fs, in_is_iq=True)])
    assert torch.equal(one, two) and r1.state == r2.state
    # (2) area preservation: sum(pixels) ~= r * sum(|x|) (the box resampler conserves area up to the open pixel)
    mag = gpu.am_demod(iq)
    ratio = w * h * fv / fs
    assert abs(one.double().sum().item() / (ratio * mag.double().sum().item()) - 1.0) < 1e-6
    # (3) a batch of frames equals the same frames fed one by one (bit-exact), and the re-centring is a permutation
    n = w * h
    frames = one[: nframes * n].contiguous()
    pa, pb = gpu.post_processor(), gpu.post_processor()
    fl = PostProcessFlags()
    A, ra = pa.process(frames, w, h, 0.0, 0.1, fl)
    B = torch.cat([pb.process(frames[k * n:(k + 1) * n], w, h, 0.0, 0.1, fl)[0] for k in range(nframes)])
    assert torch.equal(A, B)
    # AUTOSHIFT on: frame f of the output is the temporally filtered frame circularly shifted by (x_dx, y_dx) -- with motionblur 0
    # the filtered frame is the auto-gained input, so the output is a PERMUTATION of it: same multiset of values
    lo, hi = ra[0].lastmin, ra[0].lastmax
    span = np.float32(hi) - np.float32(lo) if hi != lo else np.float32(1.0)
    # tensor / tensor: a true IEEE division per element (a Python scalar divisor would be turned into a multiplication by 1/span)
    norm = torch.div(frames[:n] - float(np.float32(lo)), torch.full((n,), float(span), device="cuda"))
    assert torch.equal(torch.sort(A[:n])[0], torch.sort(norm)[0])
    # (4) FFT round trip and Parseval at 2^22
    x = torch.randn(2 << 22, device="cuda")
    y = x.clone()
    gpu.fft_perform(y, 1 << 22, False)
    e_time = (x.double() ** 2).sum().item() / (1 << 22)
    e_freq = (y.double() ** 2).sum().item()
    assert abs(e_freq / e_time - 1.0) < 1e-5
    gpu.fft_perform(y, 1 << 22, True)
    # the default FFT reproduces the reference's perturbed stage angles (fft.c:161): like the reference's own, its
    # inverse is not the exact inverse of its forward at 2^22 (reference round trip: ~3e-5); 1e-4 is the bound here
    assert (y - x).abs().max().item() < 1e-4
