"""GPU: what a context and a pipeline own is theirs alone.  The FFT's twiddle tables belong to the context that built them, so a
new context on the same device, or a second one alive beside it, computes the same bits; the streaming pipeline's superbandwidth
ranks are rebuilt whole every time the mode changes.  Each case runs in a process of its own: the first context of a fresh process
builds every table from nothing."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _in_subprocess(call, env=None, timeout=300):
    r = subprocess.run([sys.executable, "-c", f"from tests.test_resource_owners import *; {call}; print('case ok')"],
                       capture_output=True, text=True, timeout=timeout, cwd=ROOT, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0 and "case ok" in r.stdout, (r.stdout[-1500:], r.stderr[-2500:])


# ------------------------------------------------------------------------------------------------ FFT tables per context
def table_users(ctx):
    """Every kind of twiddle table: transforms of one, two and three passes, the batched half-size autocorrelation at cfg2's
    capture size (odd stride: pair loads) and one Welch report.  Returns the outputs as numpy arrays."""
    from tempestsdr_b200 import _native, api
    rng = np.random.default_rng(7)
    out = []
    for log2n in (10, 21, 24):
        x = torch.from_numpy(rng.standard_normal(2 << log2n).astype(np.float32)).cuda()
        ctx.fft_perform(x, 1 << log2n, False)
        out.append(x.cpu().numpy())
    size, batch = api.FrameRateDetector.capture_size(25_000_000), 2
    stride = size + 1
    caps = torch.from_numpy(np.abs(rng.standard_normal(batch * stride)).astype(np.float32)).cuda()
    ans = torch.empty(2 * size * batch, dtype=torch.float32, device="cuda")
    ctx.chk(_native.lib().tsdrgpu_autocorrelation_batch(ctx._h, ctx.stream, ans.data_ptr(), caps.data_ptr(), size, batch, stride))
    out.append(ans.cpu().numpy())
    spec, fs = "welch:4096:100", 2_000_000
    k = api.Spectrum.segments_per_report(spec, fs)
    sp = ctx.spectrum()
    sp.set(spec, fs)
    iq = torch.from_numpy(rng.standard_normal(2 * (k * 2048 + 2048)).astype(np.float32)).cuda()
    rep = sp.run(iq)
    assert rep.shape == (1, 4096)
    out.append(rep.cpu().numpy())
    del sp
    torch.cuda.synchronize()
    return out


def _same_bits(got, want, what):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(g.view(np.uint8), w.view(np.uint8)), f"{what}: output {i} differs"


def _free_bytes():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def context_lifetime_case():
    from tempestsdr_b200 import _native, api
    first = api.Context(0)
    want = table_users(first)
    first.close()
    again = api.Context(0)
    _same_bits(table_users(again), want, "a new context after the first was destroyed")
    other = api.Context(0)                           # two live contexts on one device, used in turn
    _same_bits(table_users(other), want, "a second live context")
    _same_bits(table_users(again), want, "the first live context after the second")
    other.close(); again.close()
    # close() frees what a context built: an autocorrelation at a size no call above used (cfg5's capture) builds an 8 MiB
    # last-stage table, which a cache that outlived the context would still hold
    free0 = _free_bytes()
    c = api.Context(0)
    size = api.FrameRateDetector.capture_size(50_000_000) & ~1     # the batched API wants an even size
    cap = torch.rand(size, device="cuda")
    ans = torch.empty(2 * size, dtype=torch.float32, device="cuda")
    c.chk(_native.lib().tsdrgpu_autocorrelation_batch(c._h, c.stream, ans.data_ptr(), cap.data_ptr(), size, 1, size))
    del cap, ans
    c.close()
    held = free0 - _free_bytes()
    assert held < 4 << 20, f"{held} bytes of device memory still held after close()"


def test_fft_tables_belong_to_their_context():
    _in_subprocess("context_lifetime_case()")


def welch_report(ctx, n):
    """One Welch report of n points over 25 MS/s of noise plus a tone, in a single run of every segment of the report."""
    from tempestsdr_b200 import api
    spec, fs = f"welch:{n}:10", 25_000_000
    k = api.Spectrum.segments_per_report(spec, fs)
    rng = np.random.default_rng(n)
    t = np.arange(k * n // 2 + n // 2)
    x = (rng.standard_normal(t.size) + 1j * rng.standard_normal(t.size)) * 0.01 + 0.3 * np.exp(2j * np.pi * 0.123 * t)
    sp = ctx.spectrum()
    sp.set(spec, fs)
    rep = sp.run(torch.from_numpy(x.astype(np.complex64).view(np.float32)).cuda())
    assert rep.shape == (1, n)
    out = rep.cpu().numpy()
    del sp
    torch.cuda.synchronize()
    return out


def spectrum_first_case(n):
    """The spectrum's first run sizes its partial-sum rows by the occupancy of the accumulating pass, whose shared memory exceeds
    48 KB from n = 8192 on: the same report whether the spectrum is the first thing a fresh process runs or follows a transform."""
    from tempestsdr_b200 import api
    first = api.Context(0)
    want = welch_report(first, n)
    first.close()
    later = api.Context(0)
    later.fft_perform(torch.zeros(2 * n, dtype=torch.float32, device="cuda"), n, False)
    _same_bits([welch_report(later, n)], [want], f"welch:{n} after a transform")
    later.close()


@pytest.mark.parametrize("n", [8192, 65536])
def test_spectrum_built_before_any_transform(n):
    _in_subprocess(f"spectrum_first_case({n})")


# ------------------------------------------------------------------------------------------------ superbandwidth ranks
def rank_rebuild_case(devs2, devs4):
    """One pipeline through four superbandwidth modes: four hops on one GPU, one hop per device with H = 2, then H = 4, then back
    to the one-GPU mode.  After each switch a stitch completes, the retunes are (k - H/2) fs and the geometry is that of H fs."""
    from oracle import oracle as orc
    from tempestsdr_b200 import pipeline, synth
    O = orc.best()
    fs, h, fv = 400_000, 80, 50.0
    items = 16384
    iq = synth.video_like_iq(200 * items // 2, fs, 200, 80, fv, seed=43, snr_db=25)
    blocks = [iq[k * items:(k + 1) * items].copy() for k in range(200)]
    retunes = []
    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=1, block_when_busy=True,
                          params={"autoshift": 1, "lowpass_before_sync": 1, "autocorr_plots_off": 1},
                          on_retune=lambda off: retunes.append(off))
    for H, devices in ((4, None), (2, devs2), (4, devs4), (4, [0])):
        p.set_param("superresolution", 0)
        p.process(blocks[0], 0)                      # leaves the superbandwidth mode: back to the front end's own rate
        p.flush()
        if devices is not None:
            p.set_superb_devices(devices)
        before, r0 = p.stats().stitches, len(retunes)
        p.set_param("superresolution", 1)
        for b in blocks:
            p.process(b, 0)
            if p.stats().stitches > before:
                break
        p.flush()
        assert p.stats().stitches > before, f"H={H} devices={devices}: no stitch"
        assert retunes[r0:r0 + H - 1] == [(k - H // 2) * fs for k in range(1, H)], (H, devices, retunes[r0:])
        assert p.geometry()[0] == O.geometry(H * fs, h, fv)[0], (H, devices, p.geometry())
    p.close()


def test_superbandwidth_ranks_rebuild_through_modes():
    ngpu = torch.cuda.device_count()
    devs2 = [0, 1] if ngpu >= 2 else [0, 0]
    devs4 = [0, 1, 2, 3] if ngpu >= 4 else [0] * 4
    _in_subprocess(f"rank_rebuild_case({devs2}, {devs4})", env={"CUDA_DEVICE_MAX_CONNECTIONS": "32", "TSDRGPU_SBM_TIMEOUT_MS": "1500"})
