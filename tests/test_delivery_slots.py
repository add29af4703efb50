"""The streaming pipeline's delivery slots while the host holds its delivery thread.

Every kind of output (frame batches, autocorrelation plots, spectrum reports, coherence reports) goes out through a pool of
page-locked slots of its own.  A plot callback that blocks holds the delivery thread, so no slot comes back: each pool then hands
out exactly its own slots, frame batches are dropped whole and the reports beyond the slots are skipped and counted, path by path.
"""
import threading

import numpy as np
import pytest

from tempestsdr_b200 import _native as N
from tests import test_coherence as tc
from tests import test_spectrum as ts

SPEC, COH = "welch:1024:100", "line:100"      # at SMALL: a spectrum report every 19968 pairs, a coherence report every 16384
BATCH, SLOTS, PLOT_SLOTS = 2, 4, 2
HOLD_S = 30.0                                 # the longest a callback holds the thread: a mistake fails instead of hanging


def _held_run(spectrum, coherence, warm, phase):
    """Warm up with the callbacks free until every pool has its final size, then hold the delivery thread at the first plot
    callback while the phase's blocks go in, release it and flush.  Returns the reports, the stats after the warm-up and at the
    end, and whether the hold ended by timeout."""
    from tempestsdr_b200 import pipeline
    fs, h, fv = ts.SMALL
    spectra, cohs = [], []
    armed, release, timed_out = threading.Event(), threading.Event(), []

    def on_plot(pid, off, v, sr):
        if armed.is_set() and not release.is_set():
            if not release.wait(HOLD_S):
                timed_out.append(pid)
                release.set()
        if pid == N.PLOT_ID_SPECTRUM:
            spectra.append((pid, off, v.copy(), sr))
        elif pid == N.PLOT_ID_COHERENCE:
            cohs.append((pid, off, v.copy(), sr))

    p = pipeline.Pipeline(samplerate=fs, height=h, refreshrate=fv, batch_frames=BATCH, batch_blocks=10 * BATCH,
                          block_when_busy=False, spectrum=spectrum, coherence=coherence, on_plot=on_plot)
    try:
        for b in warm:
            p.process(b)
        p.flush()
        st0 = p.stats()
        armed.set()
        for b in phase:
            p.process(b)
        release.set()
        p.flush()
        st1 = p.stats()
    finally:
        release.set()
        p.close()
    return spectra, cohs, st0, st1, timed_out


def _phase_reports(model_reports, warm, phase):
    """The model's reports of the warm-up and of the phase."""
    n_warm = len(model_reports(warm))
    everything = model_reports(warm + phase)
    return everything, everything[:n_warm], everything[n_warm:]


@pytest.mark.gpu
def test_each_pool_hands_out_its_own_slots_while_the_delivery_thread_is_held():
    fs, h, fv = ts.SMALL
    blocks = ts._blocks(fs, h, fv, 24, 65536, seed=51)
    warm, phase = blocks[:12], blocks[12:]
    calls = [{"iq": b} for b in blocks]
    alphas = [h * fv] * len(calls)
    sp_all, _, sp_phase = _phase_reports(lambda bs: ts.model_reports(fs, [{"iq": b} for b in bs], SPEC), warm, phase)
    ch_all, _, ch_phase = _phase_reports(lambda bs: tc.model_reports(fs, [{"iq": b} for b in bs], COH, [h * fv] * len(bs)),
                                         warm, phase)
    assert len(sp_phase) > SLOTS and len(ch_phase) > SLOTS

    both = _held_run(SPEC, COH, warm, phase)
    spectra, cohs, st0, st1, timed_out = both
    assert timed_out == []
    # each report path: exactly its own slots during the hold, the rest skipped, every report produced accounted for
    for delivered, skipped, produced in (("spectra_delivered", "spectra_skipped", len(sp_all)),
                                         ("coherence_delivered", "coherence_skipped", len(ch_all))):
        assert getattr(st1, delivered) - getattr(st0, delivered) == SLOTS
        assert getattr(st1, skipped) > 0
        assert getattr(st1, delivered) + getattr(st1, skipped) == produced
    assert st1.spectra_skipped - st0.spectra_skipped == len(sp_phase) - SLOTS
    assert st1.coherence_skipped - st0.coherence_skipped == len(ch_phase) - SLOTS
    assert len(spectra) == st1.spectra_delivered and len(cohs) == st1.coherence_delivered
    # the delivered reports are the model's, in order; during the hold the first SLOTS of the phase
    ts._check_reports(([], [], [], spectra, st1), fs, calls, SPEC)
    tc._check_reports(([], [], [], cohs, st1, [], alphas), fs, calls, COH)
    for (_, off, v, sr), want in zip(spectra[-SLOTS:], sp_phase[:SLOTS]):
        assert off == -v.size // 2 and sr == fs and ts.max_amplitude_error(v, want) <= ts.TOL
    for (_, off, v, sr), want in zip(cohs[-SLOTS:], ch_phase[:SLOTS]):
        ok, bound = tc._gamma_bound(v.size, want)
        assert off == -v.size // 2 and sr == fs and np.all(np.abs(v - want[0])[ok] <= bound[ok])
    # frame batches are dropped whole, the autocorrelation plots keep to their own two slots
    assert st1.frames_dropped - st0.frames_dropped > 0 and st1.frames_dropped % BATCH == 0
    assert st1.frames_delivered == st1.frames_processed
    assert st1.plots_delivered - st0.plots_delivered == min(PLOT_SLOTS, st1.captures - st0.captures)

    # with the other path off, each path delivers and skips the same reports, bit for bit: the pools do not share slots
    alone_sp = _held_run(SPEC, "off", warm, phase)
    alone_ch = _held_run("off", COH, warm, phase)
    assert alone_sp[4] == [] and alone_ch[4] == []
    assert alone_sp[1] == [] and alone_ch[0] == []
    for got, alone in ((spectra, alone_sp[0]), (cohs, alone_ch[1])):
        assert len(got[-SLOTS:]) == len(alone[-SLOTS:]) == SLOTS
        for (_, _, v, _), (_, _, w, _) in zip(got[-SLOTS:], alone[-SLOTS:]):
            assert np.array_equal(v.view(np.uint64), w.view(np.uint64))
    assert alone_sp[3].spectra_skipped - alone_sp[2].spectra_skipped == st1.spectra_skipped - st0.spectra_skipped
    assert alone_ch[3].coherence_skipped - alone_ch[2].coherence_skipped == st1.coherence_skipped - st0.coherence_skipped
