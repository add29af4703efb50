"""CPU: the frame sequences of the mid-batch sync hand-off tests (tests/test_production_batches.py) really hand off mid-batch.

The frame stage's sync search (csrc/framestage.cu) first walks a batch's frames with look-ups in speculation tables that
fs_sync_prep builds for the carried strip sizes within +-4*FS_SPEC_J of the size the batch starts with; the first frame that
asks for a size outside its table, or whose strip failed the exactness certificate, is handed to the cluster kernel fs_sync,
which continues from there.  Whether a sequence exercises that hand-off is decided by the reference's own per-frame strip
sizes, so the check runs on the oracle alone: a case whose input drifts out of the hand-off it was built for fails here
instead of passing silently on the GPU.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from tempestsdr_b200 import synth

FS_SPEC_J = 3                     # framestage.cu: the table covers carried sizes cur0 + 4j, |j| <= FS_SPEC_J
CERT_BITS = 29                    # framestage.cu fs_sync_prep: exact iff the blurred strip's exponent span < 29 - ceil(log2 n)

# (samplerate, height, refresh rate) of every case: BASELINE configs[0], 507 x 525 frames
FS, H, FV = 8_000_000, 525, 60.0


def candidates(cur, size, minsize):
    """syncdetector.c:73-93 (framestage.cu sweet_candidates): the carried size, clamped, and the sizes tried after it."""
    minsize = max(minsize, 1)
    half = size >> 1
    cur = min(max(cur, minsize), half)
    return [cur] + [t for t in (cur - 4, cur + 4, cur >> 1, cur << 1) if minsize <= t < half and t != cur]


def table(cur0, size, minsize):
    """The strip sizes fs_sync_prep scores for every frame of a batch that starts with carried size cur0."""
    minsize = max(minsize, 1)
    half = size >> 1
    cur0 = min(max(cur0, minsize), half)
    out = set()
    for j in range(-FS_SPEC_J, FS_SPEC_J + 1):
        c = cur0 + 4 * j
        if minsize <= c <= half:
            out.update(candidates(c, size, minsize))
    return out


def exact_ok(strip):
    """fs_sync_prep's exactness certificate on a collapsed strip (the blur taken in float here: the margins asserted below
    are far wider than the difference)."""
    b = orc.port().gaussianblur(strip)
    bits = b.view(np.uint32)
    e, m = (bits >> 23) & 0xFF, bits & 0x7FFFFF
    if np.any((e == 0) & (m != 0)) or np.any(e == 255):
        return False, 255
    live = e[e > 0]
    span = int(live.max() - live.min()) if live.size else 0
    lg = int(np.ceil(np.log2(strip.size)))
    return span < CERT_BITS - lg, span


def walker_stop(carried0, strips, w, h, cert=None):
    """(first frame of a batch the table walker cannot serve, why): why is "x" or "y" (that axis' carried size asks for a strip
    size outside its table) or "cert" (the frame's strips failed the exactness certificate); (len(strips), None) when it serves
    them all.  carried0: (x, y) strip sizes the batch starts with; strips[f] = (x, y) strip sizes the reference leaves after
    frame f; cert[f]: False where frame f's strips fail the certificate."""
    mins = (int(w * np.float32(0.05)), int(h * np.float32(0.01)))        # syncdetector.c:178-179, (int)(w * 0.05f)
    tabs = [table(carried0[ax], (w, h)[ax], mins[ax]) for ax in (0, 1)]
    carried = carried0
    for f, s in enumerate(strips):
        if cert is not None and not cert[f]:
            return f, "cert"
        for ax in (0, 1):
            if not set(candidates(carried[ax], (w, h)[ax], mins[ax])) <= tabs[ax]:
                return f, "xy"[ax]
        carried = s
    return len(strips), None


def _run_oracle(frames, w, h, po, lpbs, aap):
    return [(r.x.curr_stripsize, r.y.curr_stripsize) for r in (po.run(f, w, h, 0.0, 0.1, lpbs, aap)[1] for f in frames)]


def case_frames(name):
    """-> (w, h, [priming batch, 64-frame batch], flags).  The first batch brings the frame stage's strip sizes to where the
    case starts; the hand-off is asserted in the second."""
    w, h = 507, 525
    if name == "leave_window":
        # (a) the blanking of the second batch is 40 columns wider than that of the first: the x strip grows by 4 per frame
        # and its carried size leaves the +-12 window of the batch's starting size at frame 4
        prime = [synth.video_like_frame(w, h, seed=200 + k, shift_x=50 + 2 * k, shift_y=30) for k in range(8)]
        batch = [synth.video_like_frame(w, h, seed=300 + k, shift_x=66 + 3 * k, shift_y=30, blank_frac_x=0.22) for k in range(64)]
        return w, h, [prime, batch], dict(lpbs=1, aap=0)
    if name == "halve":
        # (b) the blanking halves in width at frame 10 of the second batch: the best x strip size halves there, and the
        # next frame's candidates (a quarter of the old size among them) are not in the table
        prime = [synth.video_like_frame(w, h, seed=400 + k, shift_x=40 + 2 * k, shift_y=30, blank_frac_x=0.28) for k in range(16)]
        batch = [synth.video_like_frame(w, h, seed=500 + k, shift_x=56 + 3 * k, shift_y=30, blank_frac_x=0.28 if k < 10 else 0.14)
                 for k in range(64)]
        return w, h, [prime, batch], dict(lpbs=1, aap=0)
    if name == "bad_frame":
        # (c) frame 20 of the second batch has 15 columns of zeros around one pixel of 1e-30: its blurred column strip spans
        # ~2^111, far past the certificate's 2^20, while every other frame spans ~2^4.  Auto-gain after processing and no
        # motion blur, so the collapse sees the raw frames (as in test_gpu_parity.py::test_sync_search_serial_fallback).
        prime = [synth.video_like_frame(w, h, seed=600 + k, shift_x=50 + 2 * k, shift_y=30) for k in range(8)]
        batch = [synth.video_like_frame(w, h, seed=700 + k, shift_x=66 + 2 * k, shift_y=30) for k in range(64)]
        f = batch[20].reshape(h, w)
        f[:, 200:215] = 0.0
        f[0, 207] = 1e-30
        return w, h, [prime, batch], dict(lpbs=1, aap=1)
    raise KeyError(name)


# where and why the walker must hand the second batch over
CASES = {"leave_window": (4, "x"), "halve": (11, "x"), "bad_frame": (20, "cert")}


def handoff(name):
    """(frame, why, per-frame strip sizes of the second batch, the sizes it starts with), from the oracle alone."""
    w, h, batches, fl = case_frames(name)
    po = orc.best().postprocessor(FS, H, FV, 1, 0)
    first = _run_oracle(batches[0], w, h, po, fl["lpbs"], fl["aap"])
    strips = _run_oracle(batches[1], w, h, po, fl["lpbs"], fl["aap"])
    cert = None
    if fl["aap"]:                  # the collapse sees the raw frames: the certificate can be evaluated on them
        cert = []
        for fr in batches[1]:
            wb, hb = orc.port().average_v_h(fr, w, h)
            cert.append(exact_ok(wb)[0] and exact_ok(hb)[0])
    f0, why = walker_stop(first[-1], strips, w, h, cert)
    return f0, why, strips, first[-1], cert


@pytest.mark.parametrize("name", list(CASES))
def test_handoff_happens_mid_batch(name):
    f0, why, strips, carried0, cert = handoff(name)
    assert (f0, why) == CASES[name], f"{name}: the walker hands over at frame {f0} ({why}); starting sizes {carried0}, strips {strips[:f0 + 2]}"
    assert 3 <= f0 <= len(strips) - 3
    if name == "halve":
        assert strips[9][0] == 2 * strips[10][0], strips[8:12]           # the strip size really halves at the blanking change
    if name == "bad_frame":
        assert cert.count(False) == 1                                   # one bad frame; the frames after it take the prefix sums
        w, h, batches, _ = case_frames(name)
        assert exact_ok(orc.port().average_v_h(batches[1][20], w, h)[0])[1] > 60
        assert walker_stop(carried0, strips, w, h)[0] == len(strips)    # without it the tables would have served the whole batch
