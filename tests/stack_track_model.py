"""The motion-tracking stack (TSDRGPU_STACK_TRACK) as include/tsdrgpu.h defines it, in numpy, on top of
tests/stack_adapt_model.py.

Registration is the align stack's and the tile statistic adapt's, so `TrackModel` lets `StackModel.run` register the frame and
then redoes step 6: adapt's per-tile residual, the local search of every changed tile, the restart rule, the levels, and the
blend with per-pixel counts gathered along each moved tile's vector.  The search is integer arithmetic (int64 numpy); D/C of two
candidates is compared in float64, which orders distinct ratios of integers below 2^24 over counts up to 256 exactly and gives
equal ratios the same value.  Every float32 operation of the blend is the one numpy float32 operation the definition gives, so
the GPU's output is expected bit for bit.  `track_literal` walks the definition pixel by pixel, tile by tile and candidate by
candidate for tiny frames.
"""
import math

import numpy as np

from tests.stack_adapt_model import FLOOR, NO_LEVEL, RATIO, TILE, AdaptModel, tile_grid, tile_sums
from tests.stack_model import F32, StackModel, quantise, rnd, valid_mask, weights

LX = 16                       # TSDRGPU_STACK_TRACK_LX
LY = 32                       # TSDRGPU_STACK_TRACK_LY
NX = 2 * LX + 1


def _neighbours(mask):
    ty, tx = mask.shape
    p = np.pad(mask, 1)
    out = np.zeros_like(mask)
    for a in range(3):
        for b in range(3):
            out |= p[a:a + ty, b:b + tx]
    return out


def search_tile(qx, ok, qA, w, h, ti, tj):
    """6t for tile (ti, tj): qx, ok = Q(x) and the valid-taps mask as (h, w) arrays, qA = Q(A) as (h, w).
    -> (vx, vy, D, C) of v*, or None when no candidate is admissible."""
    X0, Y0 = tj * TILE, ti * TILE
    tq = np.zeros((TILE, TILE), np.int64)
    tm = np.zeros((TILE, TILE), bool)
    hh, ww = min(TILE, h - Y0), min(TILE, w - X0)
    tq[:hh, :ww] = qx[Y0:Y0 + hh, X0:X0 + ww]
    tm[:hh, :ww] = ok[Y0:Y0 + hh, X0:X0 + ww]
    c0 = int(tm.sum())
    pad = np.full((h + 2 * LY + TILE, w + 2 * LX + TILE), -1, np.int64)
    pad[LY:LY + h, LX:LX + w] = qA
    win = pad[Y0:Y0 + TILE + 2 * LY, X0:X0 + TILE + 2 * LX]
    sw = np.lib.stride_tricks.sliding_window_view(win, (TILE, TILE))         # sw[a, b] = the source of v = (LX - b, LY - a)
    use = tm & (sw >= 0)
    d = np.where(use, tq - sw, 0)
    D = (d * d).sum(axis=(2, 3))[::-1, ::-1]                                  # [vy + LY, vx + LX]
    C = use.sum(axis=(2, 3))[::-1, ::-1]
    vy, vx = np.meshgrid(np.arange(-LY, LY + 1), np.arange(-LX, LX + 1), indexing="ij")
    adm = (C > 0) & (2 * C >= c0) & ~((vx == 0) & (vy == 0))
    if not adm.any():
        return None
    idx = np.arange(adm.size).reshape(adm.shape)
    ratio = D[adm] / C[adm].astype(np.float64)
    l1 = (np.abs(vx) + np.abs(vy))[adm]
    k = np.lexsort((idx[adm], l1, ratio))[0]
    i = idx[adm][k]
    return int(vx.flat[i]), int(vy.flat[i]), int(D.flat[i]), int(C.flat[i])


def warped(F, o):
    """Step 5: x (float32, n) and the mask of the pixels whose four taps are valid."""
    n = F.size
    valid = valid_mask(F)
    I = math.floor(o)
    wm1, w0, w1, w2 = weights(F32(o - I))
    base = (np.arange(n) + (I - 1)) % n
    f0, f1, f2, f3 = F[base], F[(base + 1) % n], F[(base + 2) % n], F[(base + 3) % n]
    ok = valid[base] & valid[(base + 1) % n] & valid[(base + 2) % n] & valid[(base + 3) % n]
    with np.errstate(invalid="ignore", over="ignore"):
        x = ((wm1 * f0 + w0 * f1) + w1 * f2) + w2 * f3
    return np.where(ok, x, F32(0)).astype(F32), ok


class TrackModel(AdaptModel):
    """One tracking stack's state; `run` takes one frame and returns (output, record dict with "changed").  After each frame,
    `vectors` holds (ty, tx, 2) int32: (vx, vy) of every tile that moved and did not restart, (0, 0) elsewhere; `moved` the
    number of tiles with moved_t (restarted by a neighbour or not)."""

    def restart(self):
        super().restart()
        self.c = self.vectors = None
        self.moved = 0

    def run(self, frame, w, h):
        if (w, h) != (self.w, self.h):
            self.w, self.h = w, h
            self.restart()
        ty, tx = tile_grid(w, h)
        if self.m == 0:
            out, rec = super().run(frame, w, h)          # adapt's restart frame: m_t = 1, e_t = none
            self.c = np.ones(w * h, np.int64)
            self.vectors = np.zeros((ty, tx, 2), np.int32)
            self.moved = 0
            return out, rec
        A_old, c_old = self.A, self.c
        _, rec = StackModel.run(self, frame, w, h)       # registration, o and m as align; its blend is redone below
        o = rec["offset"]
        F = np.asarray(frame, F32).reshape(-1)
        n = F.size
        x, ok = warped(F, o)
        qx, qA = quantise(x), quantise(A_old)
        d = np.where(ok, qx - qA, 0)
        D, C = tile_sums(d * d, w, h), tile_sums(ok, w, h)
        e = self.e
        changed = (C > 0) & (e != NO_LEVEL) & (16 * D > RATIO * e * C) & (D > FLOOR * C)
        moved = np.zeros_like(changed)
        vec = np.zeros((ty, tx, 2), np.int64)
        rstar = np.zeros((ty, tx), np.int64)
        for ti, tj in zip(*np.nonzero(changed)):
            best = search_tile(qx.reshape(h, w), ok.reshape(h, w), qA.reshape(h, w), w, h, ti, tj)
            if best is None:
                continue
            vx, vy, Dv, Cv = best
            if not (16 * Dv > RATIO * e[ti, tj] * Cv and Dv > FLOOR * Cv):
                moved[ti, tj] = True
                vec[ti, tj] = vx, vy
                rstar[ti, tj] = 16 * Dv // Cv
        restart = _neighbours(changed & ~moved)
        carried = moved & ~restart
        r = (16 * D) // np.maximum(C, 1)
        e_new = np.where(C > 0, np.where(e == NO_LEVEL, r, (7 * e + r) // 8), e)
        e_new = np.where(carried, (7 * e + rstar) // 8, e_new)
        self.e = np.where(restart, NO_LEVEL, e_new)
        vec = np.where(carried[..., None], vec, 0)
        expand = lambda a: np.repeat(np.repeat(a, TILE, 0), TILE, 1)[:h, :w].reshape(-1)
        X, Y = np.arange(n) % w, np.arange(n) // w
        sx, sy = X - expand(vec[..., 0]), Y - expand(vec[..., 1])
        src = ~expand(restart) & (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
        s = np.where(src, sy * w + sx, np.arange(n))
        k = np.minimum(np.where(src, c_old[s], 0) + 1, self.depth)
        wn_tab = np.array([F32(1.0 / max(kk, 1)) for kk in range(self.depth + 1)], F32)
        wo_tab = np.array([F32(1.0 - 1.0 / max(kk, 1)) for kk in range(self.depth + 1)], F32)
        As = A_old[s]
        with np.errstate(invalid="ignore", over="ignore"):
            self.A = np.where(ok, As * wo_tab[k] + x * wn_tab[k], As).astype(F32)
        self.c = k
        self.vectors = vec.astype(np.int32)
        self.moved = int(moved.sum())
        out = np.where(valid_mask(F), np.roll(self.A, int(rnd(o)) % n), F).astype(F32)
        rec["changed"] = int(restart.sum())
        return out, rec


def track_literal(frames, w, h, depth, rx=8, ry=2):
    """The definition pixel by pixel, candidate by candidate and tile by tile, for tiny frames (a reference for TrackModel).
    -> (outputs, records, per-frame vectors {(tile y, tile x): (vx, vy)} of the tiles that moved and did not restart)."""
    frames = np.asarray(frames, F32).reshape(-1, w * h)
    n = w * h
    tx, ty = (w + TILE - 1) // TILE, (h + TILE - 1) // TILE

    def valid(v):
        return not (v > 250.0 or v < -250.0) and v == v

    def q(v):
        return int(F32(F32(min(max(F32(v), F32(0)), F32(1))) * F32(255.0)) + F32(0.5))

    A, m, o1, o2, c, e = None, 0, 0.0, 0.0, None, None
    outs, recs, vecs = [], [], []
    for F in frames:
        if m == 0:
            A = [F32(v) if valid(v) else F32(0) for v in F]
            m, o1, o2 = 1, 0.0, 0.0
            c = [1] * n
            e = [[NO_LEVEL] * tx for _ in range(ty)]
            outs.append(F.copy())
            recs.append(dict(offset=0.0, score=0, dx=0, dy=0, restarted=1, changed=0))
            vecs.append({})
            continue
        qF = [q(v) if valid(v) else 0 for v in F]
        qA = [q(v) for v in A]
        r1 = math.floor(o1 + 0.5)
        b = r1 + (r1 - math.floor(o2 + 0.5) if m >= 2 else 0)
        best, bs, cand = None, None, []
        for dy in range(-ry, ry + 1):
            for dx in range(-rx, rx + 1):
                s = b + dy * w + dx
                S = sum(qF[(qq + s) % n] * qA[qq] for qq in range(n))
                cand.append(S)
                if bs is None or S > bs:
                    best, bs = (dy, dx, s, len(cand) - 1), S
        dy, dx, s, kk = best
        delta = 0.0
        if -rx < dx < rx:
            a, cc, M = float(cand[kk - 1]), float(cand[kk + 1]), float(bs)
            den = (a - 2.0 * M) + cc
            if den < 0:
                delta = min(max((a - cc) / (2.0 * den), -0.5), 0.5)
        o = float(s) + delta
        I = math.floor(o)
        wm1, w0, w1, w2 = weights(F32(o - I))
        xs = {}
        for qq in range(n):
            taps = [F[(qq + I - 1 + j) % n] for j in range(4)]
            if all(valid(v) for v in taps):
                xs[qq] = F32(F32(F32(F32(wm1 * taps[0]) + F32(w0 * taps[1])) + F32(w1 * taps[2])) + F32(w2 * taps[3]))

        def sums(a, bb, vx, vy):             # D_t(v), C_t(v) of tile (a, bb)
            Dv = Cv = 0
            for Y in range(a * TILE, min(a * TILE + TILE, h)):
                for X in range(bb * TILE, min(bb * TILE + TILE, w)):
                    sX, sY = X - vx, Y - vy
                    if Y * w + X in xs and 0 <= sX < w and 0 <= sY < h:
                        dd = q(xs[Y * w + X]) - qA[sY * w + sX]
                        Dv += dd * dd
                        Cv += 1
            return Dv, Cv

        def test(Dv, Cv, lev):               # 6b's change test
            return 16 * Dv > RATIO * lev * Cv and Dv > FLOOR * Cv

        D0 = [[sums(a, bb, 0, 0) for bb in range(tx)] for a in range(ty)]
        changed = [[D0[a][bb][1] > 0 and e[a][bb] != NO_LEVEL and test(*D0[a][bb], e[a][bb]) for bb in range(tx)] for a in range(ty)]
        vstar = {}
        for a in range(ty):
            for bb in range(tx):
                if not changed[a][bb]:
                    continue
                c0, top = D0[a][bb][1], None
                for vy in range(-LY, LY + 1):
                    for vx in range(-LX, LX + 1):
                        if vx == 0 and vy == 0:
                            continue
                        Dv, Cv = sums(a, bb, vx, vy)
                        if Cv == 0 or 2 * Cv < c0:
                            continue
                        if top is None:
                            top = (vx, vy, Dv, Cv)
                            continue
                        tvx, tvy, tD, tC = top
                        if Dv * tC < tD * Cv or (Dv * tC == tD * Cv and abs(vx) + abs(vy) < abs(tvx) + abs(tvy)):
                            top = (vx, vy, Dv, Cv)
                if top is not None and not test(top[2], top[3], e[a][bb]):
                    vstar[(a, bb)] = top
        cm = [[changed[a][bb] and (a, bb) not in vstar for bb in range(tx)] for a in range(ty)]
        restart = [[any(cm[a2][b2] for a2 in range(max(a - 1, 0), min(a + 2, ty)) for b2 in range(max(bb - 1, 0), min(bb + 2, tx)))
                    for bb in range(tx)] for a in range(ty)]
        moves = {}
        for a in range(ty):
            for bb in range(tx):
                if restart[a][bb]:
                    e[a][bb] = NO_LEVEL
                elif (a, bb) in vstar:
                    vx, vy, Dv, Cv = vstar[(a, bb)]
                    e[a][bb] = (7 * e[a][bb] + 16 * Dv // Cv) // 8
                    moves[(a, bb)] = (vx, vy)
                elif D0[a][bb][1] > 0:
                    r = 16 * D0[a][bb][0] // D0[a][bb][1]
                    e[a][bb] = r if e[a][bb] == NO_LEVEL else (7 * e[a][bb] + r) // 8
        newA, newc = list(A), list(c)
        for qq in range(n):
            X, Y = qq % w, qq // w
            a, bb = Y // TILE, X // TILE
            vx, vy = moves.get((a, bb), (0, 0))
            sX, sY = X - vx, Y - vy
            if restart[a][bb] or not (0 <= sX < w and 0 <= sY < h):
                sq, cs = qq, 0
            else:
                sq, cs = sY * w + sX, c[sY * w + sX]
            k = min(cs + 1, depth)
            if qq in xs:
                newA[qq] = F32(F32(A[sq] * F32(1.0 - 1.0 / k)) + F32(xs[qq] * F32(1.0 / k)))
            else:
                newA[qq] = A[sq]
            newc[qq] = k
        A, c = newA, newc
        m += 1
        Ro = math.floor(o + 0.5)
        outs.append(np.array([F[p] if not valid(F[p]) else A[(p - Ro) % n] for p in range(n)], F32))
        recs.append(dict(offset=o, score=bs, dx=dx, dy=dy, restarted=0, changed=sum(sum(r) for r in restart)))
        vecs.append(moves)
        o2, o1 = o1, o
    return np.stack(outs), recs, vecs
