"""The glitch-tolerant stack (TSDRGPU_STACK_ROBUST) as include/tsdrgpu.h defines it, in numpy, on top of
tests/stack_track_model.py.

`RobustModel` registers the frame as align does and measures and searches every tile as track does, then applies what robust
adds: the tile debounce (a tile restarts only when it was new in the last frame too, and is held otherwise), the frame hold (more
than half of the tiles held: the frame is left out and the offset stays on the prediction) and the pixel gate with its
persistence bit in bit 15 of the counts.  The arithmetic is track's: integers for the statistics, one numpy float32 operation per
float32 operation of the definition, so the GPU's output is expected bit for bit.  `robust_literal` walks the definition pixel by
pixel, tile by tile and candidate by candidate for tiny frames.
"""
import math

import numpy as np

from tests.stack_adapt_model import FLOOR, NO_LEVEL, RATIO, TILE, tile_grid, tile_sums
from tests.stack_model import F32, StackModel, quantise, rnd, valid_mask, weights
from tests.stack_track_model import LX, LY, TrackModel, _neighbours, search_tile, warped

GATE_MIN = 16 * FLOOR         # TSDRGPU_STACK_ROBUST_GATE_MIN
GATED = 0x8000                # bit 15 of a count: the pixel was gated in the last frame
COUNT = 0x7FFF


class RobustModel(TrackModel):
    """One robust stack's state; `run` takes one frame and returns (output, record dict with "changed").  After each frame,
    besides track's `vectors` and `moved`: `held` (tiles held), `gated` (pixels gated), `hold` (a glitch frame), as
    tsdrgpu_stack_robust_counts reports them, and `pend` (ty, tx) bool."""

    def restart(self):
        super().restart()
        self.pend = None
        self.held = self.gated = 0
        self.hold = False

    def run(self, frame, w, h):
        if (w, h) != (self.w, self.h):
            self.w, self.h = w, h
            self.restart()
        ty, tx = tile_grid(w, h)
        if self.m == 0:
            out, rec = super().run(frame, w, h)          # track's restart frame: c = 1, e_t = none
            self.pend = np.zeros((ty, tx), bool)
            self.held = self.gated = 0
            self.hold = False
            return out, rec
        r1 = rnd(self.o1)
        b = r1 + (r1 - rnd(self.o2) if self.m >= 2 else 0.0)
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
        new = changed & ~moved
        restart = _neighbours(new & self.pend)
        held = new & ~self.pend & ~restart
        self.pend = new
        self.moved = int(moved.sum())
        self.held, self.gated = int(held.sum()), 0
        self.hold = 2 * self.held > ty * tx
        valid = valid_mask(F)
        if self.hold:                                    # 6h: the frame is left out, the offset stays on the prediction
            self.o1, self.A = b, A_old
            rec["offset"], rec["changed"] = b, 0
            self.vectors = np.zeros((ty, tx, 2), np.int32)
            return np.where(valid, np.roll(A_old, int(rnd(b)) % n), F).astype(F32), rec
        carried = moved & ~restart
        r = (16 * D) // np.maximum(C, 1)
        e_new = np.where(C > 0, np.where(e == NO_LEVEL, r, (7 * e + r) // 8), e)
        e_new = np.where(carried, (7 * e + rstar) // 8, e_new)
        e_new = np.where(held, e, e_new)
        self.e = np.where(restart, NO_LEVEL, e_new)
        gate_e = np.where(restart | held, NO_LEVEL, e)
        vec = np.where(carried[..., None], vec, 0)
        expand = lambda a: np.repeat(np.repeat(a, TILE, 0), TILE, 1)[:h, :w].reshape(-1)
        X, Y = np.arange(n) % w, np.arange(n) // w
        sx, sy = X - expand(vec[..., 0]), Y - expand(vec[..., 1])
        src = ~expand(restart) & (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
        s = np.where(src, sy * w + sx, np.arange(n))
        craw = np.where(src, c_old[s], 0)
        g, cs = (craw & GATED) != 0, craw & COUNT
        k = np.minimum(cs + 1, self.depth)
        wn_tab = np.array([F32(1.0 / max(kk, 1)) for kk in range(self.depth + 1)], F32)
        wo_tab = np.array([F32(1.0 - 1.0 / max(kk, 1)) for kk in range(self.depth + 1)], F32)
        As = A_old[s]
        with np.errstate(invalid="ignore", over="ignore"):
            blend = np.where(ok, As * wo_tab[k] + x * wn_tab[k], As).astype(F32)
        ge = expand(gate_e)
        dq = qx - quantise(As)
        gated = ok & src & (ge != NO_LEVEL) & (dq * dq > np.maximum(ge, GATE_MIN))
        A_new = np.where(gated, np.where(g, x, As), blend).astype(F32)
        c_new = np.where(gated, np.where(g, 1, cs | GATED), k)
        hp = expand(held)
        self.A = np.where(hp, A_old, A_new).astype(F32)
        self.c = np.where(hp, c_old, c_new)
        self.gated = int(gated.sum())
        self.vectors = vec.astype(np.int32)
        out = np.where(valid, np.roll(self.A, int(rnd(o)) % n), F).astype(F32)
        rec["changed"] = int(restart.sum())
        return out, rec


def robust_literal(frames, w, h, depth, rx=8, ry=2):
    """The definition pixel by pixel, candidate by candidate and tile by tile, for tiny frames (a reference for RobustModel).
    -> (outputs, records, per-frame vectors {(tile y, tile x): (vx, vy)} of the tiles carried, per-frame (held, gated, hold))."""
    frames = np.asarray(frames, F32).reshape(-1, w * h)
    n = w * h
    tx, ty = (w + TILE - 1) // TILE, (h + TILE - 1) // TILE

    def valid(v):
        return not (v > 250.0 or v < -250.0) and v == v

    def q(v):
        return int(F32(F32(min(max(F32(v), F32(0)), F32(1))) * F32(255.0)) + F32(0.5))

    A, m, o1, o2, c, e, pend = None, 0, 0.0, 0.0, None, None, None
    outs, recs, vecs, counts = [], [], [], []
    for F in frames:
        if m == 0:
            A = [F32(v) if valid(v) else F32(0) for v in F]
            m, o1, o2 = 1, 0.0, 0.0
            c = [1] * n
            e = [[NO_LEVEL] * tx for _ in range(ty)]
            pend = [[False] * tx for _ in range(ty)]
            outs.append(F.copy())
            recs.append(dict(offset=0.0, score=0, dx=0, dy=0, restarted=1, changed=0))
            vecs.append({})
            counts.append((0, 0, False))
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
        # 6r: debounce
        new = [[changed[a][bb] and (a, bb) not in vstar for bb in range(tx)] for a in range(ty)]
        conf = [[new[a][bb] and pend[a][bb] for bb in range(tx)] for a in range(ty)]
        restart = [[any(conf[a2][b2] for a2 in range(max(a - 1, 0), min(a + 2, ty)) for b2 in range(max(bb - 1, 0), min(bb + 2, tx)))
                    for bb in range(tx)] for a in range(ty)]
        held = [[new[a][bb] and not pend[a][bb] and not restart[a][bb] for bb in range(tx)] for a in range(ty)]
        pend = new
        nheld = sum(sum(r) for r in held)
        m += 1
        if 2 * nheld > tx * ty:              # 6h: a glitch frame
            o = float(b)
            Ro = math.floor(o + 0.5)
            outs.append(np.array([F[p] if not valid(F[p]) else A[(p - Ro) % n] for p in range(n)], F32))
            recs.append(dict(offset=o, score=bs, dx=dx, dy=dy, restarted=0, changed=0))
            vecs.append({})
            counts.append((nheld, 0, True))
            o2, o1 = o1, o
            continue
        moves, gate = {}, {}
        for a in range(ty):
            for bb in range(tx):
                gate[(a, bb)] = NO_LEVEL if restart[a][bb] or held[a][bb] else e[a][bb]
                if restart[a][bb]:
                    e[a][bb] = NO_LEVEL
                elif held[a][bb]:
                    pass
                elif (a, bb) in vstar:
                    vx, vy, Dv, Cv = vstar[(a, bb)]
                    e[a][bb] = (7 * e[a][bb] + 16 * Dv // Cv) // 8
                    moves[(a, bb)] = (vx, vy)
                elif D0[a][bb][1] > 0:
                    r = 16 * D0[a][bb][0] // D0[a][bb][1]
                    e[a][bb] = r if e[a][bb] == NO_LEVEL else (7 * e[a][bb] + r) // 8
        newA, newc, ngated = list(A), list(c), 0
        for qq in range(n):
            X, Y = qq % w, qq // w
            a, bb = Y // TILE, X // TILE
            if held[a][bb]:
                continue                     # A and c stay, the gate bit included
            vx, vy = moves.get((a, bb), (0, 0))
            sX, sY = X - vx, Y - vy
            inside = not restart[a][bb] and 0 <= sX < w and 0 <= sY < h
            if inside:
                sq = sY * w + sX
                cs, g = c[sq] & COUNT, c[sq] & GATED
            else:
                sq, cs, g = qq, 0, 0
            k = min(cs + 1, depth)
            newA[qq], newc[qq] = A[sq], k
            if qq not in xs:
                continue
            lev = gate[(a, bb)]
            dd = q(xs[qq]) - q(A[sq])
            if inside and lev != NO_LEVEL and dd * dd > max(lev, GATE_MIN):
                ngated += 1
                if g:
                    newA[qq], newc[qq] = xs[qq], 1
                else:
                    newc[qq] = cs | GATED
            else:
                newA[qq] = F32(F32(A[sq] * F32(1.0 - 1.0 / k)) + F32(xs[qq] * F32(1.0 / k)))
        A, c = newA, newc
        Ro = math.floor(o + 0.5)
        outs.append(np.array([F[p] if not valid(F[p]) else A[(p - Ro) % n] for p in range(n)], F32))
        recs.append(dict(offset=o, score=bs, dx=dx, dy=dy, restarted=0, changed=sum(sum(r) for r in restart)))
        vecs.append(moves)
        counts.append((nheld, ngated, False))
        o2, o1 = o1, o
    return np.stack(outs), recs, vecs, counts
