"""cfmm_solve's outer iteration (cfmm_capi.cu, csrc/solver.cuh) restated in numpy, for the tests.

The restatement takes the same decisions in the same order as the device: x = P(v0) (default
start 1/n), t_init = min(1, 1/|pg|₂) on an empty history, the two-loop recursion in coefficient
space over the basis [S Y pg] with the history slots in age order, Armijo backtracking along the
projected path with the noise slack 8·eps·max(|f|, |f_new|, 1) and the quadratic step clamped to
[0.1t, 0.5t], the restart from −pg when the line search fails with a history, the curvature test
sy > 1e-10·yy, factr on two consecutive steps, and statuses 0–5.  Every reduction is math.fsum
(the device's fixed-order tree sums are within a few ulp of it); Ψ and acc come from a callback
sweep(ν) -> (Ψ, acc): the device's own DevicePools.sweep, or 50-digit pool responses.

Per accepted iteration it records the iterate and:
  margins   how far each decision was from going the other way, relative to its scale:
              armijo     |f_new − (f + 1e-4·gᵀΔx + noise)| / max(|f|, |f_new|, 1), every trial
              descent    |gᵀΔx| / Σ|g_i Δx_i|, every trial (the sign decides restart vs backtrack)
              curvature  |sy − 1e-10·yy| / max(|sy|, 1e-10·yy)
              factr      |(f_old − f) − factr·eps·max(|f_old|, |f|, 1)| / max(|f_old|, |f|, 1)
              pgtol      |‖pg‖∞ − pgtol| / pgtol, at the test that let the iteration run
  branches  backtracks (rejected trials), restart (the history was dropped before this step),
            curvature_skip (the pair was not kept), wrap (the pair overwrote a kept slot),
            activated (coordinates that moved onto a bound).
Two runs whose Ψ differ in their last bits take the same branches while every margin is well above
that noise, so iterates compare up to the first iteration with a small margin.
"""
from __future__ import annotations

import math

import numpy as np

M = 5                 # kSolverM
K = 2 * M + 1         # basis columns: s_1..s_M, y_1..y_M, pg
EPSMCH = 2.220446049250313e-16


def fsum(a):
    return math.fsum(np.asarray(a, dtype=np.float64).ravel().tolist())


def _rel(a, b, scale):
    return abs(a - b) / scale if scale > 0 else math.inf


def solve(sweep, lower, lin=None, upper=None, v0=None, pgtol=1e-5, factr=1e1, maxfun=15_000,
          maxiter=15_000):
    """Returns (x, info, trace).  info: iterations, fun_evals, status, f, pg_norm as cfmm_solve's;
    trace: one dict per accepted iteration (x, margins, branches; see the module docstring)."""
    lower = np.asarray(lower, dtype=np.float64)
    n = len(lower)
    lin = np.zeros(n) if lin is None else np.asarray(lin, dtype=np.float64)
    if upper is not None:
        upper = np.asarray(upper, dtype=np.float64)
        if not np.any(upper < 1.0e300):
            upper = None          # no finite bound: the device runs without one
    x0 = np.full(n, 1.0 / n) if v0 is None else np.asarray(v0, dtype=np.float64)

    def proj(y):
        y = np.maximum(y, lower)
        return y if upper is None else np.minimum(y, upper)

    def at_bound_out(x, g):
        out = (x <= lower) & (g > 0.0)
        if upper is not None:
            out |= (x >= upper) & (g < 0.0)
        return out

    S, Y = np.zeros((M, n)), np.zeros((M, n))
    fevals = 0

    def evaluate(xt):
        nonlocal fevals
        psi, acc = sweep(xt)
        fevals += 1
        return fsum(lin * xt) + acc, lin + np.asarray(psi, dtype=np.float64)

    def gram(pg):
        B = list(S) + list(Y) + [pg]
        W = np.zeros((K, K))
        for r in range(K):
            for c in range(r, K):
                W[r, c] = W[c, r] = fsum(B[r] * B[c])
        return W

    x = proj(x0)
    f, g = evaluate(x)
    pg = np.where(at_bound_out(x, g), 0.0, g)
    pgnorm = float(np.max(np.abs(pg))) if n else 0.0
    W = gram(pg)

    age, cnt, head, it, status, small = [0] * M, 0, 0, 0, 2, 0
    filled = [False] * M
    trace = []
    restarted = False
    while True:
        if not (f == f):
            status = 5
            break
        if pgnorm <= pgtol:
            status = 0
            break
        if it >= maxiter:
            status = 2
            break
        if fevals >= maxfun:
            status = 3
            break
        margins = {"pgtol": _rel(pgnorm, pgtol, pgtol), "armijo": [], "descent": []}
        # two-loop recursion in coefficient space
        c = np.zeros(K)
        c[K - 1] = 1.0
        t_init = 1.0
        if cnt == 0:
            nrm = math.sqrt(W[K - 1, K - 1])
            t_init = min(1.0, 1.0 / nrm) if nrm > 0.0 else 1.0
        else:
            alpha, rho = [0.0] * M, [0.0] * M
            for a in range(cnt - 1, -1, -1):
                j = age[a]
                rho[a] = 1.0 / W[j, M + j]
                alpha[a] = rho[a] * fsum(W[j] * c)
                c[M + j] -= alpha[a]
            jn = age[cnt - 1]
            c *= W[jn, M + jn] / W[M + jn, M + jn]
            for a in range(cnt):
                j = age[a]
                c[j] += alpha[a] - rho[a] * fsum(W[M + j] * c)
        r = c[K - 1] * pg
        for j in range(M):
            r = r + c[j] * S[j]
            r = r + c[M + j] * Y[j]
        d = np.where(at_bound_out(x, g), 0.0, -r)
        # Armijo backtracking along the projected path
        t, f_new = t_init, f
        accepted = stalled = False
        backtracks = 0
        ls = 0
        while ls < 30 and fevals < maxfun:
            ls += 1
            xt = proj(x + t * d)
            dx = xt - x
            gdx, step2 = fsum(g * dx), fsum(dx * dx)
            f_new, gt = evaluate(xt)
            if step2 == 0.0:
                stalled = True
                break
            noise = 8.0 * EPSMCH * max(abs(f), abs(f_new), 1.0)
            rhs = f + 1e-4 * gdx + noise
            margins["armijo"].append(_rel(f_new, rhs, max(abs(f), abs(f_new), 1.0)))
            margins["descent"].append(_rel(gdx, 0.0, fsum(np.abs(g * dx))))
            if gdx < 0.0 and f_new <= rhs:
                accepted = True
                break
            if not (gdx < 0.0) and cnt > 0:
                break
            backtracks += 1
            if f_new == f_new and f_new < 1e300 and gdx < 0.0:
                slope, denom = gdx / t, 2.0 * (f_new - f - gdx)
                tq = -slope * t * t / denom if denom > 0.0 else 0.5 * t
                t = min(0.5 * t, max(0.1 * t, tq))
            else:
                t *= 0.1
        if not accepted:
            if cnt > 0 and not stalled:
                cnt = 0
                restarted = True
                continue
            status = 1 if stalled else 4
            break
        # accept: (s, y) into the head slot, new projected gradient and Gram matrix
        slot = head
        wrap = filled[slot]
        activated = int(np.sum((xt <= lower) & (x > lower)))
        if upper is not None:
            activated += int(np.sum((xt >= upper) & (x < upper)))
        S[slot], Y[slot] = xt - x, gt - g
        filled[slot] = True
        x, g = xt, gt
        pg = np.where(at_bound_out(x, g), 0.0, g)
        pgnorm = float(np.max(np.abs(pg)))
        W = gram(pg)
        # drop the slot's old pair from the age list, append the new one if its curvature is usable
        kept_slots = [a for a in age[:cnt] if a != slot]
        cnt = len(kept_slots)
        age = kept_slots + [0] * (M - cnt)
        sy, yy = W[slot, M + slot], W[M + slot, M + slot]
        margins["curvature"] = _rel(sy, 1e-10 * yy, max(abs(sy), 1e-10 * yy))
        kept = sy > 1e-10 * yy and yy > 0.0
        if kept:
            age[cnt] = slot
            cnt += 1
            head = (head + 1) % M
        it += 1
        f_old, f = f, f_new
        thr = factr * EPSMCH * max(abs(f_old), abs(f), 1.0)
        margins["factr"] = _rel(f_old - f, thr, max(abs(f_old), abs(f), 1.0))
        trace.append({"x": x.copy(), "f": f, "pg_norm": pgnorm, "t": t, "margins": margins,
                      "min_margin": min([margins["pgtol"], margins["curvature"], margins["factr"]]
                                        + margins["armijo"] + margins["descent"]),
                      "backtracks": backtracks, "restart": restarted, "curvature_skip": not kept,
                      "wrap": wrap, "activated": activated})
        restarted = False
        if f_old - f <= thr:
            small += 1
            if small >= 2:
                status = 1
                break
        else:
            small = 0
    info = {"iterations": it, "fun_evals": fevals, "status": status, "f": f, "pg_norm": pgnorm}
    return x, info, trace
