"""Times cfmm_quote_price_arbitrage on one GPU; prints one JSON line per measurement.

  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).  A is |A| tokens reached
            breadth-first over the pools from token 1, so the mask's tokens hold pools among them.
  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.  A is
            tokens 1..|A| (the hubs first).
|A| in {8, 64, 258}.  Each row prices every token of A: the set's reference prices (ones on the
headline set, whose pools disagree on prices; the hub set's ν, which its pools follow within 2 %) times
exp(U(−0.02, 0.02)) per token and row.  Default options.  Per quote call: the wall time of the
synchronous call (host clock), the kernel time (CUDA events, option "profile": the slot graph, plan and
row kernels), the fill rate, the mean iterations and evaluations, the m_r of the rows that did not fill
(min, median, max), and the mean tokens and pools per row.  Each configuration runs on 1k rows first; the
100k-row call runs when the 1k-row kernel time predicts at most --budget-s seconds for it, and is
reported as not run (with the estimate) otherwise.

    python tools/price_arbitrage_timing.py [--only hub|headline] [--budget-s 60]
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402
from routed_order_timing import hub_set, timed  # noqa: E402
from split_order_timing import card  # noqa: E402
from subgraph_order_timing import emit  # noqa: E402

SIZES = (8, 64, 258)


def bfs_tokens(Ai, n, k, start=1):
    """k tokens (1-based) reached breadth-first over the pools from `start`, ascending."""
    a = np.concatenate([Ai[:, 0], Ai[:, 1]])
    b = np.concatenate([Ai[:, 1], Ai[:, 0]])
    o = np.argsort(a, kind="stable")
    off = np.zeros(n + 2, np.int64)
    np.add.at(off, a + 1, 1)
    off, nbr = np.cumsum(off), b[o]
    seen, frontier = [start], [start]
    got = {start}
    while frontier and len(seen) < k:
        nxt = []
        for t in frontier:
            for u in np.unique(nbr[off[t]:off[t + 1]]).tolist():
                if u not in got and len(seen) < k:
                    got.add(u)
                    seen.append(u)
                    nxt.append(u)
        frontier = nxt
    return np.array(sorted(seen), np.int64)


def run(p, name, n, A, base, rng, budget_s):
    allowed = np.zeros(n, bool)
    allowed[A - 1] = True
    est = None
    for q in (1_000, 100_000):
        if q > 1_000 and est > budget_s * 1e3:
            emit(set=name, nA=len(A), q=q, run=False, est_kernel_ms=round(est, 1))
            continue
        c = base[None, :] * np.exp(rng.uniform(-0.02, 0.02, size=(q, len(A))))
        o, wall, ms, launches = timed(p, lambda: p.quote_price_arbitrage(c, allowed))
        filled = o.status == 0
        nf = o.merit[~filled]
        emit(set=name, nA=len(A), q=q, wall_ms=round(wall, 2), kernel_ms=round(ms, 3), launches=launches,
             fill_rate=round(float(np.mean(filled)), 5), iter_mean=round(float(np.mean(o.iterations)), 1),
             fev_mean=round(float(np.mean(o.fun_evals)), 1),
             merit_not_filled=[float(np.min(nf)), float(np.median(nf)), float(np.max(nf))] if len(nf) else None,
             tokens_mean=round(float(np.mean(np.diff(o.tok_off))), 1),
             pools_mean=round(float(np.mean(np.diff(o.leg_off))), 1),
             profit_mean_filled=float(np.mean(o.profit[filled])) if np.any(filled) else 0.0)
        est = ms * 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("hub", "headline"))
    ap.add_argument("--budget-s", type=float, default=60.0)
    args = ap.parse_args()
    emit(gpu=card())
    rng = np.random.default_rng(7)
    if args.only in (None, "headline"):
        m, n = 10_000_000, 50_000
        R, g, Ai = synth.product_pools(m, n, seed=1234)
        p = cr.DevicePools(n)
        p.add_product(R, g, Ai)
        p.finalize()
        for k in SIZES:
            run(p, "headline", n, bfs_tokens(Ai, n, k), np.ones(k), rng, args.budget_s)
        p.close()
    if args.only in (None, "hub"):
        p, n, _, nu, _ = hub_set(rng)
        for k in SIZES:
            A = np.arange(1, k + 1, dtype=np.int64)
            run(p, "hub", n, A, nu[A], rng, args.budget_s)
        p.close()


if __name__ == "__main__":
    main()
