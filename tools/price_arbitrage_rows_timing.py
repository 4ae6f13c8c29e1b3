"""Times cfmm_quote_price_arbitrage_rows (inventory rows) on one GPU; prints one JSON line per measurement.

  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).  L is |L| tokens reached
            breadth-first over the pools from token 1 (at |L| = 8 a star of 7 pools: a tree).
  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools, 20k sparse direct pools.  L is tokens 1..|L| (the hubs first).
|L| in {8, 64, 258}.  Every row lists L in its own random order with price_arbitrage_timing.py's prices
(the set's reference prices times exp(U(−0.02, 0.02)) per token and row).  Holdings (--held): none (0),
three random tokens per row (3), or every listed token (all), each held token holding HOLD_VALUE / c_t.
atol: 0 or --atol.  Otherwise default options.
Per call: the kernel time (CUDA events, option "profile": the plan and row kernels), the fill rate, the
mean iterations and evaluations, the m_r of the rows that did not fill (min, median, max), and the mean
tokens and pools per row.  Each configuration runs on 1k rows first; the 100k-row call runs when the
1k-row kernel time predicts at most --budget-s seconds for it, and is reported as not run (with the
estimate) otherwise.  The card's name and power limit are printed first.

    python tools/price_arbitrage_rows_timing.py [--only hub|headline] [--budget-s 20] [--atol 1e-3]
        [--held 0 3 all] [--sizes 8 64 258]
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
from price_arbitrage_timing import SIZES, bfs_tokens  # noqa: E402
from routed_order_timing import hub_set, timed  # noqa: E402
from split_order_timing import card  # noqa: E402
from subgraph_order_timing import emit  # noqa: E402

HOLD_VALUE = 100.0  # the value at c of each held token's holding
N_HELD = 3


def rows(L, base, q, held, rng):
    """(allow_off, allow_token, price, holding or None) of q rows over L, each in its own order; held
    tokens per row (0: no holding array)."""
    k = len(L)
    perm = np.argsort(rng.random((q, k)), axis=1)
    tok = L[perm]
    c = (base[perm] * np.exp(rng.uniform(-0.02, 0.02, size=(q, k))))
    off = np.arange(q + 1, dtype=np.int64) * k
    h = None
    if held:
        h = np.zeros((q, k))
        cols = np.argsort(rng.random((q, k)), axis=1)[:, :min(held, k)]
        r = np.arange(q)[:, None]
        h[r, cols] = HOLD_VALUE / c[r, cols]
        h = h.reshape(-1)
    return off, tok.reshape(-1), c.reshape(-1), h


def run(p, name, L, base, rng, budget_s, atol, helds):
    for held in (min(int(x), len(L)) if x != "all" else len(L) for x in helds):
        for a in (0.0, atol):
            est = None
            for q in (1_000, 100_000):
                cfg = dict(set=name, nL=len(L), held=held, atol=a, q=q)
                if q > 1_000 and est > budget_s * 1e3:
                    emit(**cfg, run=False, est_kernel_ms=round(est, 1))
                    continue
                off, tok, c, h = rows(L, base, q, held, rng)
                o, wall, ms, launches = timed(p, lambda: p.quote_price_arbitrage_rows(off, tok, c, h, {"atol": a}))
                filled = o.status == 0
                nf = o.merit[~filled]
                emit(**cfg, wall_ms=round(wall, 2), kernel_ms=round(ms, 3), launches=launches,
                     kernel_ms_per_100k=round(ms * 1e5 / q, 1), fill_rate=round(float(np.mean(filled)), 5),
                     iter_mean=round(float(np.mean(o.iterations)), 1), fev_mean=round(float(np.mean(o.fun_evals)), 1),
                     merit_not_filled=[float(np.min(nf)), float(np.median(nf)), float(np.max(nf))] if len(nf) else None,
                     tokens_mean=round(float(np.mean(np.diff(o.tok_off))), 1),
                     pools_mean=round(float(np.mean(np.diff(o.leg_off))), 1),
                     profit_mean_filled=float(np.mean(o.profit[filled])) if np.any(filled) else 0.0)
                est = ms * 100


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("hub", "headline"))
    ap.add_argument("--budget-s", type=float, default=20.0)
    ap.add_argument("--atol", type=float, default=1e-3)
    ap.add_argument("--held", nargs="+", default=["0", str(N_HELD)])
    ap.add_argument("--sizes", nargs="+", type=int, default=list(SIZES))
    args = ap.parse_args()
    emit(gpu=card())
    rng = np.random.default_rng(7)
    if args.only in (None, "headline"):
        m, n = 10_000_000, 50_000
        R, g, Ai = synth.product_pools(m, n, seed=1234)
        p = cr.DevicePools(n)
        p.add_product(R, g, Ai)
        p.finalize()
        for k in args.sizes:
            run(p, "headline", bfs_tokens(Ai, n, k), np.ones(k), rng, args.budget_s, args.atol, args.held)
        p.close()
    if args.only in (None, "hub"):
        p, n, _, nu, _ = hub_set(rng)
        for k in args.sizes:
            L = np.arange(1, k + 1, dtype=np.int64)
            run(p, "hub", L, nu[L], rng, args.budget_s, args.atol, args.held)
        p.close()


if __name__ == "__main__":
    main()
