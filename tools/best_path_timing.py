"""Times cfmm_find_order_paths on one GPU; prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
B is tokens 1..|B| (the hubs first on the hub set), |B| in {8, 64, 1024}, and max_hops H in {2, 3, 4}.
Rows sell one token outside B for another at 1e-3 of a pool's depth, exact-in and exact-out.  Per
find call: the wall time of the synchronous call (host clock), the kernel time (CUDA events, option
"profile", slot 4: the B-subgraph and path kernels), the filled / unreachable / repeated-pool rows and
the mean hops of the filled ones.  Each configuration runs on 1k rows first; the 100k-row call runs
when the 1k-row kernel time predicts at most --budget-s seconds for it, and is reported as not run
otherwise.  The card's name and power limit are read in the same run (nvidia-smi, read-only query).

    python tools/best_path_timing.py [--only hub|headline] [--budget-s 20]
"""
from __future__ import annotations

import argparse
import json
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


def emit(**kw):
    print(json.dumps(kw), flush=True)


def run(p, name, n, pick, amt_of, budget_s):
    tin, tout = pick(1, 8)  # the first call builds the pair index and the token adjacency
    p.find_order_paths(tin, tout, [0], amt_of(tin, tout, 0), 2, np.ones(n, bool) & (np.arange(n) < 8))
    for nb in (8, 64, 1024):
        allowed = np.zeros(n, bool)
        allowed[:nb] = True
        for H in (2, 3, 4):
            for kind in (0, 1):
                est = None
                for q in (1_000, 100_000):
                    if q > 1_000 and est > budget_s * 1e3:
                        emit(set=name, B=nb, H=H, kind=("in", "out")[kind], rows=q, run=False,
                             estimated_kernel_ms=round(est, 1))
                        continue
                    tin, tout = pick(q, nb)
                    k = np.full(q, kind, np.uint8)
                    out, wall, ms, launches = timed(p, lambda: p.find_order_paths(tin, tout, k, amt_of(tin, tout, kind),
                                                                                 H, allowed))
                    off, status = out[0], out[7]
                    hops = np.diff(off)
                    emit(set=name, B=nb, H=H, kind=("in", "out")[kind], rows=q, wall_ms=round(wall, 3),
                         kernel_ms=round(ms, 3), profile_entries=launches, filled=int(np.sum(status == 0)),
                         unreachable=int(np.sum(status == 2)), repeats_pool=int(np.sum(status == 4)),
                         hops_mean=round(float(np.mean(hops[status == 0])), 3) if np.any(status == 0) else 0.0)
                    est = ms * 100_000 / q


def hub(rng, budget_s):
    p, n, others, nu, _ = hub_set(rng)

    def pick(q, nb):
        out = others[others > nb]
        tin = rng.choice(out, size=q)
        tout = out[(np.searchsorted(out, tin) + rng.integers(1, len(out), size=q)) % len(out)]
        return tin.astype(np.int64), tout.astype(np.int64)

    run(p, "hub", n, pick, lambda tin, tout, kind: 1e-3 * 1e4 / nu[tout if kind else tin], budget_s)
    p.close()


def headline(rng, budget_s):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    emit(set="headline", pools=m, tokens=n)
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])

    def pick(q, nb):
        ok = np.flatnonzero((Ai[:, 0] > nb) & (Ai[:, 1] > nb))
        sel = rng.choice(ok, size=q)
        side = rng.integers(0, 2, size=q)
        return Ai[sel, side].astype(np.int64), Ai[sel, 1 - side].astype(np.int64)

    run(p, "headline", n, pick, lambda tin, tout, kind: 1e-3 * depth[tout if kind else tin], budget_s)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--budget-s", type=float, default=20.0)
    args = ap.parse_args()
    emit(card=card())
    rng = np.random.default_rng(2028)
    if args.only in (None, "hub"):
        hub(rng, args.budget_s)
    if args.only in (None, "headline"):
        headline(rng, args.budget_s)


if __name__ == "__main__":
    main()
