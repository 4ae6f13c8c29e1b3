"""Times cfmm_quote_subgraph_orders on one GPU; prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
B is tokens 1..|B| (the hubs first on the hub set), |B| in {8, 64, 256}.  Rows sell one token outside
B for another at 1e-3 of a pool's depth (exact-in), default options.  Per quote call: the wall time
of the synchronous call (host clock), the kernel time (CUDA events, option "profile", slot 4: the
B-subgraph, plan and solve kernels), the filled / unreachable / not-converged rows, the mean and
largest iterations and evaluations of the solved rows, the largest m_r of the filled rows and the
smallest of the not-converged ones (the floor the default rtol meets or misses), and the mean pools
per row.  The same rows are then quoted as auto-routed orders (cfmm_choose_order_hubs with the mask,
then cfmm_quote_routed_orders) and as best paths (cfmm_find_order_paths, H = 4): the fraction of rows
where the subgraph's received is at least theirs (within 3·rtol) and the median ratio.  Each
configuration runs on 1k rows first; the 100k-row call runs when the 1k-row kernel time predicts at
most --budget-s seconds for it, and is reported as not run (with the estimate) otherwise.

    python tools/subgraph_order_timing.py [--only hub|headline] [--budget-s 20]
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


def stats(o):
    solved = o.solver_status >= 0
    filled = o.status == 0
    nc = o.status == cr._lib.ORDER_NOT_CONVERGED
    pools = np.diff(o.leg_off)
    return dict(filled=int(np.sum(filled)), unreachable=int(np.sum(o.status == 2)), not_converged=int(np.sum(nc)),
                iter_mean=round(float(np.mean(o.iterations[solved])), 1) if np.any(solved) else 0.0,
                iter_max=int(np.max(o.iterations[solved])) if np.any(solved) else 0,
                fev_mean=round(float(np.mean(o.fun_evals[solved])), 1) if np.any(solved) else 0.0,
                fev_max=int(np.max(o.fun_evals[solved])) if np.any(solved) else 0,
                merit_filled_max=float(np.max(o.merit[filled & solved])) if np.any(filled & solved) else 0.0,
                merit_nc_min=float(np.min(o.merit[nc])) if np.any(nc) else None,
                pools_mean=round(float(np.mean(pools)), 1))


def compare(p, tin, tout, amt, allowed, o):
    q = len(tin)
    kind = np.zeros(q, np.uint8)
    off, flat, _, _ = p.choose_order_hubs(tin, tout, kind, amt, 7, allowed)
    _, recv_r, _, st_r = p.quote_routed_orders(tin, tout, kind, amt, off, flat)[:4]
    value, st_p = p.find_order_paths(tin, tout, kind, amt, 4, allowed)[6:]
    out = {}
    for name, recv, st in (("auto_routed", recv_r, st_r), ("best_path", value, st_p)):
        both = (o.status == 0) & (st == 0) & (recv > 0)
        if np.any(both):
            ratio = o.received[both] / recv[both]
            out[name] = dict(rows=int(np.sum(both)), at_least=float(np.mean(ratio >= 1 - 3e-4)),
                             median_ratio=round(float(np.median(ratio)), 6))
    return out


def run(p, name, n, pick, amt_of, budget_s):
    tin, tout = pick(1, 8)  # the first call builds the pair index and the token adjacency
    p.quote_subgraph_orders(tin, tout, amt_of(tin, tout), np.arange(n) < 8)
    for nb in (8, 64, 256):
        allowed = np.arange(n) < nb
        est = None
        for q in (1_000, 100_000):
            if q > 1_000 and est > budget_s * 1e3:
                emit(set=name, B=nb, rows=q, run=False, estimated_kernel_ms=round(est, 1))
                continue
            tin, tout = pick(q, nb)
            amt = amt_of(tin, tout)
            o, wall, ms, launches = timed(p, lambda: p._subgraph(False, tin, tout, amt, allowed, None, None))
            rec = dict(set=name, B=nb, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                       profile_entries=launches, **stats(o))
            if q == 1_000:
                rec.update(compare(p, tin, tout, amt, allowed, o))
            emit(**rec)
            est = ms * 100_000 / q


def hub(rng, budget_s):
    p, n, others, nu, _ = hub_set(rng)

    def pick(q, nb):
        out = others[others > nb]
        tin = rng.choice(out, size=q)
        tout = out[(np.searchsorted(out, tin) + rng.integers(1, len(out), size=q)) % len(out)]
        return tin.astype(np.int64), tout.astype(np.int64)

    run(p, "hub", n, pick, lambda tin, tout: 1e-3 * 1e4 / nu[tin], budget_s)
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

    run(p, "headline", n, pick, lambda tin, tout: 1e-3 * depth[tin], budget_s)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--budget-s", type=float, default=20.0)
    args = ap.parse_args()
    emit(card=card())
    rng = np.random.default_rng(2029)
    if args.only in (None, "hub"):
        hub(rng, args.budget_s)
    if args.only in (None, "headline"):
        headline(rng, args.budget_s)


if __name__ == "__main__":
    main()
