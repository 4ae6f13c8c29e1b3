"""Times cfmm_quote_limit_orders on one GPU; prints one JSON line per measurement.

The sets, rows and B are basket_order_timing.py's (hub: 2k tokens, hubs 1..7 paired with every other
token by three pools plus 20k sparse pools; headline: 10M ProductTwoCoin pools over 50k tokens), with
|B| in {0, 8, 64} and K in {1, 4, 16}, each entry at 1e-3 of a pool's depth.  Each entry's limit is
drawn around its best single-pool rate in the output token: ν_k/ν_i of a one-entry row over the
pair's own pools (an empty mask) at a thousandth of the entry's amount, times 0.98, 1.0 or 1.02 at
random, so rows fill fully, partially or not at all (an entry whose pair holds no pool gets limit 0,
counted as zero_limit_entries).
Per quote call: the wall time of the synchronous call (host clock) and the kernel time (CUDA events,
option "profile", slot 4), the rows filled fully (every entry within 1e-3 of its amount), partially,
not at all (every entry below 1e-3 of it), unreachable and not converged, and basket_order_timing's
iteration, evaluation and m_r figures.  Then the same rows quoted as basket rows at zero limits
(cfmm_quote_basket_orders): the cost of the limits.  Each configuration runs on 1k rows first; the
100k-row call runs when the 1k-row kernel time predicts at most --budget-s seconds for it.

    python tools/limit_order_timing.py [--only hub|headline] [--budget-s 20]
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
from basket_order_timing import hub_pairs, make_rows, neighbours  # noqa: E402
from routed_order_timing import hub_set, timed  # noqa: E402
from split_order_timing import card  # noqa: E402
from subgraph_order_timing import emit, stats  # noqa: E402

KS = (1, 4, 16)


def limits(p, tout, boff, btok, bamt, n, rng):
    """Each entry's best single-pool rate in its row's output token times 0.98, 1.0 or 1.02: ν_k/ν_i of
    a one-entry row (i, k) over the pair's own pools (an empty mask) at a thousandth of the entry's
    amount.  0 where the pair holds no pool or that quote did not converge."""
    tin = np.repeat(tout, np.diff(boff))
    tiny = p.quote_basket_orders(tin, np.arange(len(btok) + 1, dtype=np.int64), btok, bamt * 1e-3,
                                 np.zeros(n, bool))
    ok = (tiny.status == 0) & (tiny.solver_status == 0) & (np.diff(tiny.tok_off) == 2)
    t0 = tiny.tok_off[:-1]
    c = np.where(ok, tiny.nu[np.minimum(t0 + 1, len(tiny.nu) - 1)] / tiny.nu[t0], 0.0)
    return c * rng.choice([0.98, 1.0, 1.02], size=len(c))


def fills(o, boff, bamt):
    """Rows filled fully, partially and not at all (filled rows only; every entry within 1e-3 of its
    amount, or every entry below 1e-3 of it)."""
    full = part = none = 0
    for r in np.flatnonzero(o.status == 0):
        a, pd = bamt[boff[r]:boff[r + 1]], o.paid[boff[r]:boff[r + 1]]
        if np.all(pd >= a * (1 - 1e-3)):
            full += 1
        elif np.all(pd <= a * 1e-3):
            none += 1
        else:
            part += 1
    return dict(full=full, partial=part, none=none)


def run(p, name, n, tokens, csr, amt_of, budget_s, rng):
    allowed8 = np.arange(n) < 8
    p.quote_basket_orders([2], [0, 1], [1], [1.0], allowed8)  # builds the pair index and the adjacency
    for nb in (0, 8, 64):
        allowed = np.arange(n) < nb
        for K in KS:
            est = None
            for q in (1_000, 100_000):
                if q > 1_000 and est > budget_s * 1e3:
                    emit(set=name, B=nb, K=K, rows=q, run=False, estimated_kernel_ms=round(est, 1))
                    continue
                tout, boff, btok, bamt = make_rows(rng, q, (K,), nb, tokens, csr, amt_of)
                c = limits(p, tout, boff, btok, bamt, n, rng)
                o, wall, ms, launches = timed(
                    p, lambda: p._limit(False, tout, boff, btok, bamt, c, allowed, None, None))
                emit(set=name, B=nb, K=K, rows=q, mode="limit", wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                     profile_entries=launches, tokens_mean=round(float(np.mean(np.diff(o.tok_off))), 1),
                     zero_limit_entries=int(np.sum(c == 0.0)), **fills(o, boff, bamt), **stats(o))
                b, wall_b, ms_b, _ = timed(
                    p, lambda: p._basket(False, tout, boff, btok, bamt, allowed, None, None))
                emit(set=name, B=nb, K=K, rows=q, mode="basket_zero_limits", wall_ms=round(wall_b, 3),
                     kernel_ms=round(ms_b, 3), **stats(b))
                est = ms * 100_000 / q


def hub(budget_s):
    p, n, others, nu, _ = hub_set(np.random.default_rng(7))
    Ai = hub_pairs(np.random.default_rng(7))
    csr = neighbours(Ai, n)
    amt_of = lambda t: 1e-3 * 1e4 / nu[t]  # noqa: E731
    run(p, "hub", n, others, csr, amt_of, budget_s, np.random.default_rng(2040))
    p.close()


def headline(budget_s):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    emit(set="headline", pools=m, tokens=n)
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])
    csr = neighbours(Ai, n)
    amt_of = lambda t: 1e-3 * depth[t]  # noqa: E731
    run(p, "headline", n, np.arange(1, n + 1), csr, amt_of, budget_s, np.random.default_rng(2041))
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--budget-s", type=float, default=20.0)
    args = ap.parse_args()
    emit(card=card())
    if args.only in (None, "hub"):
        hub(args.budget_s)
    if args.only in (None, "headline"):
        headline(args.budget_s)


if __name__ == "__main__":
    main()
