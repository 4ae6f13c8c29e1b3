"""Times cfmm_quote_basket_orders on one GPU; prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
B is tokens 1..|B| (the hubs first on the hub set), |B| in {0, 8, 64}.  A row sells K in {1, 2, 4, 8,
16} tokens for an output token outside B: the basket is K of the output token's pool neighbours outside
B (topped up with random tokens when it has fewer), each at 1e-3 of a pool's depth, default options.
Per quote call: the wall time of the synchronous call (host clock), the kernel time (CUDA events,
option "profile", slot 4: the B-subgraph, plan and solve kernels), the filled / unreachable /
not-converged rows, the mean and largest iterations and evaluations of the solved rows, the largest
m_r of the filled rows and the smallest of the not-converged ones, and the mean tokens and pools per
row.  Each configuration runs on 1k rows first; the 100k-row call runs when the 1k-row kernel time
predicts at most --budget-s seconds for it, and is reported as not run (with the estimate) otherwise.

Then, on two copies of the state, up to 1k rows with K cycling through 2, 4, 8, 16, |B| = 0 and
pairwise disjoint token sets (so every basket and its sequence start from the same pool state) run
as one cfmm_execute_basket_orders on one copy, and as their entries sold one by one (K rows of
cfmm_execute_subgraph_orders per basket, in the same order) on the other: per K, the fraction of rows
where the basket receives at least the sequence's total (within 3·rtol) and the median ratio.

With --buy KS,KB the tool times buy rows instead (cfmm_quote_basket_swap_orders): each row sells KS
and buys KB tokens around its output token (chosen as above, every amount at 1e-3 of a pool's depth),
|B| in {0, 8, 64}, 1k rows and then 100k under the same budget rule.  Per call it reports what the
sell-only rows report, and then the same rows quoted the way a caller would have to without buy rows:
the KS sold tokens as one cfmm_quote_basket_orders row and each bought token as one exact-out
cfmm_quote_subgraph_swap_orders row paying in the output token (their kernel times summed, and each
call's fill, iteration and m_r figures).  Buy rows also report their not-converged rows by solver
status (0: converged short of a bought y, 1: stalled, 2 / 3: max_iter / max_fun) and the median m_r
those rows reached.

    python tools/basket_order_timing.py [--only hub|headline] [--budget-s 20] [--buy KS,KB]
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
from subgraph_order_timing import emit, stats  # noqa: E402

KS = (1, 2, 4, 8, 16)


def neighbours(Ai, n):
    """CSR of each token's pool neighbours (with repeats): (off [n + 2], nbr)."""
    a = np.concatenate([Ai[:, 0], Ai[:, 1]])
    b = np.concatenate([Ai[:, 1], Ai[:, 0]])
    o = np.argsort(a, kind="stable")
    off = np.zeros(n + 2, np.int64)
    np.add.at(off, a + 1, 1)
    return np.cumsum(off), b[o]


def make_rows(rng, q, Ks, nb, tokens, csr, amt_of):
    """q rows (token_out, basket_off, basket_token, basket_amount), row r with Ks[r % len(Ks)] entries."""
    off, nbr = csr
    tout = rng.choice(tokens[tokens > nb], size=q).astype(np.int64)
    boff, btok = [0], []
    for r in range(q):
        K, i = Ks[r % len(Ks)], int(tout[r])
        cand = np.unique(nbr[off[i]:off[i + 1]])
        cand = cand[(cand > nb) & (cand != i)]
        pick = rng.choice(cand, size=min(K, len(cand)), replace=False).tolist()
        while len(pick) < K:
            t = int(rng.choice(tokens))
            if t > nb and t != i and t not in pick:
                pick.append(t)
        btok += pick
        boff.append(len(btok))
    btok = np.array(btok, np.int64)
    return tout, np.array(boff, np.int64), btok, amt_of(btok)


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
                o, wall, ms, launches = timed(
                    p, lambda: p._basket(False, tout, boff, btok, bamt, allowed, None, None))
                emit(set=name, B=nb, K=K, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                     profile_entries=launches, tokens_mean=round(float(np.mean(np.diff(o.tok_off))), 1), **stats(o))
                est = ms * 100_000 / q


def run_buy(p, name, n, tokens, csr, amt_of, budget_s, rng, ks, kb):
    """Buy rows of ks sold and kb bought entries, then the same rows as a sell-only basket plus kb
    exact-out rows."""
    allowed8 = np.arange(n) < 8
    p.quote_basket_orders([2], [0, 1], [1], [1.0], allowed8)  # builds the pair index and the adjacency
    for nb in (0, 8, 64):
        allowed = np.arange(n) < nb
        est = None
        for q in (1_000, 100_000):
            if q > 1_000 and est > budget_s * 1e3:
                emit(set=name, B=nb, K_sell=ks, K_buy=kb, rows=q, run=False, estimated_kernel_ms=round(est, 1))
                continue
            tout, boff, btok, bamt = make_rows(rng, q, (ks + kb,), nb, tokens, csr, amt_of)
            kind = np.tile(np.r_[np.zeros(ks), np.full(kb, cr._lib.SWAP_EXACT_OUT)].astype(np.uint8), q)
            o, wall, ms, launches = timed(
                p, lambda: p._basket(False, tout, boff, btok, bamt, allowed, None, None, kind))
            nc = o.status == cr._lib.ORDER_NOT_CONVERGED
            by = {str(v): int(np.sum(o.solver_status[nc] == v)) for v in np.unique(o.solver_status[nc])}
            emit(set=name, B=nb, K_sell=ks, K_buy=kb, rows=q, mode="buy_rows", wall_ms=round(wall, 3),
                 kernel_ms=round(ms, 3), profile_entries=launches,
                 tokens_mean=round(float(np.mean(np.diff(o.tok_off))), 1), not_converged_by_solver_status=by,
                 merit_nc_median=float(np.median(o.merit[nc])) if np.any(nc) else None, **stats(o))
            sold = kind == 0
            split, split_ms = {}, 0.0
            if ks:
                s_off = np.arange(0, q * ks + 1, ks, dtype=np.int64)
                os_, _, ms_s, _ = timed(
                    p, lambda: p._basket(False, tout, s_off, btok[sold], bamt[sold], allowed, None, None))
                split["basket"], split_ms = stats(os_), split_ms + ms_s
            ob, _, ms_b, _ = timed(
                p, lambda: p._subgraph(False, np.repeat(tout, kb), btok[~sold], bamt[~sold], allowed, None, None,
                                       cr._lib.SWAP_EXACT_OUT))
            split["exact_out"], split_ms = stats(ob), split_ms + ms_b
            emit(set=name, B=nb, K_sell=ks, K_buy=kb, rows=q, mode="basket_plus_exact_out",
                 kernel_ms=round(split_ms, 3), **split)
            est = ms * 100_000 / q


def disjoint_rows(rng, q, Ks, tokens, csr, amt_of):
    """Up to q rows as make_rows with |B| = 0 whose token sets {i} ∪ basket are pairwise disjoint."""
    off, nbr = csr
    used = set()
    tout, boff, btok = [], [0], []
    for t in rng.permutation(tokens):
        K, i = Ks[len(tout) % len(Ks)], int(t)
        if len(tout) == q or i in used:
            continue
        cand = [int(c) for c in np.unique(nbr[off[i]:off[i + 1]]) if c != i and int(c) not in used]
        if len(cand) < K:
            continue
        pick = rng.choice(cand, size=K, replace=False).tolist()
        used.update(pick + [i])
        tout.append(i)
        btok += pick
        boff.append(len(btok))
    btok = np.array(btok, np.int64)
    return np.array(tout, np.int64), np.array(boff, np.int64), btok, amt_of(btok)


def compare(a, b, name, n, tokens, csr, amt_of, rng):
    """Baskets executed on a against their entries sold one by one on b (a and b hold the same state).
    The rows' token sets are disjoint and B is empty, so no row trades a pool another row trades: each
    basket and its sequence start from the same pool state."""
    Ks = (2, 4, 8, 16)
    none = np.zeros(n, bool)
    tout, boff, btok, bamt = disjoint_rows(rng, 1_000, Ks, tokens, csr, amt_of)
    o = a.execute_basket_orders(tout, boff, btok, bamt, none)
    s = b.execute_subgraph_orders(btok, np.repeat(tout, np.diff(boff)), bamt, none)
    row = np.repeat(np.arange(len(tout)), np.diff(boff))
    seq = np.bincount(row, weights=s.received, minlength=len(tout))
    seq_ok = np.bincount(row, weights=(s.status != 0).astype(float), minlength=len(tout)) == 0
    for K in Ks:
        sel = (np.diff(boff) == K) & (o.status == 0) & seq_ok & (seq > 0)
        if np.any(sel):
            ratio = o.received[sel] / seq[sel]
            emit(set=name, B=0, K=K, compare="sequential_subgraph", rows=int(np.sum(sel)),
                 rows_of_k=int(np.sum(np.diff(boff) == K)), at_least=float(np.mean(ratio >= 1 - 3e-4)),
                 median_ratio=round(float(np.median(ratio)), 6), min_ratio=round(float(np.min(ratio)), 6))


def hub(budget_s, buy=None):
    p, n, others, nu, pools_of = hub_set(np.random.default_rng(7))
    Ai = hub_pairs(np.random.default_rng(7))
    assert all(len(pools_of(int(a), int(b))) for a, b in Ai[-5:]), "hub_pairs no longer replays hub_set"
    csr = neighbours(Ai, n)
    amt_of = lambda t: 1e-3 * 1e4 / nu[t]  # noqa: E731
    rng = np.random.default_rng(2030)
    if buy:
        run_buy(p, "hub", n, others, csr, amt_of, budget_s, rng, *buy)
        p.close()
        return
    run(p, "hub", n, others, csr, amt_of, budget_s, rng)
    q, _, _, _, _ = hub_set(np.random.default_rng(7))
    compare(p, q, "hub", n, others, csr, amt_of, rng)
    p.close()
    q.close()


def hub_pairs(rng):
    """The hub set's pool token pairs: hub_set's draws replayed from an rng in the same state (the
    context does not hand its pools' tokens back)."""
    from routed_order_timing import HUBS
    n, md = 2_000, 20_000
    rng.uniform(-1, 1, size=n + 1)
    others = np.arange(8, n + 1)
    A = np.array([(h, x) for h in HUBS for x in others], dtype=np.int64)
    m = len(A)
    rng.uniform(1e3, 1e5, size=m)
    rng.uniform(-0.02, 0.02, size=(m, 2))
    rng.choice([0.997, 0.9995], size=m)
    rng.uniform(-0.02, 0.02, size=(m, 2))
    rng.uniform(0.3, 0.7, size=(m, 2))
    rng.uniform(-0.02, 0.02, size=m)
    D = np.array([rng.choice(others, size=2, replace=False) for _ in range(md)], dtype=np.int64)
    return np.concatenate([A, D])


def headline(budget_s, buy=None):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)

    def ctx():
        p = cr.DevicePools(n)
        p.add_product(R, g, Ai)
        p.finalize()
        return p

    p = ctx()
    emit(set="headline", pools=m, tokens=n)
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])
    csr = neighbours(Ai, n)
    amt_of = lambda t: 1e-3 * depth[t]  # noqa: E731
    rng = np.random.default_rng(2031)
    tokens = np.arange(1, n + 1)
    if buy:
        run_buy(p, "headline", n, tokens, csr, amt_of, budget_s, rng, *buy)
        p.close()
        return
    run(p, "headline", n, tokens, csr, amt_of, budget_s, rng)
    q = ctx()
    compare(p, q, "headline", n, tokens, csr, amt_of, rng)
    p.close()
    q.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--budget-s", type=float, default=20.0)
    ap.add_argument("--buy", help="KS,KB: time buy rows selling KS and buying KB tokens")
    args = ap.parse_args()
    buy = None
    if args.buy:
        buy = tuple(int(x) for x in args.buy.split(","))
        if len(buy) != 2 or buy[1] < 1 or buy[0] < 0 or sum(buy) > 16:
            ap.error("--buy needs KS,KB with KS >= 0, KB >= 1 and KS + KB <= 16")
    emit(card=card())
    if args.only in (None, "hub"):
        hub(args.budget_s, buy)
    if args.only in (None, "headline"):
        headline(args.budget_s, buy)


if __name__ == "__main__":
    main()
