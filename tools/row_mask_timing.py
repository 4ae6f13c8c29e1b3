"""Times the per-row mask calls (cfmm_*_rows) on one GPU; prints one JSON line per measurement.

The sets are subgraph_order_timing.py's: hub (2k tokens, hubs 1..7 paired with every other token by
three pools, plus 20k sparse pools) and headline (10M ProductTwoCoin pools over 50k tokens).  The
first line is the card's name and power limit.

  quote    the same exact-in rows with one mask B = tokens 1..|B|, |B| in {8, 64, 256}, quoted through
           cfmm_quote_subgraph_swap_orders and through cfmm_quote_subgraph_swap_orders_rows with every
           row given B: wall time (host clock around the synchronous call) and kernel time (CUDA events,
           option "profile", slot 4) of each, and whether every output is the same bit for bit.  --rows
           rows (1k for |B| = 256).
  execute  headline set, --exec-rows orders, each with its own hubs (cfmm_choose_order_hubs, at most 7,
           no mask): the execute's levels and row-kernel launches, wall and kernel time, executed
           through the _rows call; then the same orders on a second copy of the set through the one-mask
           call with the union of their hubs (its 256 most chosen tokens when the union is larger).
  fill     headline set, --rows orders: the filled rows with each order's own hubs against one shared
           mask of the union's 256 most chosen hubs and against tokens 1..8.

    python tools/row_mask_timing.py [--only quote|execute|fill] [--rows 10000] [--exec-rows 2000]
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
from subgraph_order_timing import emit, stats  # noqa: E402

FIELDS = ("paid", "received", "status", "solver_status", "iterations", "fun_evals", "merit", "tok_off", "token",
          "nu", "psi", "leg_off", "leg_type", "leg_pool", "leg_delta", "leg_lambda")


def same(a, b):
    return all(np.array_equal(getattr(a, f), getattr(b, f)) for f in FIELDS)


def levels(own):
    """The execute's level of each row: 1 + the largest level of an earlier row sharing a token."""
    last, lev = {}, []
    for s in own:
        L = 1 + max((last.get(t, 0) for t in s), default=0)
        for t in s:
            last[t] = L
        lev.append(L)
    return lev


def headline_set(seed=1234):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=seed)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])
    return p, n, Ai, depth


def headline_rows(rng, Ai, depth, q, nb):
    ok = np.flatnonzero((Ai[:, 0] > nb) & (Ai[:, 1] > nb))
    sel = rng.choice(ok, size=q)
    side = rng.integers(0, 2, size=q)
    tin, tout = Ai[sel, side].astype(np.int64), Ai[sel, 1 - side].astype(np.int64)
    return tin, tout, 1e-3 * depth[tin]


def quote(p, name, n, pick, q):
    tin, tout, amt = pick(8, 8)
    p.quote_subgraph_orders(tin, tout, amt, np.arange(n) < 8)  # builds the pair index and the adjacency
    for nb in (8, 64, 256):
        rows = q if nb < 256 else min(q, 1_000)
        tin, tout, amt = pick(rows, nb)
        allowed = np.arange(n) < nb
        lists = [np.arange(1, nb + 1, dtype=np.int64)] * rows
        a, wa, ka, _ = timed(p, lambda: p.quote_subgraph_orders(tin, tout, amt, allowed))
        b, wb, kb, _ = timed(p, lambda: p.quote_subgraph_orders(tin, tout, amt, lists))
        emit(part="quote", set=name, B=nb, rows=rows, mask_wall_ms=round(wa, 3), mask_kernel_ms=round(ka, 3),
             rows_wall_ms=round(wb, 3), rows_kernel_ms=round(kb, 3), same_bits=same(a, b), **stats(a))


def chosen(p, tin, tout, amt):
    off, flat, _, _ = p.choose_order_hubs(tin, tout, np.zeros(len(tin), np.uint8), amt, 7)
    hubs = [flat[off[r]:off[r + 1]] for r in range(len(tin))]
    uniq, cnt = np.unique(flat, return_counts=True)
    top = uniq[np.argsort(-cnt, kind="stable")[:256]]
    return hubs, uniq, top


def execute(rng, q):
    p, n, Ai, depth = headline_set()
    tin, tout, amt = headline_rows(rng, Ai, depth, q, 0)
    hubs, uniq, top = chosen(p, tin, tout, amt)
    lev = levels([{int(a), int(b)} | set(h.tolist()) for a, b, h in zip(tin, tout, hubs)])
    o, wall, ms, launches = timed(p, lambda: p.execute_subgraph_orders(tin, tout, amt, hubs))
    emit(part="execute", call="rows", rows=q, levels=int(max(lev)), hubs_mean=round(float(np.mean([len(h) for h in hubs])), 2),
         wall_ms=round(wall, 3), kernel_ms=round(ms, 3), profile_entries=launches, **stats(o))
    p.close()
    p, n, Ai, depth = headline_set()
    allowed = np.zeros(n, bool)
    allowed[top - 1] = True
    o, wall, ms, launches = timed(p, lambda: p.execute_subgraph_orders(tin, tout, amt, allowed))
    lev = levels([{int(a), int(b)} | set(top.tolist()) for a, b in zip(tin, tout)])
    emit(part="execute", call="one_mask", rows=q, levels=int(max(lev)), union=int(len(uniq)), mask=int(len(top)),
         wall_ms=round(wall, 3), kernel_ms=round(ms, 3), profile_entries=launches, **stats(o))
    p.close()


def fill(rng, q):
    p, n, Ai, depth = headline_set()
    tin, tout, amt = headline_rows(rng, Ai, depth, q, 8)
    hubs, uniq, top = chosen(p, tin, tout, amt)
    union = np.zeros(n, bool)
    union[top - 1] = True
    for name, allowed in (("own_hubs", hubs), ("union_top256", union), ("tokens_1_8", np.arange(n) < 8)):
        o, wall, ms, _ = timed(p, lambda: p.quote_subgraph_orders(tin, tout, amt, allowed))
        emit(part="fill", mask=name, rows=q, union=int(len(uniq)), wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
             **stats(o))
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["quote", "execute", "fill"])
    ap.add_argument("--rows", type=int, default=10_000)
    ap.add_argument("--exec-rows", type=int, default=2_000)
    args = ap.parse_args()
    emit(card=card())
    rng = np.random.default_rng(2031)
    if args.only in (None, "quote"):
        p, n, others, nu, _ = hub_set(rng)

        def pick_hub(q, nb):
            out = others[others > nb]
            tin = rng.choice(out, size=q)
            tout = out[(np.searchsorted(out, tin) + rng.integers(1, len(out), size=q)) % len(out)]
            return tin.astype(np.int64), tout.astype(np.int64), 1e-3 * 1e4 / nu[tin]

        quote(p, "hub", n, pick_hub, args.rows)
        p.close()
        p, n, Ai, depth = headline_set()
        quote(p, "headline", n, lambda q, nb: headline_rows(rng, Ai, depth, q, nb), args.rows)
        p.close()
    if args.only in (None, "execute"):
        execute(rng, args.exec_rows)
    if args.only in (None, "fill"):
        fill(rng, args.rows)


if __name__ == "__main__":
    main()
