"""Times cfmm_choose_order_hubs on one GPU and compares auto-routed orders with named hubs and split
orders; prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
Rows sell one non-hub token for another at 1e-3 of a pool's depth (exact-in: of the tendered token;
exact-out: of the wanted one), 1k and 100k rows.  Per choose call (max_hubs 7): the wall time of the
synchronous call (host clock) and the kernel time (CUDA events, option "profile", slot 4); the first
call on each set also builds the pair index and the token adjacency, reported apart.  Then the same
rows are quoted with the auto hubs, with hubs 1..7 named by the caller, and as split orders over
their pair alone: per
variant the quote's wall and kernel time, the filled rows, and the total received (exact-in) or paid
(exact-out) over the rows every variant fills.  The card's name and power limit are read in the same
run (nvidia-smi, read-only query).

    python tools/hub_choice_timing.py [--only hub|headline]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402
from routed_order_timing import HUBS, hub_set, timed  # noqa: E402
from split_order_timing import card  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def run(p, name, tin, tout, kind, amt):
    q = len(tin)
    k = "in" if kind[0] == 0 else "out"
    (off, hubs, _, n_el), wall, ms, launches = timed(p, lambda: p.choose_order_hubs(tin, tout, kind, amt, 7))
    emit(set=name, call="choose", kind=k, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3), launches=launches,
         hubs_mean=round(float(np.mean(np.diff(off))), 2), eligible_mean=round(float(np.mean(n_el)), 2))
    named_off = np.arange(q + 1, dtype=np.int64) * len(HUBS)
    variants = {
        "auto": lambda: p.quote_routed_orders(tin, tout, kind, amt, off, hubs)[:4],
        "named 1..7": lambda: p.quote_routed_orders(tin, tout, kind, amt, named_off, np.tile(HUBS, q))[:4],
        "split": lambda: p.quote_split_orders(tin, tout, kind, amt),
    }
    res = {}
    for v, fn in variants.items():
        res[v] = timed(p, fn)
    every = np.logical_and.reduce([r[0][3] == 0 for r in res.values()])
    for v, (out, wall, ms, launches) in res.items():
        total = float(np.sum(out[1][every] if kind[0] == 0 else out[0][every]))
        emit(set=name, call=f"quote {v}", kind=k, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
             filled=int(np.sum(out[3] == 0)), common_rows=int(np.sum(every)),
             **{("received" if kind[0] == 0 else "paid"): total})


def rows_for(rng, q, pick_in, amt_in, amt_out):
    tin, tout = pick_in(q)
    return [(tin, tout, np.zeros(q, np.uint8), amt_in(tin)), (tin, tout, np.ones(q, np.uint8), amt_out(tout))]


def build_adjacency(p, name, tin, tout):
    """The first choose call after finalize builds the pair index and the adjacency: its extra time
    over a second call, and its extra profile entries."""
    one = lambda: p.choose_order_hubs(tin[:1], tout[:1], np.zeros(1, np.uint8), np.ones(1), 7)
    _, cold, _, l_cold = timed(p, one)
    _, warm, _, l_warm = timed(p, one)
    emit(set=name, call="pair index and adjacency build (first call less second)", wall_ms=round(cold - warm, 3),
         profile_entries=l_cold - l_warm)


def hub(rng):
    p, n, others, nu, _ = hub_set(rng)

    def pick(q):
        tin = rng.choice(others, size=q)
        tout = others[(np.searchsorted(others, tin) + rng.integers(1, len(others), size=q)) % len(others)]
        return tin.astype(np.int64), tout.astype(np.int64)

    build_adjacency(p, "hub", *pick(1))
    for q in (1_000, 100_000):
        for rows in rows_for(rng, q, pick, lambda t: 1e-3 * 1e4 / nu[t], lambda t: 1e-3 * 1e4 / nu[t]):
            run(p, "hub", *rows)
    p.close()


def headline(rng):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    emit(set="headline", pools=m, tokens=n)
    ok = np.flatnonzero((Ai[:, 0] > 7) & (Ai[:, 1] > 7))
    last = {}

    def pick(q):
        sel = rng.choice(ok, size=q)
        side = rng.integers(0, 2, size=q)
        last["sel"], last["side"] = sel, side
        return Ai[sel, side].astype(np.int64), Ai[sel, 1 - side].astype(np.int64)

    build_adjacency(p, "headline", *pick(1))
    for q in (1_000, 100_000):
        for rows in rows_for(rng, q, pick, lambda t: 1e-3 * R[last["sel"], last["side"]],
                             lambda t: 1e-3 * R[last["sel"], 1 - last["side"]]):
            run(p, "headline", *rows)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    args = ap.parse_args()
    emit(card=card())
    rng = np.random.default_rng(2027)
    if args.only in (None, "hub"):
        hub(rng)
    if args.only in (None, "headline"):
        headline(rng)


if __name__ == "__main__":
    main()
