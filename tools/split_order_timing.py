"""Times cfmm_pair_pools / cfmm_quote_split_orders / cfmm_execute_split_orders on one GPU and prints
one JSON line per measurement.

  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set): almost every pair holds
            one pool, so this is the per-row floor.  Quote and execute 1k and 1M rows.
  hub       1M ProductTwoCoin and 100k UniV3 pools (4 ticks) over 1k token pairs of 2k tokens:
            about 1100 pools per pair.  Quote and execute 10k rows, exact-in and exact-out.

For each: the wall time of the synchronous call (host clock) and the kernel time (CUDA events, option
"profile", slot 4: the pair lookup and the split kernel), and the evaluations of the pair's pools
per row, counted by the host mirror (tests/split_oracle.py, which takes the device's steps) on a
sample of the rows.  The pair index is built by the first call after finalize: its one-off cost is
that call's wall time less the same call's second time.  Exact-in rows tender 1e-4 of a pool's
reserve on the tendered side (UniV3 pools in the hub set are priced near 1); exact-out rows want what
the exact-in quote of the same row received.  The card's name and power limit are read in the same
run (nvidia-smi, read-only query).

    python tools/split_order_timing.py [--only headline|hub] [--sample 8]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402

SLOT = 4  # cfmm_profile_read: the swap kernels' slot


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # (no nvidia-smi: the number still stands, without its label)
        return f"unknown ({e})"


def timed(p, fn):
    p.set_option("profile", 64)
    p.profile_reset()
    t0 = time.perf_counter()
    out = fn()
    wall = time.perf_counter() - t0
    ms, launches = p.profile_read(SLOT)
    return out, wall * 1e3, ms, launches


def mirror_evals(objs_of_row, rows, kind, amount, tin, tout):
    import split_oracle as so
    ev = [so.split_row(objs_of_row(r), tin[r], tout[r], kind[r], amount[r])["evals"] for r in rows]
    return float(np.mean(ev)), int(np.max(ev))


def run(p, name, tin, tout, amt, objs_of_row, sample, rng, kinds=(0,)):
    q = len(tin)
    for kind in kinds:
        k = np.full(q, kind, np.uint8)
        a = amt
        if kind == 1:  # want what the exact-in quote receives
            a = p.quote_split_orders(tin, tout, np.zeros(q, np.uint8), amt)[1]
            a = np.where(a > 0, a, amt)
        (paid, got, price, st), wall, ms, launches = timed(p, lambda: p.quote_split_orders(tin, tout, k, a))
        rows = rng.choice(q, size=min(sample, q), replace=False)
        mean_ev, max_ev = mirror_evals(objs_of_row, rows, k, a, tin, tout)
        print(json.dumps(dict(set=name, call="quote", kind=int(kind), rows=q, wall_ms=round(wall, 3),
                              kernel_ms=round(ms, 3), launches=launches, filled=int(np.sum(st == 0)),
                              evals_per_row_mean=round(mean_ev, 1), evals_per_row_max=max_ev)), flush=True)
        (_, _, _, st), wall, ms, launches = timed(p, lambda: p.execute_split_orders(tin, tout, k, a))
        print(json.dumps(dict(set=name, call="execute", kind=int(kind), rows=q, wall_ms=round(wall, 3),
                              kernel_ms=round(ms, 3), launches=launches, filled=int(np.sum(st == 0)))), flush=True)


def headline(args, rng):
    import split_oracle as so
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    t0 = time.perf_counter()
    p.pair_pools([int(Ai[0, 0])], [int(Ai[0, 1])])
    first = time.perf_counter() - t0
    t0 = time.perf_counter()
    p.pair_pools([int(Ai[0, 0])], [int(Ai[0, 1])])
    second = time.perf_counter() - t0
    print(json.dumps(dict(set="headline", call="pair_index_build", pools=m, ms=round((first - second) * 1e3, 3))),
          flush=True)
    for q in (1_000, 1_000_000):
        pick = rng.integers(0, m, size=q)
        side = rng.integers(0, 2, size=q)
        tin, tout = Ai[pick, side], Ai[pick, 1 - side]
        amt = 1e-4 * R[pick, side]

        def objs(r, tin=tin, tout=tout):
            _, _, idx, _ = p.pair_pools([tin[r]], [tout[r]])
            return [so.Product(R[i], g[i], Ai[i]) for i in idx]
        run(p, "headline", tin, tout, amt, objs, args.sample, rng, kinds=(0, 1))
    p.close()


def hub(args, rng):
    import split_oracle as so
    n, n_pairs, mp, mu = 2_000, 1_000, 1_000_000, 100_000
    pairs = synth.token_pairs(rng, n_pairs, n)
    price = np.exp(rng.uniform(-0.05, 0.05, size=n_pairs))  # token a in units of b, per pair
    R, g, _ = synth.product_pools(mp, n, seed=5)
    pp = rng.integers(0, n_pairs, size=mp)
    Ap = pairs[pp]
    R[:, 1] = R[:, 0] * price[pp] * np.exp(rng.uniform(-0.01, 0.01, size=mp))
    cp, gu, _, off, lt, lq = synth.univ3_pools(mu, n, seed=6)
    pu = rng.integers(0, n_pairs, size=mu)
    Au = pairs[pu]
    scale = price[pu] / cp
    cp = cp * scale
    lt = lt * np.repeat(scale, np.diff(off))
    p = cr.DevicePools(n)
    p.add_product(R, g, Ap)
    p.add_univ3(cp, gu, Au, off, lt, lq)
    p.finalize()
    t0 = time.perf_counter()
    p.pair_pools([int(pairs[0, 0])], [int(pairs[0, 1])])
    first = time.perf_counter() - t0
    t0 = time.perf_counter()
    p.pair_pools([int(pairs[0, 0])], [int(pairs[0, 1])])
    second = time.perf_counter() - t0
    print(json.dumps(dict(set="hub", call="pair_index_build", pools=mp + mu, ms=round((first - second) * 1e3, 3))),
          flush=True)
    q = 10_000
    pr = rng.integers(0, n_pairs, size=q)
    side = rng.integers(0, 2, size=q)
    tin, tout = pairs[pr, side], pairs[pr, 1 - side]
    amt = np.full(q, 1e-4 * 500.0 * 1100)  # about 1e-4 of the pair's depth

    def objs(r):
        out = []
        o, typ, idx, _ = p.pair_pools([tin[r]], [tout[r]])
        for t, i in zip(typ, idx):
            if t == 0:
                out.append(so.Product(R[i], g[i], Ap[i]))
            else:
                out.append(so.Univ3(cp[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], gu[i], Au[i]))
        return out
    run(p, "hub", tin, tout, amt, objs, args.sample, rng, kinds=(0, 1))
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["headline", "hub"])
    ap.add_argument("--sample", type=int, default=8)
    args = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    rng = np.random.default_rng(2026)
    if args.only in (None, "headline"):
        headline(args, rng)
    if args.only in (None, "hub"):
        hub(args, rng)


if __name__ == "__main__":
    main()
