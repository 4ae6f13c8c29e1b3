"""Times cfmm_quote_routed_orders / cfmm_execute_routed_orders on one GPU and prints one JSON line per
measurement.

  hub       2k tokens; hub tokens 1..7 each paired with every other token by three pools (one
            ProductTwoCoin, one GeometricMeanTwoCoin, one UniV3 with a ragged ladder), and 20k sparse
            direct ProductTwoCoin pools between the other tokens, all priced near one ν per token.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set) with hubs 1..7: almost
            every pair holds at most one pool, and most hub pairs none.
For each set, rows sell a random non-hub token for another, exact-in, 1e-3 of a pool's depth, with 0,
1, 3 and 7 hubs (the first k of 1..7), 1k and 100k rows, quoted and then executed.  Per call: the wall
time of the synchronous call (host clock) and the kernel time (CUDA events, option "profile", slot 4:
the pair lookup and the route kernels, one launch per execute level), and, on a sample of rows, the
outer and inner evaluations per row (1k-row calls) counted by the host mirror (tests/route_oracle.py, which takes
the device's steps; its GeometricMeanTwoCoin pools are close to the device's, not equal, so their
counts can differ by a step).  The card's name and power limit are read in the same run (nvidia-smi,
read-only query).

    python tools/routed_order_timing.py [--only hub|headline] [--sample 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402
from split_order_timing import SLOT, card  # noqa: E402

HUBS = np.arange(1, 8, dtype=np.int64)


def timed(p, fn):
    """(fn(), wall ms, kernel ms, launches), with enough event pairs for one launch per execute level."""
    p.set_option("profile", 8192)
    p.profile_reset()
    t0 = time.perf_counter()
    out = fn()
    wall = time.perf_counter() - t0
    ms, launches = p.profile_read(SLOT)
    return out, wall * 1e3, ms, launches


def mirror_evals(p, pools_of, tin, tout, amt, hub_off, hubs, rows):
    import route_oracle as ro
    outer, inner = [], []
    for r in rows:
        hs = [(int(h), pools_of(tin[r], h), pools_of(h, tout[r])) for h in hubs[hub_off[r]:hub_off[r + 1]]]
        row = ro.route_row(pools_of(tin[r], tout[r]), hs, tin[r], tout[r], 0, amt[r])
        outer.append(row["outer"])
        inner += row["inner"]
    inner = inner or [0]
    return dict(outer_mean=round(float(np.mean(outer)), 1), outer_max=int(np.max(outer)),
                inner_per_hub_mean=round(float(np.mean(inner)), 1), inner_per_hub_max=int(np.max(inner)))


def run(p, name, tin, tout, amt, pools_of, sample, rng):
    for k in (0, 1, 3, 7):
        q = len(tin)
        hub_off = np.arange(q + 1, dtype=np.int64) * k
        hubs = np.tile(HUBS[:k], q)
        kind = np.zeros(q, np.uint8)
        out, wall, ms, launches = timed(p, lambda: p.quote_routed_orders(tin, tout, kind, amt, hub_off, hubs))
        rec = dict(set=name, call="quote", hubs=k, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                   launches=launches, filled=int(np.sum(out[3] == 0)))
        if sample:
            rec.update(mirror_evals(p, pools_of, tin, tout, amt, hub_off, hubs,
                                    rng.choice(q, size=min(sample, q), replace=False)))
        print(json.dumps(rec), flush=True)
        out, wall, ms, launches = timed(p, lambda: p.execute_routed_orders(tin, tout, kind, amt, hub_off, hubs))
        print(json.dumps(dict(set=name, call="execute", hubs=k, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                              launches=launches, filled=int(np.sum(out[3] == 0)))), flush=True)


def mirror_pools_of(p, R, g, Ai, w=None, u=None):
    """pools_of(a, b) for the mirror, from the host copies: the counts are on the set as built, while
    the device's state moves with every execute."""
    import split_oracle as so

    def pools_of(a, b):
        _, typ, idx, _ = p.pair_pools([int(a)], [int(b)])
        out = []
        for t, i in zip(typ, idx):
            if t == 0:
                out.append(so.Product(R[0][i], g[0][i], Ai[0][i]))
            elif t == 1:
                out.append(so.GeoMean(R[1][i], g[1][i], w[i], Ai[1][i]))
            else:
                cp, off, lt, lq = u
                out.append(so.Univ3(cp[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], g[2][i], Ai[2][i]))
        return out
    return pools_of


def hub_set(rng):
    """The hub set on a new context: (p, n, the non-hub tokens, ν, the mirror's pools_of)."""
    n, md = 2_000, 20_000
    nu = np.exp(rng.uniform(-1, 1, size=n + 1))
    others = np.arange(8, n + 1)
    A = np.array([(h, x) for h in HUBS for x in others], dtype=np.int64)
    m = len(A)
    depth = rng.uniform(1e3, 1e5, size=m)
    noise = lambda: np.exp(rng.uniform(-0.02, 0.02, size=(m, 2)))
    Rp, gp = depth[:, None] / nu[A] * noise(), rng.choice([0.997, 0.9995], size=m)
    Rg, gg, wg = depth[:, None] / nu[A] * noise(), np.full(m, 0.997), rng.uniform(0.3, 0.7, size=(m, 2))
    cp, gu, _, off, lt, lq = synth.univ3_pools(m, 2, seed=8, ragged=True)
    target = nu[A[:, 0]] / nu[A[:, 1]] * np.exp(rng.uniform(-0.02, 0.02, size=m))
    scale = np.repeat(target / cp, np.diff(off))
    lt, lq, cp = lt * scale, lq * np.repeat(depth / 100.0, np.diff(off)), target
    D = np.array([rng.choice(others, size=2, replace=False) for _ in range(md)], dtype=np.int64)
    dd = rng.uniform(1e3, 1e5, size=md)
    Rd = dd[:, None] / nu[D] * np.exp(rng.uniform(-0.02, 0.02, size=(md, 2)))
    Rp, gp, Ap = np.concatenate([Rp, Rd]), np.concatenate([gp, np.full(md, 0.997)]), np.concatenate([A, D])
    p = cr.DevicePools(n)
    p.add_product(Rp, gp, Ap)
    p.add_geomean(Rg, gg, A, wg)
    p.add_univ3(cp, gu, A, off, lt, lq)
    p.finalize()
    pools_of = mirror_pools_of(p, [Rp, Rg], [gp, gg, gu], [Ap, A, A], wg, (cp, off, lt, lq))
    print(json.dumps(dict(set="hub", pools=len(Ap) + 2 * m, tokens=n)), flush=True)
    return p, n, others, nu, pools_of


def hub(args, rng):
    p, n, others, nu, pools_of = hub_set(rng)
    for q in (1_000, 100_000):
        tin = rng.choice(others, size=q)
        tout = others[(np.searchsorted(others, tin) + rng.integers(1, len(others), size=q)) % len(others)]
        amt = 1e-3 * 1e4 / nu[tin]
        run(p, "hub", tin.astype(np.int64), tout.astype(np.int64), amt, pools_of, args.sample if q == 1_000 else 0,
            rng)
    p.close()


def headline(args, rng):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    pools_of = mirror_pools_of(p, [R], [g], [Ai])
    ok = np.flatnonzero((Ai[:, 0] > 7) & (Ai[:, 1] > 7))
    for q in (1_000, 100_000):
        pick = rng.choice(ok, size=q)
        side = rng.integers(0, 2, size=q)
        tin, tout = Ai[pick, side], Ai[pick, 1 - side]
        amt = 1e-3 * R[pick, side]
        run(p, "headline", tin.astype(np.int64), tout.astype(np.int64), amt, pools_of,
            args.sample if q == 1_000 else 0, rng)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--sample", type=int, default=3)
    args = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    rng = np.random.default_rng(2026)
    if args.only in (None, "hub"):
        hub(args, rng)
    if args.only in (None, "headline"):
        headline(args, rng)


if __name__ == "__main__":
    main()
