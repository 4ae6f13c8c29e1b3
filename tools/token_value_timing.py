"""Times cfmm_quote_token_values on one GPU and prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hub tokens 1..7 each paired with every other
            token by a ProductTwoCoin, a GeometricMeanTwoCoin and a UniV3 pool, 20k sparse direct
            ProductTwoCoin pools between the other tokens.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
For each set: q = 1, 8 and 64 rows (random roots), max_hops 2, 4 and 8, exact-in and exact-out, amounts
at 1e-3 of a pool's depth in the root.  Per call: the wall time of the synchronous call (host clock,
after one untimed call of the same shape), the kernel time (CUDA events, option "profile", slot 4), the
levels actually run (the last level at which some row changed a token, plus one when that is below
max_hops: the level that found nothing) and the per-level frontier sizes summed over the rows.  The
card's name and power limit are read in the same run (nvidia-smi, read-only query).

    python tools/token_value_timing.py [--only hub|headline]
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
from routed_order_timing import hub_set  # noqa: E402
from split_order_timing import SLOT, card  # noqa: E402


def timed(p, fn):
    p.set_option("profile", 4096)
    p.profile_reset()
    t0 = time.perf_counter()
    out = fn()
    wall = time.perf_counter() - t0
    ms, launches = p.profile_read(SLOT)
    return out, wall * 1e3, ms, launches


def run(p, name, roots_of, depth_of, rng):
    for q in (1, 8, 64):
        roots = roots_of(q)
        amount = 1e-3 * depth_of(roots)
        for H in (2, 4, 8):
            for kind in (0, 1):
                kinds = np.full(q, kind, np.uint8)
                p.quote_token_values(roots, kinds, amount, H)  # warm: the workspace is sized once
                out, wall, ms, launches = timed(p, lambda: p.quote_token_values(roots, kinds, amount, H))
                value, _, status, front = out
                per_level = front.sum(axis=0)
                changed = np.flatnonzero(per_level > 0)
                levels = int(changed[-1]) + 1 if len(changed) else 0
                levels = min(levels + 1, H)  # the level that found no change, when there is one
                print(json.dumps(dict(set=name, rows=q, max_hops=H, kind=("exact_in", "exact_out")[kind],
                                      wall_ms=round(wall, 3), kernel_ms=round(ms, 3), launches=launches,
                                      levels_run=levels, frontier=per_level.tolist(),
                                      reached_per_row=round(float(np.mean(np.sum(status == 0, axis=1))), 1),
                                      repeats_pool=int(np.sum(status == 4)))), flush=True)


def hub(rng):
    p, n, others, nu, _ = hub_set(rng)
    run(p, "hub", lambda q: rng.choice(others, size=q).astype(np.int64), lambda r: 1e4 / nu[r], rng)
    p.close()


def headline(rng):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    print(json.dumps(dict(set="headline", pools=m, tokens=n)), flush=True)
    # a pool's depth in token t: the mean reserve of t over its pools
    depth = np.zeros(n + 1)
    cnt = np.zeros(n + 1)
    for side in (0, 1):
        np.add.at(depth, Ai[:, side], R[:, side])
        np.add.at(cnt, Ai[:, side], 1.0)
    depth = depth / np.maximum(cnt, 1.0)
    run(p, "headline", lambda q: rng.integers(1, n + 1, size=q).astype(np.int64), lambda r: depth[r], rng)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    args = ap.parse_args()
    print(json.dumps(dict(card=card())), flush=True)
    rng = np.random.default_rng(2026)
    if args.only in (None, "hub"):
        hub(rng)
    if args.only in (None, "headline"):
        headline(rng)


if __name__ == "__main__":
    main()
