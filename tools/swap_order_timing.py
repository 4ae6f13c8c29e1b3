"""Times cfmm_quote_swaps_exact_out / cfmm_execute_swap_orders on one GPU and prints one JSON line
per measurement.

  exact-in quote (cfmm_quote_swaps, for comparison) and exact-out quote of every pool (one row
  each) and of 1k pools: the wall time of the synchronous call (host clock) and the kernel time
  (CUDA events, option "profile", slot 4)
  a mixed execute with limits: every pool, or 1k pools, one row each, half exact-in and half
  exact-out, each limit within 0.1 % of the row's isolated quote so that about half revert
  f evaluations per exact-out row: mean and maximum, from the host mirror
  (tests/swap_order_oracle.py) on a sample of the quoted rows

Sets: the headline (10M ProductTwoCoin pools, 50k tokens) and config 4 of bench.py (500k UniV3
pools of 4 ticks, 5k tokens).  The wanted outputs are what the exact-in quote of a tender of
1e-4 of the tender side's reserve (ProductTwoCoin) or of 1e-4 (UniV3) receives, so both quotes
price the same trades.  The card's name and power limit are read in the same run (nvidia-smi,
read-only query).

    python tools/swap_order_timing.py [--only headline|config4] [--sample 2000]
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
import swap_order_oracle as oo  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # (no nvidia-smi: the number still stands, without its label)
        return f"unknown ({e})"


def timed_call(p, fn, *args):
    p.set_option("profile", 16)
    t0 = time.perf_counter()
    out = fn(*args)
    wall = time.perf_counter() - t0
    ms, launches = p.profile_read(4)
    p.set_option("profile", 0)
    return out, wall, ms, launches


def host_pool(t, pools, i):
    if t == 0:
        R, g, _ = pools
        return oo.ProductPool(R[i], g[i])
    cp, g, _, off, lt, lq = pools
    return oo.Univ3Pool(cp[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], g[i])


def run_set(name, t, n, pools, sample, gpu):
    def emit(what, **kw):
        print(json.dumps({"set": name, "what": what, **kw, "gpu": gpu}), flush=True)

    p = cr.DevicePools(n)
    (p.add_product if t == 0 else p.add_univ3)(*pools)
    p.finalize()
    m = len(pools[1])
    rng = np.random.default_rng(1)
    scale = pools[0] if t == 0 else np.ones((m, 2))
    side = rng.integers(0, 2, size=m)
    T = np.zeros((m, 2))
    T[np.arange(m), side] = scale[np.arange(m), side] * 1e-4
    all_rows = np.arange(m)
    p.quote_swaps(t, all_rows[:8], T[:8])  # (first launch of each kernel)
    W, wall, ms, launches = timed_call(p, p.quote_swaps, t, all_rows, T)
    emit(f"exact-in quote, all {m} pools", rows=m, wall_ms=wall * 1e3, kernel_ms=ms, launches=launches)
    p.quote_swaps_exact_out(t, all_rows[:8], W[:8])
    X, wall, ms, launches = timed_call(p, p.quote_swaps_exact_out, t, all_rows, W)
    emit(f"exact-out quote, all {m} pools", rows=m, wall_ms=wall * 1e3, kernel_ms=ms, launches=launches,
         unreachable=int(np.isinf(X).any(axis=1).sum()))
    k1 = rng.choice(m, size=1000, replace=False)
    for op, fn, A in (("exact-in quote", p.quote_swaps, T), ("exact-out quote", p.quote_swaps_exact_out, W)):
        _, wall, ms, launches = timed_call(p, fn, t, k1, A[k1])
        emit(f"{op}, 1k pools", rows=1000, wall_ms=wall * 1e3, kernel_ms=ms, launches=launches)
    # f evaluations per exact-out row, from the host mirror on a sample of the rows just quoted
    evals, same = [], 0
    for i in rng.choice(m, size=sample, replace=False):
        y = W[i].max()
        x, k = oo.exact_out(host_pool(t, pools, i), y, W[i, 1] > 0)
        evals.append(k)
        same += x == X[i].max()
    emit("f evaluations per exact-out row (host mirror)", sample=sample, mean=float(np.mean(evals)),
         max=int(np.max(evals)), p50=float(np.median(evals)), mirror_equal=int(same))
    # a mixed execute with limits, one row per pool
    kind = rng.integers(0, 2, size=m).astype(np.uint8)
    amount = np.where(kind[:, None] == 1, W, T)
    iso = np.where(kind == 1, X.max(axis=1), W.max(axis=1))
    limit = iso * rng.uniform(0.999, 1.001, size=m)
    for rows, label in ((k1, "1k pools"), (all_rows, f"all {m} pools")):
        p.execute_swap_orders(t, rows[:8], kind[rows[:8]], amount[rows[:8]], limit[rows[:8]])
        (_, _, st), wall, ms, launches = timed_call(p, p.execute_swap_orders, t, rows, kind[rows], amount[rows],
                                                    limit[rows])
        emit(f"mixed execute with limits, {label}", rows=len(rows), wall_ms=wall * 1e3, kernel_ms=ms,
             launches=launches, status_counts=np.bincount(st, minlength=4).tolist())
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("headline", "config4"))
    ap.add_argument("--sample", type=int, default=2000)
    a = ap.parse_args()
    gpu = card()
    if a.only in (None, "headline"):
        run_set("headline (ProductTwoCoin)", 0, 50_000, synth.product_pools(10_000_000, 50_000, seed=1), a.sample,
                gpu)
    if a.only in (None, "config4"):
        run_set("config4 (UniV3, 4 ticks)", 2, 5_000, synth.univ3_pools(500_000, 5_000, seed=1), a.sample, gpu)


if __name__ == "__main__":
    main()
