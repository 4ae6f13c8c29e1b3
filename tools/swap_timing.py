"""Times cfmm_quote_swaps / cfmm_execute_swaps on one GPU and prints one JSON line per measurement.

  quote and execute of every pool (one row each) and of 1k pools: the wall time of the
  synchronous call (host clock) and the kernel time (CUDA events, option "profile", slot 4)
  the gradient sweep before and after an execute (median of CUDA events, option "sweep_events")

Sets: the headline (10M ProductTwoCoin pools, 50k tokens) and config 4 of bench.py (500k UniV3
pools of 4 ticks, 5k tokens).  GB/s is the byte model below over the kernel time; the card's name
and power limit are read in the same run (nvidia-smi, read-only query).

Byte model per row (DRAM traffic the kernel cannot avoid; index arrays are int64):
  ProductTwoCoin quote     tender 16 + received 16 + row 8 + pos 8 + R 16 + γ 8 + gidx 8 = 80
  ProductTwoCoin execute   the same + segment offset 8 + R written back 16             = 104
  UniV3 quote              tender 16 + received 16 + row 8 + pos 8 + γ 8 + tick 8 + price 16
                           + the ticks walked (lower 8 + liq 8 each; the walk reads 2 ticks
                           at least: the current one and its neighbour for the bounds)   = 112
  UniV3 execute            the same + segment offset 8 + price written 8                 = 128

    python tools/swap_timing.py [--only headline|config4] [--sweeps 50]
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

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402

BYTES = {("product", "quote"): 80, ("product", "execute"): 104, ("univ3", "quote"): 112, ("univ3", "execute"): 128}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as e:  # (no nvidia-smi: the number still stands, without its label)
        return f"unknown ({e})"


def sweep_us(p, v, k):
    p.set_option("sweep_events", 1)
    p.sweep(v)
    ts = []
    for _ in range(k):
        p.sweep(v)
        ts.append(p.last_sweep_ms() * 1e3)
    p.set_option("sweep_events", 0)
    return float(np.median(ts))


def timed_call(p, fn, *args):
    p.set_option("profile", 16)
    t0 = time.perf_counter()
    fn(*args)
    wall = time.perf_counter() - t0
    ms, launches = p.profile_read(4)
    p.set_option("profile", 0)
    return wall, ms, launches


def run_set(name, kind, t, n, pools, k, gpu):
    def emit(what, **kw):
        print(json.dumps({"set": name, "what": what, **kw, "gpu": gpu}), flush=True)

    p = cr.DevicePools(n)
    (p.add_product if t == 0 else p.add_univ3)(*pools)
    p.finalize()
    m = len(pools[1])
    v = synth.dual_prices(n, "near")
    emit("gradient sweep before execute", us=sweep_us(p, v, k))
    rng = np.random.default_rng(1)
    scale = pools[0] if t == 0 else np.ones((m, 2))
    side = rng.integers(0, 2, size=m)
    T = np.zeros((m, 2))
    T[np.arange(m), side] = scale[np.arange(m), side] * 1e-4
    for rows, label in ((np.arange(m), f"all {m} pools"), (rng.choice(m, size=1000, replace=False), "1k pools")):
        for op, fn in (("quote", p.quote_swaps), ("execute", p.execute_swaps)):
            fn(t, rows[:8], T[rows[:8]])  # (first launch of the kernel)
            wall, ms, launches = timed_call(p, fn, t, rows, T[rows])
            gbs = BYTES[(kind, op)] * len(rows) / (ms * 1e-3) / 1e9 if ms > 0 else None
            emit(f"{op}, {label}", rows=len(rows), wall_ms=wall * 1e3, kernel_ms=ms, launches=launches,
                 model_bytes_per_row=BYTES[(kind, op)], GBps=gbs)
    emit("gradient sweep after execute", us=sweep_us(p, v, k))
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=50)
    ap.add_argument("--only", choices=("headline", "config4"))
    a = ap.parse_args()
    gpu = card()
    if a.only in (None, "headline"):
        run_set("headline (ProductTwoCoin)", "product", 0, 50_000, synth.product_pools(10_000_000, 50_000, seed=1),
                a.sweeps, gpu)
    if a.only in (None, "config4"):
        run_set("config4 (UniV3, 4 ticks)", "univ3", 2, 5_000, synth.univ3_pools(500_000, 5_000, seed=1), a.sweeps,
                gpu)


if __name__ == "__main__":
    main()
