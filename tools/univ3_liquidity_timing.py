"""Times cfmm_modify_univ3_liquidity on one GPU and prints one JSON line per measurement.

  1k rows on existing boundaries         tick counts unchanged: liquidities rewritten in place
  1k rows with new boundaries            ladders grow: the set's tick arrays are spliced
  one new-boundary row on every pool     every ladder grows by one or two ticks
  the gradient sweep before and after that last batch (CUDA events, median of 50): a grown ladder
  costs walk time
  destroy + add + finalize of the same set, the alternative without the entry point

Sets: those of tools/univ3_state_timing.py, config 4 of bench.py (500k UniV3 pools of 4 ticks, 5k
tokens) and the ragged set (1..16 ticks per pool).  Wall times are medians of a host clock around
the (synchronous) calls; the kernel time per call is the sum of the library's kernels over the
call, from torch.profiler.  The GPU name and power limit are read in the same run.

    python tools/univ3_liquidity_timing.py [--pools 500000] [--tokens 5000] [--reps 10]
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


def emit(rec):
    print(json.dumps(rec), flush=True)


def gpu_info():
    out = {"gpu": None, "power_limit_W": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = (x.strip() for x in q.split(","))
        out = {"gpu": name, "power_limit_W": float(pl)}
    except Exception:
        pass
    return out


def kernel_s(fn, reps):
    """Device time per call of the library's kernels, from torch.profiler (None without torch)."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except Exception:
        return None
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for e in prof.events():
        if "cfmm::univ3" in e.name or "univ3_" in e.name:
            us += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return us * 1e-6 / reps if us > 0 else None


def sweep_ms(p, v, reps=50):
    p.set_option("sweep_events", 1)
    for _ in range(5):
        p.sweep(v)
    ts = []
    for _ in range(reps):
        p.sweep(v)
        ts.append(p.last_sweep_ms())
    p.set_option("sweep_events", 0)
    return float(np.median(ts))


def build(n, pools):
    p = cr.DevicePools(n)
    p.add_univ3(*pools)
    p.finalize()
    return p


def rows(off, lt, rng, q, new):
    """q rows on random pools: on existing boundaries (new=False; pools with >= 2 ticks) or with
    bounds below and above the ingested ladder (new=True; the first call on a pool grows it by two
    ticks).  Distinct pools, each minted and then burned by the same amount, so that repeated calls
    never drive a tick below zero."""
    m = len(off) - 1
    nt = np.diff(off)
    pools = rng.choice(np.flatnonzero(nt >= 2) if not new else m, size=q // 2, replace=False)
    a, b = off[pools], off[pools + 1] - 1
    if new:
        lo, hi = lt[b] * 0.9, lt[a] * 1.1
    else:
        lo, hi = lt[b], lt[a]
    d = rng.uniform(1.0, 10.0, size=len(pools))
    return (np.concatenate([pools, pools]), np.concatenate([lo, lo]), np.concatenate([hi, hi]),
            np.concatenate([d, -d]))


def run_set(name, n, pools, reps, info):
    cp, g, Ai, off, lt, lq = pools
    m = len(cp)
    base = {"set": name, "pools": m, "ticks": int(off[-1]), **info}
    rng = np.random.default_rng(1)
    p = build(n, pools)
    for what, new in (("1k rows on existing boundaries (in place)", False),
                      ("1k rows with new boundaries (splice)", True)):
        r = rows(off, lt, rng, 1000, new)
        p.modify_univ3_liquidity(*r)  # warm-up
        calls = [rows(off, lt, np.random.default_rng(100 + k), 1000, new) for k in range(reps)]
        ts = []
        for c in calls:
            t0 = time.perf_counter()
            p.modify_univ3_liquidity(*c)
            ts.append(time.perf_counter() - t0)
        kcalls = iter([rows(off, lt, np.random.default_rng(200 + k), 1000, new) for k in range(reps)])
        k = kernel_s(lambda: p.modify_univ3_liquidity(*next(kcalls)), reps)
        emit({**base, "what": what, "s": float(np.median(ts)), "kernels_s": k})
    p.close()
    p = build(n, pools)
    v = synth.dual_prices(n, "wide")
    before = sweep_ms(p, v)
    every = np.arange(m)
    mid = lt[off[1:] - 1] * 0.5  # below the last tick: one new boundary per pool
    t0 = time.perf_counter()
    p.modify_univ3_liquidity(every, mid, lt[off[:-1]] * 1.25, np.full(m, 1.0))
    wall = time.perf_counter() - t0
    after = sweep_ms(p, v)
    p.close()
    q = build(n, pools)
    kk = kernel_s(lambda: q.modify_univ3_liquidity(every, mid, lt[off[:-1]] * 1.25, np.full(m, 1.0)), 1)
    q.close()
    emit({**base, "what": "one new-boundary row on every pool (splice)", "s": wall, "kernels_s": kk,
          "ticks_after": int(off[-1]) + 2 * m})
    emit({**base, "what": "gradient sweep before / after that batch, ms (CUDA events, median of 50)",
          "before_ms": before, "after_ms": after})
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        build(n, pools).close()
        ts.append(time.perf_counter() - t0)
    emit({**base, "what": "destroy + add + finalize", "s": float(np.median(ts))})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=500_000)
    ap.add_argument("--tokens", type=int, default=5_000)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    info = gpu_info()
    sets = [("config4 (4 ticks)", synth.univ3_pools(a.pools, a.tokens, seed=1)),
            ("ragged (1..16 ticks)", synth.univ3_pools(a.pools, a.tokens, seed=2, ragged=True))]
    for name, pools in sets:
        run_set(name, a.tokens, pools, a.reps, info)


if __name__ == "__main__":
    main()
