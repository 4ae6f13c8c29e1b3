"""Times the pool-membership entry points on one GPU and prints one JSON line per measurement.

  cfmm_append_* of 1k pools, then of 100k more, into a finalized set (the tail is re-laid out)
  cfmm_set_active: retire 1 % of the set's pools, then restore them
  cfmm_compact (folds the tail into the main layout, reruns the calibration sweeps)
  the gradient sweep with a 100k-pool tail, and the same pools after cfmm_compact

Sets: the headline (10M ProductTwoCoin pools, 50k tokens) and config 4 of bench.py (500k UniV3
pools of 4 ticks, 5k tokens); the appended pools come from the same generator.  Call times are a
synchronised host clock around the (synchronous) calls; sweep times are the medians of CUDA
events around the sweep kernels (option "sweep_events").

    python tools/pool_membership_timing.py [--sweeps 50] [--only headline|config4]
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

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402


def cut(t, a, lo, hi):
    if t != 2:
        return tuple(x[lo:hi] for x in a)
    cp, g, Ai, off, lt, lq = a
    return cp[lo:hi], g[lo:hi], Ai[lo:hi], off[lo:hi + 1] - off[lo], lt[off[lo]:off[hi]], lq[off[lo]:off[hi]]


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def sweep_us(p, v, k):
    p.set_option("sweep_events", 1)
    p.sweep(v)
    ts = []
    for _ in range(k):
        p.sweep(v)
        ts.append(p.last_sweep_ms() * 1e3)
    p.set_option("sweep_events", 0)
    return float(np.median(ts))


def run_set(name, t, n, pools, m_main, k, gpu):
    add = ("add_product", "add_geomean", "add_univ3")[t]
    app = ("append_product", "append_geomean", "append_univ3")[t]

    def emit(what, **kw):
        print(json.dumps({"set": name, "what": what, **kw, "gpu": gpu}), flush=True)

    p = cr.DevicePools(n)
    getattr(p, add)(*cut(t, pools, 0, m_main))
    emit("cfmm_finalize", pools=m_main, s=timed(p.finalize))
    v = synth.dual_prices(n, "near")
    base = sweep_us(p, v, k)
    emit("gradient sweep, no tail", us=base)
    emit("append 1k pools (empty tail)", s=timed(lambda: getattr(p, app)(*cut(t, pools, m_main, m_main + 1_000))))
    emit("append 100k pools (tail of 1k)",
         s=timed(lambda: getattr(p, app)(*cut(t, pools, m_main + 1_000, m_main + 101_000))))
    tail = sweep_us(p, v, k)
    emit("gradient sweep with a 101k-pool tail", us=tail)
    m = m_main + 101_000
    active = np.ones(m, dtype=bool)
    active[np.random.default_rng(1).choice(m, size=m // 100, replace=False)] = False
    emit("retire 1 % of the pools", s=timed(lambda: p.set_active(t, 0, active)))
    emit("restore them", s=timed(lambda: p.set_active(t, 0, np.ones(m, dtype=bool))))
    emit("cfmm_compact", pools=m, s=timed(p.compact))
    emit("gradient sweep after compact", us=sweep_us(p, v, k))
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=50)
    ap.add_argument("--only", choices=("headline", "config4"))
    a = ap.parse_args()
    gpu = None
    try:
        import torch
        gpu = torch.cuda.get_device_name(0)
    except Exception:
        pass
    if a.only in (None, "headline"):
        run_set("headline (ProductTwoCoin)", 0, 50_000, synth.product_pools(10_101_000, 50_000, seed=1),
                10_000_000, a.sweeps, gpu)
    if a.only in (None, "config4"):
        run_set("config4 (UniV3, 4 ticks)", 2, 5_000, synth.univ3_pools(601_000, 5_000, seed=1), 500_000,
                a.sweeps, gpu)


if __name__ == "__main__":
    main()
