"""Times the UniV3 state entry points on one GPU and prints one JSON line per measurement.

  cfmm_update_univ3, prices only and prices + liquidity, of every pool of the set
  cfmm_apply_trades after a materialising sweep
  the alternative without them: destroy, add and finalize the same set again
  cfmm_finalize alone

Sets: config 4 of bench.py (500k UniV3 pools of 4 ticks, 5k tokens) and the ragged set
(1..16 ticks per pool).  Wall times are medians of a synchronised host clock around the
(synchronous) calls.  With torch available, the device time of the rebuild kernels
(univ3_current_tick_kernel + univ3_ticks_kernel) is read from torch.profiler as well, and the
achieved bandwidth is the rebuild's byte count (80 B/tick + 72 B/pool) over that time.

    python tools/univ3_state_timing.py [--pools 500000] [--tokens 5000] [--reps 10]
    CFMM_B200_LIB=/path/to/other/libcfmm_b200.so python tools/univ3_state_timing.py --finalize-only
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


def median_s(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def rebuild_kernel_s(fn, reps):
    """Device time per call of the rebuild kernels, from torch.profiler (None without torch)."""
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
        if "univ3_current_tick_kernel" in e.name or "univ3_ticks_kernel" in e.name:
            us += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return us * 1e-6 / reps if us > 0 else None


def build(n, pools):
    p = cr.DevicePools(n)
    p.add_univ3(*pools)
    t0 = time.perf_counter()
    p.finalize()
    return p, time.perf_counter() - t0


def emit(rec):
    print(json.dumps(rec), flush=True)


def run_set(name, n, pools, reps, gpu):
    cp, g, Ai, off, lt, lq = pools
    m, ticks = len(cp), int(off[-1])
    rebuild_bytes = 80 * ticks + 72 * m
    fin = []
    for _ in range(3):
        p, t = build(n, pools)
        fin.append(t)
        p.close()
    emit({"set": name, "pools": m, "ticks": ticks, "what": "cfmm_finalize", "s": float(np.median(fin)), "gpu": gpu})
    p, _ = build(n, pools)
    rng = np.random.default_rng(1)
    cp2 = np.minimum(cp * rng.uniform(0.5, 1.5, size=m), lt[off[:-1]])
    lq2 = lq * rng.uniform(0.5, 1.5, size=len(lq))
    for what, fn in (("cfmm_update_univ3 prices", lambda: p.update_univ3(0, cp2)),
                     ("cfmm_update_univ3 prices+liquidity", lambda: p.update_univ3(0, cp2, lq2))):
        fn()
        s = median_s(fn, reps)
        k = rebuild_kernel_s(fn, reps)
        rec = {"set": name, "pools": m, "ticks": ticks, "what": what, "s": s, "gpu": gpu,
               "rebuild_bytes": rebuild_bytes}
        if k:
            rec.update(rebuild_kernels_s=k, rebuild_GBps=rebuild_bytes / k / 1e9)
        emit(rec)
    v = synth.dual_prices(n, "wide")
    ts = []
    for r in range(reps):
        p.sweep(v * (1.0 + 0.01 * r), materialize=True)
        t0 = time.perf_counter()
        p.apply_trades()
        ts.append(time.perf_counter() - t0)
    emit({"set": name, "pools": m, "ticks": ticks, "what": "cfmm_apply_trades after a materialising sweep",
          "s": float(np.median(ts)), "gpu": gpu})
    p.close()

    def rebuild_all():
        q, _ = build(n, pools)
        q.close()
    emit({"set": name, "pools": m, "ticks": ticks, "what": "destroy + add + finalize", "s": median_s(rebuild_all, 3),
          "gpu": gpu})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pools", type=int, default=500_000)
    ap.add_argument("--tokens", type=int, default=5_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--finalize-only", action="store_true")
    a = ap.parse_args()
    gpu = None
    try:
        import torch
        gpu = torch.cuda.get_device_name(0)
    except Exception:
        pass
    sets = [("config4 (4 ticks)", synth.univ3_pools(a.pools, a.tokens, seed=1)),
            ("ragged (1..16 ticks)", synth.univ3_pools(a.pools, a.tokens, seed=2, ragged=True))]
    for name, pools in sets:
        if a.finalize_only:
            fin = []
            for _ in range(3):
                p, t = build(a.tokens, pools)
                fin.append(t)
                p.close()
            emit({"set": name, "pools": a.pools, "ticks": int(pools[3][-1]), "what": "cfmm_finalize",
                  "s": float(np.median(fin)), "lib": cr.LIB_PATH, "gpu": gpu})
        else:
            run_set(name, a.tokens, pools, a.reps, gpu)


if __name__ == "__main__":
    main()
