"""Times cfmm_scan_arbitrage and cfmm_execute_arbitrage on one GPU and prints one JSON line per
measurement.

  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set), base tokens 1..8.
  hub       tools/routed_order_timing.py's hub set (2k tokens, hubs 1..7 paired with every other
            token by a ProductTwoCoin, a GeometricMeanTwoCoin and a UniV3 pool, 20k sparse pools),
            base tokens 1..8.
For each set: the first-call adjacency build (the first scan's wall time less a second identical
scan's), then per max_hubs in 0 / 3 / 7 the scan's wall time (host clock), its kernel time per stage
(torch.profiler's CUDA kernel times: adjacency, rates, candidates, quote, sort = the scans, keep,
select, radix sorts and output), the candidate and row counts, and the execute of the returned rows
with their profits as minimums.  min_profit is 1e-9 of a base token.  The card's name and power limit
are read in the same run (nvidia-smi, read-only query).

    python tools/arbitrage_timing.py [--only hub|headline]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402
from split_order_timing import card  # noqa: E402

BASES = np.arange(1, 9, dtype=np.int64)
STAGES = (("adjacency", ("adj_",)), ("rates", ("arb_rates",)), ("candidates", ("arb_candidates", "arb_rows")),
          ("quote", ("arb_quote",)))


def stage_ms(prof):
    """Kernel ms per stage from a torch.profiler run; every other kernel counts as sort."""
    out = {k: 0.0 for k, _ in STAGES}
    out["sort"] = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name, ms = e.name, e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        for k, keys in STAGES:
            if any(s in name for s in keys):
                out[k] += ms
                break
        else:
            if "memset" not in name.lower() and "memcpy" not in name.lower():
                out["sort"] += ms
    return {k: round(v, 3) for k, v in out.items()}


def scan_once(p, mh):
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        out = p.scan_arbitrage(BASES, np.full(len(BASES), 1e-9), mh, cap=1 << 22)
        wall = (time.perf_counter() - t0) * 1e3
    return out, wall, stage_ms(prof)


def run(p, name):
    t0 = time.perf_counter()
    p.scan_arbitrage(BASES, np.full(len(BASES), 1e-9), 0, cap=0)
    first = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    p.scan_arbitrage(BASES, np.full(len(BASES), 1e-9), 0, cap=0)
    second = (time.perf_counter() - t0) * 1e3
    print(json.dumps(dict(set=name, call="adjacency_build", first_scan_ms=round(first, 3),
                          second_scan_ms=round(second, 3), build_ms=round(first - second, 3))), flush=True)
    for mh in (0, 3, 7):
        (found, rb, ro, hub_off, hubs, profit, _), wall, stages = scan_once(p, mh)
        print(json.dumps(dict(set=name, call="scan", max_hubs=mh, wall_ms=round(wall, 3), kernel_ms=stages,
                              rows=int(found), hubbed_rows=int(np.sum(np.diff(hub_off) > 0)),
                              hubs=int(len(hubs)))), flush=True)
        t0 = time.perf_counter()
        out = p.execute_arbitrage(rb, ro, hub_off, hubs, profit * 0.5)
        wall = (time.perf_counter() - t0) * 1e3
        print(json.dumps(dict(set=name, call="execute", max_hubs=mh, rows=len(rb), wall_ms=round(wall, 3),
                              filled=int(np.sum(out[3] == 0)), reverted=int(np.sum(out[3] == 1)))), flush=True)
        # the state moved: later max_hubs scans run on the state this execute left


def headline():
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    deg = np.bincount(Ai.reshape(-1), minlength=n + 1)
    print(json.dumps(dict(set="headline", pools=m, tokens=n, base_degree=deg[BASES].tolist())), flush=True)
    run(p, "headline")
    p.close()


def hub(rng):
    import routed_order_timing as rt
    n, md = 2_000, 20_000
    nu = np.exp(rng.uniform(-1, 1, size=n + 1))
    others = np.arange(8, n + 1)
    A = np.array([(h, x) for h in rt.HUBS for x in others], dtype=np.int64)
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
    print(json.dumps(dict(set="hub", pools=len(Ap) + 2 * m, tokens=n)), flush=True)
    run(p, "hub")
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
        headline()


if __name__ == "__main__":
    main()
