"""Times cfmm_quote_paths / cfmm_execute_paths on one GPU and prints one JSON line per measurement.

  quote 1M random 3-hop paths, exact-in and exact-out
  execute a 1k-path block in which 20 % of the paths cross one hub pool (a level per hub path)
  execute 1M random 3-hop paths, nearly pool-disjoint (few levels)

For each: the wall time of the synchronous call (host clock), the kernel time (CUDA events,
option "profile", slot 4: the token check plus the quote or level launches), the number of
levels and the context's launch count over the call (levels, the token check and the bookkeeping
after an execute).  Paths are random walks on the set's own token pairs (Ai), three distinct pools
each.  Exact-in paths tender 1e-4 of the first pool's reserve on the tendered side
(ProductTwoCoin) or 1e-4 (UniV3); exact-out paths want what the exact-in quote of the same path
received, so both quotes price the same trades.

Sets: the headline (10M ProductTwoCoin pools, 50k tokens) and config 4 of bench.py (500k UniV3
pools of 4 ticks, 5k tokens).  The card's name and power limit are read in the same run
(nvidia-smi, read-only query).

    python tools/path_timing.py [--only headline|config4] [--paths 1000000]
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


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # (no nvidia-smi: the number still stands, without its label)
        return f"unknown ({e})"


def walks(Ai, n, q, hops, rng, first=None):
    """q random walks of `hops` distinct pools over the 1-based token pairs Ai: (pools [q, hops],
    token_in [q]).  first: the first pool of every walk (else random)."""
    m = len(Ai)
    tok = (Ai - 1).reshape(-1)
    order = np.argsort(tok, kind="stable")
    by_tok = order // 2                               # pools sorted by token, each pool twice
    start = np.searchsorted(tok[order], np.arange(n + 1))
    deg = np.diff(start)
    pools = np.zeros((q, hops), np.int64)
    pools[:, 0] = rng.integers(0, m, size=q) if first is None else first
    side = rng.integers(0, 2, size=q)
    t_in = Ai[pools[:, 0], side]
    t = Ai[pools[:, 0], 1 - side]
    for h in range(1, hops):
        todo = np.arange(q)
        while len(todo):
            tt = t[todo] - 1
            pick = by_tok[start[tt] + (rng.random(len(todo)) * deg[tt]).astype(np.int64)]
            pools[todo, h] = pick
            bad = np.any(pools[todo, :h] == pick[:, None], axis=1)
            todo = todo[bad]
        a, b = Ai[pools[:, h], 0], Ai[pools[:, h], 1]
        t = np.where(t == a, b, a)
    return pools, t_in


def timed(p, fn, *args):
    p.set_option("profile", 1 << 13)
    l0 = p.launch_count
    t0 = time.perf_counter()
    out = fn(*args)
    wall = time.perf_counter() - t0
    ms, prof = p.profile_read(4)
    p.set_option("profile", 0)
    return out, dict(wall_ms=wall * 1e3, kernel_ms=ms, levels=int(prof) - 1, launches=int(p.launch_count - l0))


def csr(t, pools, t_in, kind, amount):
    q, hops = pools.shape
    return (np.arange(q + 1, dtype=np.int64) * hops, np.full(q * hops, t, np.int32), pools.reshape(-1), t_in,
            np.full(q, kind, np.uint8) if np.isscalar(kind) else kind, amount)


def run_set(name, t, n, pools, q, gpu):
    def emit(what, **kw):
        print(json.dumps({"set": name, "what": what, **kw, "gpu": gpu}), flush=True)

    p = cr.DevicePools(n)
    (p.add_product if t == 0 else p.add_univ3)(*pools)
    p.finalize()
    Ai = pools[2]
    m = len(Ai)
    rng = np.random.default_rng(1)
    P, t_in = walks(Ai, n, q, 3, rng)
    first_side = (Ai[P[:, 0], 0] == t_in).astype(int)  # 1: tenders token 1
    x_in = (pools[0][P[:, 0], 1 - first_side] if t == 0 else np.ones(q)) * 1e-4
    p.quote_paths(*csr(t, P[:8], t_in[:8], 0, x_in[:8]))  # (first launch of each kernel)
    (_, rec, st), kw = timed(p, p.quote_paths, *csr(t, P, t_in, 0, x_in))
    emit(f"quote {q} 3-hop paths, exact-in", paths=q, **kw, status_counts=np.bincount(st, minlength=4).tolist())
    want = np.maximum(rec[2::3], 0.0)
    (_, _, st), kw = timed(p, p.quote_paths, *csr(t, P, t_in, 1, want))
    emit(f"quote {q} 3-hop paths, exact-out", paths=q, **kw, status_counts=np.bincount(st, minlength=4).tolist())
    # a 1k-path block, 20 % of it through one hub pool
    k = 1000
    hub = int(rng.integers(0, m))
    B, b_in = walks(Ai, n, k, 3, rng)
    H, h_in = walks(Ai, n, k // 5, 3, rng, first=np.full(k // 5, hub))
    at = rng.choice(k, size=k // 5, replace=False)
    B[at], b_in[at] = H, h_in
    kind = (np.arange(k) % 2).astype(np.uint8)
    side = (Ai[B[:, 0], 0] == b_in).astype(int)
    amt = np.where(kind == 0, (pools[0][B[:, 0], 1 - side] if t == 0 else np.ones(k)) * 1e-4, 0.0)
    _, rk, _ = p.quote_paths(*csr(t, B, b_in, 0, amt))
    amt = np.where(kind == 0, amt, np.maximum(rk[2::3], 0.0) * 0.5)
    p.execute_paths(*csr(t, B[:4], b_in[:4], kind[:4], amt[:4]))
    (_, _, st), kw = timed(p, p.execute_paths, *csr(t, B, b_in, kind, amt))
    emit(f"execute {k} paths, 20 % through one hub pool", paths=k, **kw,
         status_counts=np.bincount(st, minlength=4).tolist())
    # 1M near-disjoint paths
    (_, _, st), kw = timed(p, p.execute_paths, *csr(t, P, t_in, 0, x_in))
    emit(f"execute {q} 3-hop paths, near-disjoint", paths=q, **kw,
         status_counts=np.bincount(st, minlength=4).tolist())
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=("headline", "config4"))
    ap.add_argument("--paths", type=int, default=1_000_000)
    a = ap.parse_args()
    gpu = card()
    if a.only in (None, "headline"):
        run_set("headline (ProductTwoCoin)", 0, 50_000, synth.product_pools(10_000_000, 50_000, seed=1), a.paths, gpu)
    if a.only in (None, "config4"):
        run_set("config4 (UniV3, 4 ticks)", 2, 5_000, synth.univ3_pools(500_000, 5_000, seed=1), a.paths, gpu)


if __name__ == "__main__":
    main()
