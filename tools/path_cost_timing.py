"""Times cfmm_find_order_paths_net and cfmm_quote_token_values_net against the existing calls on the
same rows, on one GPU; prints one JSON line per measurement.

The set is bench.py's headline set: 10M ProductTwoCoin pools, 50k tokens.
  best paths    100k rows at 1e-3 of a pool's depth, B = tokens 1..64, H = 4 and 8, exact-in and
                exact-out; hop costs 1e-6 of the amount.  Rows with a larger |B| take longer per level
                (best_path_timing.py) and the _net kernel adds one final pass per level.
  token values  one root at 8 hops, exact-in and exact-out; hop costs of 1e-6 of the amount per token.
Per call: the wall time of the synchronous call (host clock, after one untimed call of the same shape)
and the kernel time (CUDA events, option "profile", slot 4), for the existing call and the _net call in
turn, and how many rows or tokens took fewer hops than the existing call.  The card's name and power
limit are read in the same run (nvidia-smi, read-only query).

    python tools/path_cost_timing.py
"""
from __future__ import annotations

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
from split_order_timing import SLOT, card  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def timed(p, fn):
    fn()  # warm: the same shape once, untimed
    p.set_option("profile", 4096)
    p.profile_reset()
    t0 = time.perf_counter()
    out = fn()
    wall = time.perf_counter() - t0
    ms, _ = p.profile_read(SLOT)
    p.set_option("profile", 0)
    return out, round(wall * 1e3, 3), round(ms, 3)


def main():
    emit(card=card())
    rng = np.random.default_rng(2029)
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    emit(set="headline", pools=m, tokens=n)
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])
    nb, q = 64, 100_000
    allowed = np.arange(n) < nb
    ok = np.flatnonzero((Ai[:, 0] > nb) & (Ai[:, 1] > nb))
    for kind in (0, 1):
        sel = rng.choice(ok, size=q)
        side = rng.integers(0, 2, size=q)
        tin, tout = Ai[sel, side].astype(np.int64), Ai[sel, 1 - side].astype(np.int64)
        amount = 1e-3 * depth[tout if kind else tin]
        k = np.full(q, kind, np.uint8)
        for H in (4, 8):
            base, bw, bk = timed(p, lambda: p.find_order_paths(tin, tout, k, amount, H, allowed))
            got, nw, nk = timed(p, lambda: p.find_order_paths_net(tin, tout, k, amount, H, allowed, amount * 1e-6))
            fewer = int(np.sum(np.diff(got[0]) < np.diff(base[0])))
            emit(call="best_paths", B=nb, rows=q, max_hops=H, kind=("in", "out")[kind], wall_ms=bw, kernel_ms=bk,
                 net_wall_ms=nw, net_kernel_ms=nk, filled=int(np.sum(got[7] == 0)), fewer_hops=fewer)
    for kind in (0, 1):
        root = np.array([int(rng.integers(1, n + 1))], np.int64)
        amount = np.array([1e-3 * depth[root[0]]])
        k = np.array([kind], np.uint8)
        kappa = np.full(n, amount[0] * 1e-6)
        base, bw, bk = timed(p, lambda: p.quote_token_values(root, k, amount, 8))
        got, nw, nk = timed(p, lambda: p.quote_token_values_net(root, k, amount, 8, kappa))
        emit(call="token_values", rows=1, max_hops=8, kind=("in", "out")[kind], wall_ms=bw, kernel_ms=bk,
             net_wall_ms=nw, net_kernel_ms=nk, reached=int(np.sum(got[2] == 0)),
             fewer_hops=int(np.sum(got[1] < base[1])))
    p.close()


if __name__ == "__main__":
    main()
