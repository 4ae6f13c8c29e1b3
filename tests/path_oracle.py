"""Host mirror of cfmm_quote_paths / cfmm_execute_paths (include/cfmm_b200.h), for the tests.  It
composes the pool objects and exact_out of swap_order_oracle.py, so for ProductTwoCoin and UniV3
hops it gives the device's bits (GeometricMeanTwoCoin hops are close, not equal: numpy's log1p /
expm1 are not CUDA's).

  hop_sides      the token walk of one path: per hop, does it tender its pool's token 1
  quote_path     one path on the current state: per-hop tender and received, and the status
  quote_paths    every path of a CSR batch on its own
  replay_paths   the batch in order, filled paths executed hop by hop, reverted ones changing nothing
"""
from __future__ import annotations

import numpy as np

import swap_order_oracle as oo
from swap_order_oracle import EXACT_IN, EXACT_OUT, FILLED, INF, LIMIT, RETIRED, UNREACHABLE  # noqa: F401


def hop_sides(pairs, token_in):
    """tok1 per hop for a path starting with token_in (1-based) through pools whose ingest token
    pairs are pairs; None when some pool does not hold the token that reaches it."""
    t, out = int(token_in), []
    for a, b in pairs:
        if t == int(a):
            out.append(True)
            t = int(b)
        elif t == int(b):
            out.append(False)
            t = int(a)
        else:
            return None
    return out


def quote_path(pools, tok1, kind, amount, limit=None, retired=False, execute=False):
    """One path over the pool objects pools (hop order) with sides tok1: (tender [n], received [n],
    status).  execute: the limit decides (None: 0 for exact-in, +inf for exact-out) and a filled
    path runs each hop's transition, changing the pool objects."""
    n = len(pools)
    x, lam = np.zeros(n), np.zeros(n)
    st = FILLED
    if retired:
        st = RETIRED
    elif int(kind) == EXACT_IN:
        v, last = float(amount), 0.0
        for h in range(n):
            last = pools[h].f(v, tok1[h]) if v > 0.0 else 0.0
            x[h], lam[h] = v, last
            v = last if last > 0.0 else 0.0
        if execute and last < (0.0 if limit is None else float(limit)):
            st = LIMIT
    else:
        y = float(amount)
        for h in range(n - 1, -1, -1):
            xh = oo.exact_out(pools[h], y, tok1[h])[0]
            if xh == INF:
                st = UNREACHABLE
                break
            x[h] = xh
            lam[h] = pools[h].f(xh, tok1[h]) if xh > 0.0 else 0.0
            y = xh
        if execute and st == FILLED and y > (INF if limit is None else float(limit)):
            st = LIMIT
    if st != FILLED:
        return np.zeros(n), np.zeros(n), st
    if execute:
        for h in range(n):
            if x[h] > 0.0:
                lam[h] = pools[h].execute(x[h], tok1[h])
    return x, lam, st


def _batch(pools, hop_off, hops, tok1, kind, amount, limit, retired, execute):
    q, H = len(hop_off) - 1, int(hop_off[-1])
    tender, received = np.zeros(H), np.zeros(H)
    status = np.zeros(q, dtype=np.uint8)
    for j in range(q):
        s = slice(int(hop_off[j]), int(hop_off[j + 1]))
        keys = list(hops[s])
        tender[s], received[s], status[j] = quote_path(
            [pools[k] for k in keys], list(tok1[s]), kind[j], amount[j],
            None if limit is None else limit[j], any(k in retired for k in keys), execute)
    return tender, received, status


def quote_paths(pools, hop_off, hops, tok1, kind, amount, retired=()):
    """cfmm_quote_paths on the host: pools maps the hop keys hops [H] to pool objects; tok1 [H] the
    hop sides.  Returns (hop_tender [H], hop_received [H], status [q])."""
    return _batch(pools, hop_off, hops, tok1, kind, amount, None, retired, False)


def replay_paths(pools, hop_off, hops, tok1, kind, amount, limit=None, retired=()):
    """cfmm_execute_paths on the host, in batch order; the pool objects change in place."""
    return _batch(pools, hop_off, hops, tok1, kind, amount, limit, retired, True)
