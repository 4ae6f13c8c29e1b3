"""Host mirror of cfmm_quote_split_orders / cfmm_execute_split_orders (include/cfmm_b200.h), for the
tests.  Each pool's response at s is the CPU oracle's find_arb! (oracle_lib: product_arb,
geomean_arb, univ3_arb), the sums follow the header's warp tree, the search is the header's gallop
and bisection on the ordinals of the doubles in [DBL_MIN, DBL_MAX], and execute applies the
transition of cfmm_apply_trades.  For ProductTwoCoin and UniV3 pools the mirror gives the device's
bits (GeometricMeanTwoCoin: the C library's pow is not CUDA's, so close, not equal).

  Product / GeoMean / Univ3   one pool of a pair: legs at ν, no-trade boundary, transition
  warp_sum                    the fixed summation order of N(s) and O(s)
  split_row                   one row on the current state of its pair's pools (optionally executed)
  quote_split / replay_split  rows on their own / in batch order
"""
from __future__ import annotations

import numpy as np

import oracle_lib
from swap_order_oracle import ORD_MAX, from_ordinal, ordinal

F = np.float64
ORD_MIN = 0x0010000000000000  # the ordinal of DBL_MIN
DBL_MIN = float(np.finfo(np.float64).tiny)
INF = float("inf")
EXACT_IN, EXACT_OUT = 0, 1
FILLED, LIMIT, UNREACHABLE = 0, 1, 2
MAX_EVALS = 1 + 63 + 62 + 1  # search, plus the evaluation at s* that writes the legs
_LANE = np.arange(32)


def warp_sum(terms):
    """Partial l adds terms l, l + 32, … from +0.0; then p_l <- p_l + p_(l xor m), m = 16 … 1."""
    p = np.zeros(32, dtype=F)
    for k, t in enumerate(terms):
        p[k % 32] = p[k % 32] + F(t)
    for m in (16, 8, 4, 2, 1):
        p = p + p[_LANE ^ m]
    return float(p[0])


class _Pool:
    active = True

    def nu(self, ti, s):
        """ν at the pool's tokens (ingest order) for ν_i = 1, ν_j = s."""
        return np.array([1.0 if int(a) == ti else s for a in self.Ai], dtype=F)


class Product(_Pool):
    def __init__(self, R, g, Ai):
        self.R, self.g, self.Ai = np.array(R, dtype=F), F(g), [int(a) for a in Ai]

    def legs(self, v):
        return oracle_lib.load().product_arb(self.R, self.g, v)

    def boundary(self, ti, tj):
        ri, rj = (self.R[0], self.R[1]) if self.Ai[0] == ti else (self.R[1], self.R[0])
        with np.errstate(all="ignore"):
            return float((self.g * ri) / rj)

    def apply(self, D, L, v):
        self.R = (self.R + self.g * D) - L


class GeoMean(Product):
    def __init__(self, R, g, w, Ai):
        super().__init__(R, g, Ai)
        self.w = np.array(w, dtype=F)

    def legs(self, v):
        return oracle_lib.load().geomean_arb(self.R, self.w, self.g, v)

    def boundary(self, ti, tj):
        i = 0 if self.Ai[0] == ti else 1
        with np.errstate(all="ignore"):
            return float(((self.g * self.w[1 - i]) * self.R[i]) / (self.w[i] * self.R[1 - i]))


class Univ3(_Pool):
    def __init__(self, price, lower_ticks, liquidity, g, Ai):
        self.price, self.g, self.Ai = F(price), F(g), [int(a) for a in Ai]
        self.lt, self.lq = np.asarray(lower_ticks, dtype=F), np.asarray(liquidity, dtype=F)

    def legs(self, v):
        return oracle_lib.load().univ3_arb(self.price, self.lt, self.lq, self.g, v)

    def boundary(self, ti, tj):
        return float(self.g * self.price) if self.Ai[0] == tj else float(self.g / self.price)

    def apply(self, D, L, v):
        """cfmm_apply_trades' price rule at ν: p = ν[a]/ν[b]."""
        with np.errstate(all="ignore"):
            q, g, pr = self.price, self.g, F(v[0]) / F(v[1])
            lo = g * q
            if lo <= pr <= q / g:
                return
            target = pr / g if pr < lo else g * pr
            if not (target > 0.0):
                return
            self.price = F(target) if target < self.lt[0] else F(self.lt[0])


def evaluate(pools, ti, tj, s):
    """(N(s), O(s), legs Δ [n, 2], Λ [n, 2]) of the pair's pools at ν_i = 1, ν_j = s."""
    n = len(pools)
    D, L = np.zeros((n, 2)), np.zeros((n, 2))
    tn, to = [], []
    for k, p in enumerate(pools):
        if p.active:
            D[k], L[k] = p.legs(p.nu(ti, s))
        j = 0 if p.Ai[0] == tj else 1
        tn.append(F(D[k, j]) - F(L[k, j]))
        to.append(F(L[k, 1 - j]) - F(D[k, 1 - j]))
    return warp_sum(tn), warp_sum(to), D, L


def split_row(pools, token_in, token_out, kind, amount, limit=None, execute=False):
    """One row over the pair's pools (pair order).  Returns a dict: paid, received, price, status,
    D, L (legs, ingest order; zero unless filled) and evals (evaluations of the pools)."""
    ti, tj, amt, out = int(token_out), int(token_in), float(amount), int(kind) == EXACT_OUT
    n = len(pools)
    res = dict(paid=0.0, received=0.0, price=0.0, status=FILLED, D=np.zeros((n, 2)), L=np.zeros((n, 2)), evals=0)
    if not (amt > 0.0):
        return res
    act = [p for p in pools if p.active]
    if not act:
        res["status"] = UNREACHABLE
        return res
    e = -INF
    for p in act:
        b = p.boundary(ti, tj)
        e = b if b > e else e
    evals = 0
    sums = {}

    def enough(o):
        nonlocal evals
        evals += 1
        N, O, _, _ = evaluate(pools, ti, tj, from_ordinal(o))
        sums[o] = (N, O)
        return O >= amt if out else not (N <= amt)

    o = ORD_MIN if not (e >= DBL_MIN) else min(ordinal(e), ORD_MAX)
    ok = True
    if enough(o):
        lo, step = o, 1
        while True:
            if lo == ORD_MAX:
                ok = False
                break
            c = ORD_MAX if ORD_MAX - lo <= step else lo + step
            if enough(c):
                lo = c
            else:
                hi = c
                break
            step *= 2
    else:
        hi, step = o, 1
        while True:
            if hi == ORD_MIN:
                ok = False
                break
            c = ORD_MIN if hi - ORD_MIN <= step else hi - step
            if enough(c):
                lo = c
                break
            hi = c
            step *= 2
    res["evals"] = evals
    if not ok:
        res["status"] = UNREACHABLE
        return res
    while hi - lo > 1:
        mid = lo + ((hi - lo) >> 1)
        if enough(mid):
            lo = mid
        else:
            hi = mid
    so = lo if out else hi
    s = from_ordinal(so)
    N, O = sums[so]
    res["price"] = s
    if execute and limit is not None and (N > float(limit) if out else O < float(limit)):
        res["status"] = LIMIT
        res["evals"] = evals
        return res
    _, _, D, L = evaluate(pools, ti, tj, s)
    res.update(paid=N, received=O, D=D, L=L, evals=evals + 1)
    if execute:
        for k, p in enumerate(pools):
            if p.active:
                p.apply(D[k], L[k], p.nu(ti, s))
    return res


def _batch(pairs, token_in, token_out, kind, amount, limit, execute):
    """pairs(a, b) -> the pool objects of the pair (pair order)."""
    rows = []
    for r in range(len(token_in)):
        pools = pairs(int(token_in[r]), int(token_out[r]))
        rows.append(split_row(pools, token_in[r], token_out[r], kind[r], amount[r],
                              None if limit is None else limit[r], execute))
    return rows


def quote_split(pairs, token_in, token_out, kind, amount):
    """cfmm_quote_split_orders on the host: every row on the current state on its own."""
    return _batch(pairs, token_in, token_out, kind, amount, None, False)


def replay_split(pairs, token_in, token_out, kind, amount, limit=None):
    """cfmm_execute_split_orders on the host, in batch order; the pool objects change in place."""
    return _batch(pairs, token_in, token_out, kind, amount, limit, True)
