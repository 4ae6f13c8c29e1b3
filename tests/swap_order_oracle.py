"""Host mirror of cfmm_quote_swaps_exact_out / cfmm_execute_swap_orders (include/cfmm_b200.h), for
the tests: the estimate, the ordinal gallop and bisection, and the in-order replay with limits.
f is the exact-input quote of swap_oracle.py (product_forward, univ3_swap), so for
ProductTwoCoin and UniV3 the mirror gives the device's bits.  GeometricMeanTwoCoin uses numpy's
log1p / expm1 in the device's expression order, which are not CUDA's: its results are close to
the device's, not equal.

  ordinal / from_ordinal   a double >= 0 as its int64 bit pattern, and back
  crossing                 the search of the header, with its evaluation count
  ProductPool / GeoMeanPool / Univ3Pool   f, the estimate and the execute transition of one pool
  exact_out                x* of one pool for a wanted output
  replay_orders            the rows of cfmm_execute_swap_orders in batch order
"""
from __future__ import annotations

import numpy as np

from swap_oracle import F, current_tick, product_forward, univ3_swap, univ3_tick

ORD_MAX = 0x7FEFFFFFFFFFFFFF  # the ordinal of DBL_MAX
INF = float("inf")
EXACT_IN, EXACT_OUT = 0, 1
FILLED, LIMIT, UNREACHABLE, RETIRED = 0, 1, 2, 3


def ordinal(x) -> int:
    return int(np.array(x, dtype=np.float64).view(np.int64))


def from_ordinal(o: int) -> float:
    return float(np.array(o, dtype=np.int64).view(np.float64))


def start_ordinal(e) -> int:
    """The ordinal the search starts from: 1 for a NaN or e <= 0, capped at DBL_MAX."""
    if not (e > 0.0):
        return 1
    return min(ordinal(e), ORD_MAX)


def crossing(f, y, e):
    """(ordinal of x*, number of f evaluations) of the search for y > 0 from the estimate e;
    the ordinal is -1 when f(DBL_MAX) < y."""
    n = 0

    def reaches(o):
        nonlocal n
        n += 1
        return f(from_ordinal(o)) >= y

    o = start_ordinal(e)
    lo, hi = 0, o
    if reaches(o):  # gallop down
        step = 1
        while hi > 1:
            c = hi - step
            if c <= 0:
                break
            if reaches(c):
                hi = c
            else:
                lo = c
                break
            step *= 2
    else:  # gallop up
        lo, step = o, 1
        while True:
            if lo == ORD_MAX:
                return -1, n
            c = ORD_MAX if ORD_MAX - lo <= step else lo + step
            if reaches(c):
                hi = c
                break
            lo = c
            step *= 2
    while hi - lo > 1:
        mid = lo + ((hi - lo) >> 1)
        if reaches(mid):
            hi = mid
        else:
            lo = mid
    return hi, n


def _tender(x, tok1):
    return (x, 0.0) if tok1 else (0.0, x)


class ProductPool:
    """A ProductTwoCoin pool: reserves R in ingest order, fee g."""

    def __init__(self, R, g):
        self.R, self.g = np.array(R, dtype=F), F(g)

    def f(self, x, tok1):
        return product_forward(self.R, self.g, _tender(x, tok1))[1 if tok1 else 0]

    def estimate(self, y, tok1):
        """((R_in·R_out)/(R_out − y) − R_in)/γ, +inf when y >= R_out."""
        with np.errstate(all="ignore"):
            r_in, r_out, y = (self.R[0], self.R[1], F(y)) if tok1 else (self.R[1], self.R[0], F(y))
            if not (y < r_out):
                return INF
            return float(((r_in * r_out) / (r_out - y) - r_in) / self.g)

    def execute(self, x, tok1):
        T = np.array(_tender(x, tok1), dtype=F)
        lam = np.array(product_forward(self.R, self.g, T), dtype=F)
        self.R = (self.R + self.g * T) - lam
        return float(lam[1 if tok1 else 0])


class GeoMeanPool(ProductPool):
    """A GeometricMeanTwoCoin pool (weights w); numpy's log1p / expm1 stand in for CUDA's."""

    def __init__(self, R, g, w):
        super().__init__(R, g)
        self.w = np.array(w, dtype=F)

    def _sides(self, tok1):
        i, o = (0, 1) if tok1 else (1, 0)
        return self.R[i], self.R[o], self.w[i] / self.w[o]

    def f(self, x, tok1):
        with np.errstate(all="ignore"):
            r_in, r_out, eta = self._sides(tok1)
            lam = r_out * -np.expm1(-(eta * np.log1p((self.g * F(x)) / r_in)))
            return float(F(0.0) if lam < 0.0 else (r_out if lam > r_out else lam))

    def estimate(self, y, tok1):
        """(R_in·expm1(−log1p(−(y/R_out))/η))/γ, +inf when y >= R_out."""
        with np.errstate(all="ignore"):
            r_in, r_out, eta = self._sides(tok1)
            y = F(y)
            if not (y < r_out):
                return INF
            return float((r_in * np.expm1(-np.log1p(-(y / r_out)) / eta)) / self.g)

    def execute(self, x, tok1):
        T = np.array(_tender(x, tok1), dtype=F)
        lam = np.zeros(2, dtype=F)
        lam[1 if tok1 else 0] = self.f(x, tok1)
        self.R = (self.R + self.g * T) - lam
        return float(lam[1 if tok1 else 0])


class Univ3Pool:
    """A UniV3 pool: price, ladder (lower_ticks, liquidity), fee g."""

    def __init__(self, price, lower_ticks, liquidity, g):
        self.price, self.g = F(price), F(g)
        self.lt, self.lq = np.asarray(lower_ticks, dtype=F), np.asarray(liquidity, dtype=F)

    def f(self, x, tok1):
        return univ3_swap(self.price, self.lt, self.lq, self.g, _tender(x, tok1))[0]

    def estimate(self, y, tok1):
        """The reverse walk: full ticks add max_amount_pos to s and take R_out off y′; the tick
        with y′ <= R_out gives e = (s + (k/((R_out + β) − y′) − (R_in + α)))/γ."""
        with np.errstate(all="ignore"):
            n, cur = len(self.lt), current_tick(self.lt, self.price)
            s, y = F(0.0), F(y)
            for idx in (range(cur, n + 1) if tok1 else range(cur, 0, -1)):
                k, a, b, r_in, r_out = univ3_tick(self.price, cur, self.lt, self.lq, idx)
                if not tok1:
                    a, b, r_in, r_out = b, a, r_out, r_in
                ra = r_in + a
                if y <= r_out:
                    return float((s + (k / ((r_out + b) - y) - ra)) / self.g)
                mx = k / b - ra if b > 0.0 else (F(np.inf) if a > 0.0 else F(0.0))
                s = s + mx
                y = y - r_out
            return INF

    def execute(self, x, tok1):
        lam, q = univ3_swap(self.price, self.lt, self.lq, self.g, _tender(x, tok1))
        self.price = F(q)
        return lam


def exact_out(pool, y, tok1):
    """(x*, evaluations of f) for a wanted output y >= 0 of the side opposite a token-1 (tok1) or
    token-2 tender; x* = +inf when y cannot be reached."""
    if not (y > 0.0):
        return 0.0, 0
    o, n = crossing(lambda x: pool.f(x, tok1), F(y), pool.estimate(y, tok1))
    return (INF if o < 0 else from_ordinal(o)), n


def quote_exact_out(pool, want, retired=False):
    """The tender row of cfmm_quote_swaps_exact_out for want (0, y) or (y, 0)."""
    tok1 = want[1] > 0.0
    y = want[1] if tok1 else want[0]
    x = INF if (retired and y > 0.0) else exact_out(pool, y, tok1)[0]
    return (x, 0.0) if tok1 else (0.0, x)


def replay_orders(pools, idx, kind, amount, limit=None, retired=()):
    """cfmm_execute_swap_orders on the host: pools is a dict or list of *Pool objects, changed in
    place; rows j = (idx[j], kind[j], amount[j], limit[j]) in batch order.  Returns (paid [q, 2],
    received [q, 2], status [q], evaluations of f per exact-out row [q])."""
    q = len(idx)
    paid, received = np.zeros((q, 2)), np.zeros((q, 2))
    status, evals = np.zeros(q, dtype=np.uint8), np.zeros(q, dtype=np.int64)
    for j in range(q):
        p = pools[idx[j]]
        a1, a2 = float(amount[j][0]), float(amount[j][1])
        out = int(kind[j]) == EXACT_OUT
        lim = float(limit[j]) if limit is not None else (INF if out else 0.0)
        tok1 = a2 > 0.0 if out else a1 > 0.0
        amt = a1 if a1 > 0.0 else a2
        x, lam, st = 0.0, 0.0, FILLED
        if idx[j] in retired:
            st = RETIRED
        elif not out:
            x = amt
            lam = p.f(x, tok1) if x > 0.0 else 0.0
            if lam < lim:
                st = LIMIT
        elif amt > 0.0:
            x, evals[j] = exact_out(p, amt, tok1)
            if x == INF:
                st = UNREACHABLE
            elif x > lim:
                st = LIMIT
        if st == FILLED:
            if x > 0.0:
                lam = p.execute(x, tok1)
        else:
            x = lam = 0.0
        paid[j] = (x, 0.0) if tok1 else (0.0, x)
        received[j] = (0.0, lam) if tok1 else (lam, 0.0)
        status[j] = st
    return paid, received, status, evals
