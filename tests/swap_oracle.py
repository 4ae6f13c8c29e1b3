"""Host restatements of the swap rules of cfmm_quote_swaps / cfmm_execute_swaps
(include/cfmm_b200.h), for the tests: one IEEE double operation per step, in the reference's
order (src/cfmms.jl:401-449), so that the results are the device's bits.  numpy float64 scalars
never fuse a*b+c, and np.sqrt is correctly rounded.

  product_forward   forward_amount of the BoundedProduct (R₁R₂, 0, 0, R₁, R₂)
  univ3_swap        forward_trade of a UniV3 pool and the price q′ the pool moves to
  geomean_truth     the GeometricMeanTwoCoin amount out in 50-digit arithmetic (mpmath)
"""
from __future__ import annotations

import numpy as np

F = np.float64


def product_forward(R, gamma, tender):
    """(λ₁, λ₂) of ProductTwoCoin reserves R for the tender (x₁, x₂), at most one side > 0."""
    with np.errstate(all="ignore"):
        r1, r2, g = F(R[0]), F(R[1]), F(gamma)
        x1, x2 = F(tender[0]), F(tender[1])
        if x1 > 0.0:
            return 0.0, float(_product_out(r1, r2, g * x1))
        if x2 > 0.0:
            return float(_product_out(r2, r1, g * x2)), 0.0
        return 0.0, 0.0


def _product_out(r_in, r_out, d):
    k = r_in * r_out
    lam = (r_out + F(0.0)) - k / ((r_in + F(0.0)) + d)  # forward_amount with α = β = 0 (the + 0 are exact)
    return r_out if r_out < lam else lam


def current_tick(lower_ticks, price):
    """searchsortedlast(lower_ticks, price, rev=true) (src/cfmms.jl:235)."""
    return int(np.sum(np.asarray(lower_ticks, dtype=F) >= F(price)))


def univ3_tick(price, cur, lower_ticks, liquidity, idx):
    """compute_at_tick (src/cfmms.jl:294-313), idx 1-based: (k, α, β, R₁, R₂)."""
    n = len(lower_ticks)
    k = F(liquidity[idx - 1])
    pplus = F(lower_ticks[idx - 1])
    pminus = F(lower_ticks[idx]) if idx < n else F(0.0)
    alpha = np.sqrt(k / pplus)
    beta = np.sqrt(k * pminus)
    p = pplus if idx > cur else (pminus if idx < cur else F(price))
    return k, alpha, beta, np.sqrt(k / p) - alpha, np.sqrt(k * p) - beta


def univ3_swap(price, lower_ticks, liquidity, gamma, tender, end_tick=False):
    """(λ, q′): forward_trade(Δ, cfmm) (src/cfmms.jl:436-449) of a UniV3 pool at `price`, and the
    price the pool moves to by the rule of cfmm_execute_swaps.  λ is received on the side
    opposite the tender.  end_tick: also the tick the walk ended inside (1-based; 0 when it
    exhausted every tick it reached or did not walk)."""
    out = _univ3_swap(price, lower_ticks, liquidity, gamma, tender)
    return out if end_tick else out[:2]


def _univ3_swap(price, lower_ticks, liquidity, gamma, tender):
    with np.errstate(all="ignore"):
        lt = np.asarray(lower_ticks, dtype=F)
        n = len(lt)
        price = F(price)
        x1, x2 = F(tender[0]), F(tender[1])
        if not (x1 > 0.0 or x2 > 0.0):
            return 0.0, float(price), 0
        tok1 = x1 > 0.0
        d = F(gamma) * (x1 if tok1 else x2)
        cur = current_tick(lt, price)
        lam, last = F(0.0), 0
        idxs = range(cur, n + 1) if tok1 else range(cur, 0, -1)
        for idx in idxs:
            k, alpha, beta, R1, R2 = univ3_tick(price, cur, lt, liquidity, idx)
            if not tok1:  # flip_sides, src/cfmms.jl:289
                alpha, beta, R1, R2 = beta, alpha, R2, R1
            hi, lo = lt[idx - 1], (lt[idx] if idx < n else F(0.0))
            if beta > 0.0:  # max_amount_pos, src/cfmms.jl:401-409
                mx = k / beta - (R1 + alpha)
            elif alpha > 0.0:
                mx = F(np.inf)
            else:
                mx = F(0.0)
            if mx > d:
                y = (R1 + alpha) + d
                out = (R2 + beta) - k / y
                lam = lam + (R2 if R2 < out else out)
                q = (k / y) / y if tok1 else (y / k) * y
                q = lo if q < lo else (hi if q > hi else q)
                return float(lam), float(q), idx
            lam = lam + R2
            d = d - mx
            if k != 0.0:
                last = idx
        if last == 0:
            return float(lam), float(price), 0
        if tok1:
            return float(lam), float(lt[last] if last < n else 0.0), 0
        return float(lam), float(lt[last - 1]), 0


def geomean_truth(R, w, gamma, tender, dps=50):
    """(λ₁, λ₂) of a GeometricMeanTwoCoin pool in dps-digit arithmetic: λ_out =
    R_out·(1 − (R_in/(R_in + δ))^(w_in/w_out)) with δ = γ·x rounded to double, as the device forms it."""
    import mpmath as mp
    with mp.workdps(dps):
        x1, x2 = float(tender[0]), float(tender[1])
        if x1 > 0.0:
            i, o, x = 0, 1, x1
        elif x2 > 0.0:
            i, o, x = 1, 0, x2
        else:
            return 0.0, 0.0
        d = mp.mpf(float(F(gamma) * F(x)))
        eta = mp.mpf(float(w[i])) / mp.mpf(float(w[o]))
        rin, rout = mp.mpf(float(R[i])), mp.mpf(float(R[o]))
        lam = rout * (1 - (rin / (rin + d)) ** eta)
        out = [0.0, 0.0]
        out[o] = lam
        return out[0], out[1]
