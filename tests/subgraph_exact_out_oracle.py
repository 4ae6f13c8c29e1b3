"""Host statements of the exact-out rows of cfmm_quote_subgraph_swap_orders (include/cfmm_b200.h): the
dual's box and linear term, the capacity pre-check, and the bounds the stop m_r <= rtol gives.

A row buys y of i and pays in j.  Its dual minimises −y′·ν_i + Σ_k π_k(ν) with ν_j fixed at 1 and
ν_t >= √eps otherwise, y′ = y·(1 + rtol) rounded up."""
import math

import numpy as np

import solve_certificate as sc
import swap_oracle

SQRT_EPS = sc.SQRT_EPS
DBL_MAX = float(np.finfo(np.float64).max)


def y_prime(y, rtol):
    """y·(1 + rtol) rounded up, as fma(y, rtol, y) toward +inf: the exact value, rounded to nearest,
    then one step up when that lies below it."""
    from fractions import Fraction
    exact = Fraction(y) * Fraction(rtol) + Fraction(y)
    v = float(exact)
    return v if Fraction(v) >= exact else math.nextafter(v, math.inf)


def box(n, i, j, y, rtol):
    """The raw box of an exact-out row over n tokens (i, j 1-based): lin = −y′ at i, ν_j = 1, ν_t >=
    √eps otherwise; the primal's reference ℓ̂ is ℓ except ℓ̂_i = 0."""
    lin = np.zeros(n)
    lin[i - 1] = -y_prime(y, rtol)
    lower = np.full(n, SQRT_EPS)
    upper = np.full(n, np.inf)
    lower[j - 1] = upper[j - 1] = 1.0
    ref = lower.copy()
    ref[i - 1] = 0.0
    return sc.Box(lin, lower, upper, ref)


def pool_capacity(kind, side, R=None, price=None, lt=None, lq=None, g=1.0):
    """What one active pool could ever pay out of its token `side` (0 or 1, ingest order): a two-coin
    pool's reserve; a UniV3 pool's cfmm_quote_swaps output for a tender of DBL_MAX of its other token
    (the walk to the end of its ladder)."""
    if kind in ("product", "geomean"):
        return float(R[side])
    tender = (0.0, DBL_MAX) if side == 0 else (DBL_MAX, 0.0)
    return swap_oracle.univ3_swap(price, lt, lq, g, tender)[0]


def capacity(terms):
    """C_i: the sum of the row's pool capacities in pool order, as the kernel adds them (thread l of
    256 from +0.0 over pools ≡ l mod 256, the xor butterfly in each warp, then the warps in order)."""
    t = [0.0] * 256
    for e, c in enumerate(terms):
        t[e % 256] = float(np.float64(t[e % 256]) + np.float64(c))
    for w in range(8):
        p = t[32 * w:32 * w + 32]
        for m in (16, 8, 4, 2, 1):
            p = [float(np.float64(p[l]) + np.float64(p[l ^ m])) for l in range(32)]
        t[32 * w:32 * w + 32] = p
    s = 0.0
    for w in range(8):
        s = float(np.float64(s) + np.float64(t[32 * w]))
    return s


def unreachable(y, terms, j_in_T=True):
    """The pre-check: j ∉ T or y >= C_i."""
    return (not j_in_T) or y >= capacity(terms)


def stop_bounds(nu, grad, lower, y, i, j, rtol):
    """What m_r = max_t ν_t·|pg_t| / (y·ν_i) <= rtol promises (i, j 0-based slots): (m_r, ok), with pg the
    clipped gradient and pg_j = 0 (ν_j is fixed).  ok: every free token off its bound has
    |grad_t| <= rtol·y·ν_i/ν_t, every token on its bound has grad_t >= −rtol·y·ν_i/ν_t, and
    Σ_t ν_t·|pg_t| <= |T|·rtol·y·ν_i."""
    nu, grad, lower = (np.asarray(x, dtype=np.float64) for x in (nu, grad, lower))
    pg = np.where((nu <= lower) & (grad > 0.0), 0.0, grad)
    pg[j] = 0.0
    scale = y * nu[i]
    m = float(np.max(nu * np.abs(pg)) / scale)
    if m > rtol:
        return m, False
    tol = rtol * scale / nu * (1 + 1e-12)
    free = np.ones(len(nu), bool)
    free[j] = False
    off = free & (nu > lower)
    on = free & ~off
    ok = bool(np.all(np.abs(grad[off]) <= tol[off]) and np.all(grad[on] >= -tol[on])
              and np.sum(nu * np.abs(pg)) <= len(nu) * rtol * scale * (1 + 1e-12))
    return m, ok
