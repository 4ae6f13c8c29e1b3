"""A restatement of an inventory arbitrage row (cfmm_quote_price_arbitrage_rows, include/cfmm_b200.h) for
the tests: its token set and pool list from its list, its box, P̄, its stop, its profit, and the fill and
gap bounds the header promises.  Shares nothing with the kernels."""
from __future__ import annotations

import numpy as np

import price_arb_oracle as pa
import solve_certificate as sc

BOX = pa.BOX


def row_order(lists, tokens):
    """(T, pools) of one row listing `tokens` (1-based, any order): T the listed tokens (ascending) with
    an active pool to another listed token, whatever their prices; pools every (type, index) of every
    pair inside T.  lists: {(a, b): [(type, index, active)]} for a < b, as cfmm_pair_pools reports them."""
    L = sorted(int(t) for t in tokens)
    T = [t for t in L if any(any(act for _, _, act in lists.get((min(t, u), max(t, u)), ())) for u in L if u != t)]
    pools = [(typ, idx) for a in T for b in T if a < b for typ, idx, _ in lists.get((a, b), ())]
    return T, pools


def local(tokens, values, T):
    """values (aligned with the caller's list `tokens`) in the local order T."""
    at = {int(t): float(v) for t, v in zip(tokens, values)}
    return np.array([at[t] for t in T], dtype=np.float64)


def box(c):
    """The lower bound in local order, c + 1e-8 (one IEEE addition); also ν⁰."""
    return pa.box(c)


def hc(h, c):
    """hᵀc over the held tokens in local order, the first term alone (0.0 when nothing is held)."""
    s, first = 0.0, True
    for a, b in zip(h, c):
        if a > 0.0:
            s = float(a) * float(b) if first else s + float(a) * float(b)
            first = False
    return s


def pbar(nu, psi, h, c):
    """P̄ = G − hᵀc = π(ν) + hᵀ(ν − c), with π(ν) = νᵀΨ (π positively homogeneous)."""
    return float(nu @ psi) + float(h @ (nu - c))


def cbar(prices):
    """c̄: the least positive price of a row's list (every row has one)."""
    p = np.asarray(prices, dtype=np.float64)
    return float(np.min(p[p > 0.0]))


def scale(nu, cb):
    """The stop's per-token scale s_t = max(ν_t, c̄): ν_t wherever c_t > 0 (ν_t > c_t >= c̄)."""
    return np.maximum(nu, cb)


def mx(nu, psi, h, c, cb):
    """max_t s_t·|pg_t|: the gradient h + Ψ, clipped to 0 on the bound where it is > 0."""
    g = h + psi
    pg = np.where((nu <= box(c)) & (g > 0.0), 0.0, g)
    return float(np.max(scale(nu, cb) * np.abs(pg))) if len(nu) else 0.0


def merit(nu, psi, h, c, cb, P):
    """m_r = mx / P̄: 0 when mx = 0, +inf when P̄ <= 0 < mx."""
    m = mx(nu, psi, h, c, cb)
    if not m > 0.0:
        return 0.0
    return m / P if P > 0.0 else np.inf


def profit(c, psi):
    """Σ_t c_t·Ψ_t in local order, the first term alone."""
    return pa.profit(c, psi)


def eps(P, rtol, atol):
    """ε = max(rtol·P̄, atol): the bound on s_t·|pg_t| at a stop."""
    return max(rtol * max(P, 0.0), atol)


def fill_floor(nu, h, e, cb):
    """The least net the fill promise allows each token: −h_t − ε/max(ν_t, c̄), so no token is
    overdrawn by more than ε/c̄ units."""
    return -h - e / scale(nu, cb)


def gap_bound(nu, psi, h, c, e):
    """The header's bound on P̄ − cᵀΨ: |T|·ε plus 1e-8·(Ψ_t + h_t) for each token on its bound."""
    on = nu <= box(c)
    return len(nu) * e + float(np.sum((nu[on] - c[on]) * np.maximum(psi[on] + h[on], 0.0)))


def cert_box(c, h):
    """The 50-digit certificate's box of LinearHoldings(c, h): lin h, lower c + 1e-8, reference c."""
    c = np.asarray(c, dtype=np.float64)
    return sc.Box(np.asarray(h, dtype=np.float64), c + BOX, ref=c)


def product_sold(R, gamma, ca, cb, h):
    """One ProductTwoCoin pool (R_a, R_b, γ) at prices (c_a, c_b), holding h of a: the row sells
    min(h, x*) of a, x* the reference's find_arb! amount at ν = c (prod_arb_δ(c_b/c_a, R_a, k, γ))."""
    k = R[0] * R[1]
    x = max(np.sqrt(gamma * (cb / ca) * k) - R[0], 0.0) / gamma
    return min(h, x)
