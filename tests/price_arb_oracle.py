"""A restatement of a price arbitrage row (cfmm_quote_price_arbitrage, include/cfmm_b200.h) for the tests:
its token set and pool list, its box and start, its stop and its profit, in the kernel's operation order
where the kernel's bits are compared.  Shares nothing with the kernels."""
from __future__ import annotations

import numpy as np

import solve_certificate as sc

BOX = 1e-8  # LinearNonnegative's lower limit c + 1e-8 (objectives.jl:78)


def row_order(lists, allowed, price_row):
    """(T, pools) of one row: T the priced allowed tokens (1-based, ascending) with an active pool to
    another priced token; pools every (type, index) of every pair inside T.  lists: {(a, b): [(type,
    index, active)]} for a < b, as cfmm_pair_pools reports them."""
    A = (np.flatnonzero(np.asarray(allowed, bool)) + 1).tolist()
    priced = [t for t, c in zip(A, price_row) if c > 0.0]
    T = [t for t in priced if any(any(act for _, _, act in lists.get((min(t, u), max(t, u)), ()))
                                  for u in priced if u != t)]
    pools = [(typ, idx) for a in T for b in T if a < b for typ, idx, _ in lists.get((a, b), ())]
    return T, pools


def box(c):
    """The row's lower bound in local order: c + 1e-8, one IEEE addition per token; also ν⁰."""
    return np.asarray(c, dtype=np.float64) + BOX


def merit(nu, psi, lower, g):
    """m_r = max_t ν_t·|pg_t| / g, pg = Ψ clipped at the lower bound (0 where ν_t <= ℓ_t and Ψ_t > 0);
    0 when that max is 0, +inf when it is not and g <= 0."""
    pg = np.where((nu <= lower) & (psi > 0.0), 0.0, psi)
    mx = float(np.max(nu * np.abs(pg))) if len(nu) else 0.0
    if not mx > 0.0:
        return 0.0
    return mx / g if g > 0.0 else np.inf


def profit(c, psi):
    """Σ_t c_t·Ψ_t in local order: the first term alone, then one IEEE addition per term."""
    if len(c) == 0:
        return 0.0
    s = float(c[0]) * float(psi[0])
    for a, b in zip(c[1:], psi[1:]):
        s = s + float(a) * float(b)
    return s


def gap_bound(nu, psi, c, rtol, g):
    """The header's bound on g − cᵀΨ: |T|·rtol·g plus 1e-8·max(Ψ_t, 0) for each token on its bound."""
    on = nu <= box(c)
    return len(nu) * rtol * g + float(np.sum((nu[on] - c[on]) * np.maximum(psi[on], 0.0)))


def certify(cert, n, toks, c, nu_r, D, L, merit_r, g):
    """solve_certificate.certify of a row under LinearNonnegative(c) over its pools (cert: the pools in
    the order of D, L), in an n-token space where the tokens outside the row sit at ν = 1 with price
    1 and hold no pool.  pgtol is the per-token tolerance m_r <= rtol gives: max_t m_r·g/ν_t."""
    full_c, nu = np.ones(n), np.ones(n) + BOX
    full_c[toks - 1] = c
    nu[toks - 1] = nu_r
    pgtol = float(np.max(merit_r * g / nu_r)) * (1 + 1e-9) if len(nu_r) else 0.0
    return sc.certify(cert, sc.linear_nonnegative(full_c), nu, D, L, pgtol=max(pgtol, 1e-300))
