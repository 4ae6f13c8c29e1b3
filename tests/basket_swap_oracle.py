"""Host statements of the buy rows of cfmm_quote_basket_swap_orders (include/cfmm_b200.h): a row's local
token order, its dual's box and linear term, the stop m_r with its per-bought-entry term, and the bounds
that stop gives.

A buy row settles in i and has sold entries (sell up to δ_k of b_k) and bought entries (buy y_l of b_l,
at least one).  Its dual minimises Σ_k δ_k·ν_k − Σ_l y′_l·ν_l + Σ_p π_p(ν) with ν_i fixed at 1 and
ν_t >= √eps otherwise, y′ = y·(1 + rtol) rounded up."""
import numpy as np

import basket_oracle as bo
import solve_certificate as sc
from subgraph_exact_out_oracle import y_prime

SQRT_EPS = sc.SQRT_EPS


def row_order(lists, tokens, amounts, bought, i, allowed):
    """basket_oracle.row_basket with the buy row's local order: the bought entries in T in the caller's
    order, then i, then the sold entries in T in the caller's order, then B ∩ T ascending."""
    T, pools, unreach = bo.row_basket(lists, tokens, amounts, i, allowed)
    inT = set(T)
    ent = [int(t) for t in tokens]
    buy = [t for t, b in zip(ent, bought) if b and t in inT]
    sell = [t for t, b in zip(ent, bought) if not b and t in inT]
    return buy + [i] + sell + [t for t in T if t not in set(ent) | {i}], pools, unreach


def entry_terms(toks, tokens, amounts, bought, rtol):
    """For the listed tokens toks (local order): lin (δ at sold, −y′ at bought entries, 0 elsewhere)
    and amt (δ or y at entries, 0 elsewhere), and the local slots of the entries in local order."""
    loc = {int(t): k for k, t in enumerate(toks)}
    lin, amt = np.zeros(len(toks)), np.zeros(len(toks))
    for t, a, b in zip(tokens, amounts, bought):
        if int(t) in loc:
            lin[loc[int(t)]] = -y_prime(float(a), rtol) if b else float(a)
            amt[loc[int(t)]] = float(a)
    slots = sorted(loc[int(t)] for t in tokens if int(t) in loc)
    return lin, amt, slots


def local_sum(c, nu, slots):
    """Σ c_e·ν_e over the entries in local order, the first term alone (fp64, as the kernel adds it)."""
    return bo.basket_value([c[s] for s in slots], [nu[s] for s in slots])


def merit(nu, grad, root, amt, slots, n_buy):
    """m_r of a buy row: max(max_t ν_t·|pg_t| / V, max over bought slots l < n_buy with y_l > 0 of
    ν_l·|pg_l| / (y_l·ν_l)); pg is the clipped gradient with pg_root = 0 (ν_i fixed).  Returns (m_r, pg)."""
    nu, grad = np.asarray(nu, np.float64), np.asarray(grad, np.float64)
    pg = np.where((nu <= SQRT_EPS) & (grad > 0.0), 0.0, grad)
    pg[root] = 0.0
    V = local_sum(amt, nu, slots)
    m = float(np.max(nu * np.abs(pg)) / V)
    for l in range(n_buy):
        if amt[l] > 0.0:
            m = max(m, float((nu[l] * abs(pg[l])) / (amt[l] * nu[l])))
    return m, pg


def stop_bounds(nu, grad, root, amt, slots, n_buy, rtol):
    """What m_r <= rtol promises: (m_r, ok), ok when every free token off its bound has
    |grad_t| <= rtol·V/ν_t, every token on its bound grad_t >= −rtol·V/ν_t, every bought entry with
    y_l > 0 |grad_l| <= rtol·y_l (so Ψ_l >= y′_l − rtol·y_l >= y_l), and Σ ν_t·|pg_t| <= |T|·rtol·V."""
    nu, grad = np.asarray(nu, np.float64), np.asarray(grad, np.float64)
    m, pg = merit(nu, grad, root, amt, slots, n_buy)
    if m > rtol:
        return m, False
    V = local_sum(amt, nu, slots)
    tol = rtol * V / nu * (1 + 1e-12)
    free = np.ones(len(nu), bool)
    free[root] = False
    off = free & (nu > SQRT_EPS)
    on = free & ~off
    ok = bool(np.all(np.abs(grad[off]) <= tol[off]) and np.all(grad[on] >= -tol[on])
              and np.sum(nu * np.abs(pg)) <= len(nu) * rtol * V * (1 + 1e-12))
    for l in range(n_buy):
        if amt[l] > 0.0 and nu[l] > SQRT_EPS:
            ok = ok and abs(grad[l]) <= rtol * amt[l] * (1 + 1e-12)
    return m, ok


def box(n, i, delta_in, y_out, rtol):
    """The raw box of a buy row over n tokens (i 1-based; delta_in, y_out per token): lin = Δin − y′,
    ν_i = 1, ν_t >= √eps otherwise; the primal's reference ℓ̂ is ℓ except ℓ̂_t = 0 at bought tokens."""
    lin = np.asarray(delta_in, np.float64).copy()
    ref = np.full(n, SQRT_EPS)
    for t in range(n):
        if y_out[t] > 0.0:
            lin[t] -= y_prime(float(y_out[t]), rtol)
            ref[t] = 0.0
    lin[i - 1] = 0.0
    lower = np.full(n, SQRT_EPS)
    upper = np.full(n, np.inf)
    lower[i - 1] = upper[i - 1] = ref[i - 1] = 1.0
    return sc.Box(lin, lower, upper, ref)
