"""Host statements of cfmm_quote_basket_orders' rules (include/cfmm_b200.h): a row's token set T, its
listed tokens and pool list, whether it is reachable, and the bounds its stop (m_r <= rtol) gives.
The Ψ sums and the ingest tokens are subgraph orders' (subgraph_oracle).

Pair lists are {(a, b): [(type, index, active), ...]} with a < b, as cfmm_pair_pools lists them."""
import numpy as np

from subgraph_oracle import SQRT_EPS, ingest_tokens, warp_psi, warp_sum  # noqa: F401  (re-exported)


def row_basket(lists, basket, amounts, i, allowed):
    """(T in the row's local order: i, the basket tokens in T in basket order, then B ∩ T ascending;
    the pools of every pair inside T as (type, index), in pair order; unreachable: an entry with a
    positive amount lies outside T).  B = the allowed tokens other than i and the basket."""
    Bk = [int(t) for t in basket]
    B = {t for t in range(1, len(allowed) + 1) if allowed[t - 1]} - set(Bk) - {i}
    V = B | set(Bk) | {i}
    adj = {t: set() for t in V}
    for (a, b), pools in lists.items():
        if a in V and b in V and any(act for _, _, act in pools):
            adj[a].add(b)
            adj[b].add(a)
    T, todo = {i}, [i]
    while todo:
        u = todo.pop()
        for w in adj[u] - T:
            T.add(w)
            todo.append(w)
    order = [i] + [t for t in Bk if t in T] + sorted(T - {i} - set(Bk))
    pools = [(t, k) for (a, b), lst in lists.items() if a in T and b in T for t, k, _ in lst]
    unreachable = any(a > 0 and t not in T for t, a in zip(Bk, amounts))
    return order, pools, unreachable


def basket_value(lin_b, nu_b):
    """V = Σ_k δ_k·ν_k in basket order, the first term alone (fp64, as the kernel adds it)."""
    s = np.float64(lin_b[0]) * np.float64(nu_b[0])
    for d, v in zip(lin_b[1:], nu_b[1:]):
        s = s + np.float64(d) * np.float64(v)
    return float(s)


def stop_bounds(nu, grad, lower, V, rtol):
    """What m_r = max_t ν_t·|pg_t| / V <= rtol promises, for the clipped projected gradient pg of
    grad = lin + Ψ at ν (V = Σ_k δ_k·ν_k): (m_r, ok) where ok says that every token off its bound
    has |grad_t| <= rtol·V/ν_t (a basket token is paid within rtol·V/ν_k of δ_k), every token on its
    bound has grad_t >= −rtol·V/ν_t (an intermediate's net is at least that), and
    Σ_t ν_t·|pg_t| <= |T|·rtol·V (the gap's complementary-slackness part)."""
    nu, grad, lower = (np.asarray(x, dtype=np.float64) for x in (nu, grad, lower))
    pg = np.where((nu <= lower) & (grad > 0.0), 0.0, grad)
    m = float(np.max(nu * np.abs(pg)) / V)
    if m > rtol:
        return m, False
    tol = rtol * V / nu * (1 + 1e-12)
    off = nu > lower
    ok = bool(np.all(np.abs(grad[off]) <= tol[off]) and np.all(grad[~off] >= -tol[~off])
              and np.sum(nu * np.abs(pg)) <= len(nu) * rtol * V * (1 + 1e-12))
    return m, ok


def scipy_basket(pools, n, i, delta_in, gtol=1e-10):
    """route!'s host path (scipy L-BFGS-B, m = 5) with BasketLiquidation(i, Δin) over `pools`
    (order_certificate pools), each evaluation from the 50-digit responses.  Returns (ν, Ψ, box)."""
    from scipy.optimize import minimize

    import solve_certificate as sc

    box = sc.basket(i, delta_in)
    sweep = sc.oracle_sweep(pools, n)
    res = minimize(lambda x: float(box.lin @ x) + sweep(x)[1], np.maximum(np.ones(n), box.lower),
                   jac=lambda x: box.lin + sweep(x)[0], method="L-BFGS-B", bounds=[(lo, None) for lo in box.lower],
                   options=dict(maxcor=5, ftol=0.0, gtol=gtol, maxiter=2000))
    return res.x, sweep(res.x)[0], box
