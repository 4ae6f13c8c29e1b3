"""Host statements of cfmm_quote_subgraph_orders' rules (include/cfmm_b200.h): a row's token set T and
pool list, the fixed-order Ψ sums, and the bounds its stop (m_r <= rtol) gives on the gradient.

Pair lists are {(a, b): [(type, index, active), ...]} with a < b, as cfmm_pair_pools lists them."""
import numpy as np

SQRT_EPS = float(np.sqrt(np.finfo(float).eps))


def row_subgraph(lists, j, i, allowed):
    """(T in the call's local order: i, j when j ∈ T, then B ∩ T ascending; the pools of every pair
    inside T as (type, index), in pair order).  B = the allowed tokens other than j and i; T = the
    tokens of {j, i} ∪ B connected to i through active pools between two of them."""
    B = {t for t in range(1, len(allowed) + 1) if allowed[t - 1]} - {j, i}
    V = B | {j, i}
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
    order = [i] + ([j] if j in T else []) + sorted(T - {i, j})
    pools = [(t, k) for (a, b), lst in lists.items() if a in T and b in T for t, k, _ in lst]
    return order, pools


def ingest_tokens(Ai, types, pools):
    """The ingest token pair (1-based) of each (type, index)."""
    return [tuple(int(x) for x in Ai[int(t)][int(k)]) for t, k in zip(types, pools)]


def warp_sum(terms):
    """Split orders' warp tree: partial l adds terms l, l + 32, … from +0.0; then the xor butterfly."""
    p = [0.0] * 32
    for n, x in enumerate(terms):
        p[n % 32] = float(np.float64(p[n % 32]) + np.float64(x))
    for m in (16, 8, 4, 2, 1):
        p = [float(np.float64(p[l]) + np.float64(p[l ^ m])) for l in range(32)]
    return p[0]


def warp_psi(A, D, L, tokens):
    """Ψ_t for each token of the row: Λ_t − Δ_t of the pools holding t, in list order, warp-summed."""
    out = np.zeros(len(tokens))
    for n, t in enumerate(tokens):
        terms = []
        for e, (a, b) in enumerate(A):
            if a == t:
                terms.append(np.float64(L[e][0]) - np.float64(D[e][0]))
            elif b == t:
                terms.append(np.float64(L[e][1]) - np.float64(D[e][1]))
        out[n] = warp_sum(terms)
    return out


def stop_bounds(nu, grad, lower, delta, j, rtol):
    """What m_r = max_t ν_t·|pg_t| / (δ·ν_j) <= rtol promises, for the clipped projected gradient pg
    of the gradient grad = lin + Ψ at ν (lin = δ at j): (m_r, ok) where ok says that every token off
    its bound has |grad_t| <= rtol·δ·ν_j/ν_t, every token on its bound has grad_t >= −rtol·δ·ν_j/ν_t,
    and Σ_t ν_t·|pg_t| <= |T|·rtol·δ·ν_j (the gap's complementary-slackness part)."""
    nu, grad, lower = (np.asarray(x, dtype=np.float64) for x in (nu, grad, lower))
    pg = np.where((nu <= lower) & (grad > 0.0), 0.0, grad)
    scale = delta * nu[j]
    m = float(np.max(nu * np.abs(pg)) / scale)
    if m > rtol:
        return m, False
    tol = rtol * scale / nu * (1 + 1e-12)
    off = nu > lower
    ok = bool(np.all(np.abs(grad[off]) <= tol[off]) and np.all(grad[~off] >= -tol[~off])
              and np.sum(nu * np.abs(pg)) <= len(nu) * rtol * scale * (1 + 1e-12))
    return m, ok
