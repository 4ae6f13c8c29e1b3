"""Host statements of cfmm_quote_limit_orders' rules (include/cfmm_b200.h): a limit row's reachability
and dropped entries, its box per listed token, the start's clamp to that box, the surplus in its
operation order, and the surplus's lower bound.  A limit row's token set, listed tokens and pools are
basket rows' (basket_oracle.row_basket): they do not depend on the amounts or the limits."""
import numpy as np

from basket_oracle import SQRT_EPS, basket_value, row_basket  # noqa: F401  (re-exported)


def row_limit(lists, basket, amounts, limits, i, allowed):
    """(T in local order, the pools, unreachable, dropped, solve).  An entry outside T with a positive
    limit is dropped (paid 0); one with limit 0 follows the basket rule (a positive amount makes the row
    unreachable).  solve: the row runs a solve (reachable, and an entry it keeps has a positive amount)."""
    T, pools, _ = row_basket(lists, basket, [0.0] * len(basket), i, allowed)
    inT = set(T)
    dropped = [int(t) not in inT and c > 0.0 for t, c in zip(basket, limits)]
    kept = [int(t) in inT or c == 0.0 for t, c in zip(basket, limits)]
    unreachable = any(a > 0.0 and int(t) not in inT and c == 0.0 for t, a, c in zip(basket, amounts, limits))
    any_amount = any(a > 0.0 for a, k in zip(amounts, kept) if k)
    return T, pools, unreachable, dropped, any_amount and not unreachable


def box(T, basket, limits):
    """The lower bound of every listed token: 1 + √eps at i (T[0]), fmax(c_k, √eps) at an entry in T
    (one IEEE operation; a zero limit gives √eps, the basket bound), √eps elsewhere."""
    lower = np.full(len(T), SQRT_EPS)
    lower[0] = 1.0 + SQRT_EPS
    loc = {int(t): k for k, t in enumerate(T)}
    for t, c in zip(basket, limits):
        if int(t) in loc:
            lower[loc[int(t)]] = np.fmax(np.float64(c), SQRT_EPS)
    return lower


def ref(T, basket, limits):
    """The primal's reference bound ℓ̂ per listed token: 1 at i, c_k at an entry, 0 elsewhere."""
    r = np.zeros(len(T))
    r[0] = 1.0
    loc = {int(t): k for k, t in enumerate(T)}
    for t, c in zip(basket, limits):
        if int(t) in loc:
            r[loc[int(t)]] = c
    return r


def start_clamp(x, lower):
    """sg_start's last step for a limit row: the breadth-first prices clamped to the row's box."""
    return np.fmax(np.asarray(x, np.float64), lower)


def surplus(received, paid, limits):
    """S = received − Σ_k c_k·paid_k in entry order: the first term received, then each term a multiply
    and a subtract (no fma)."""
    s = np.float64(received)
    for p, c in zip(paid, limits):
        s = s - np.float64(c) * np.float64(p)
    return float(s)


def surplus_floor(T, basket, amounts, limits, nu, psi, rtol):
    """−(|T|·rtol·V + Σ_{t on its bound} (lo_t − c_t)·max(Ψ_t + δ_t, 0)), c_i = 1, c_t = δ_t = 0 off
    the entries, V = Σ_k δ_k·ν_k over the entries in T in local order: the header's lower bound on a
    filled row's surplus."""
    lower, c = box(T, basket, limits), ref(T, basket, limits)
    loc = {int(t): k for k, t in enumerate(T)}
    d = np.zeros(len(T))
    ins = [(loc[int(t)], a) for t, a in zip(basket, amounts) if int(t) in loc]
    for k, a in ins:
        d[k] = a
    V = basket_value([a for _, a in ins], [nu[k] for k, _ in ins])
    on = np.asarray(nu) <= lower
    terms = float(np.sum((lower[on] - c[on]) * np.maximum(np.asarray(psi)[on] + d[on], 0.0)))
    return -(len(T) * rtol * V + terms), V
