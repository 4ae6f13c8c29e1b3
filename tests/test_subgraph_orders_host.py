"""Host checks of subgraph_oracle: the row token set and pool list on hand-built pair lists (a component
cut off from i, retired pools, j unreachable), the warp-tree sum's shape, and the bounds that the
weighted stop m_r <= rtol gives on synthetic gradients.  No GPU."""
import numpy as np
import pytest

import subgraph_oracle as so


def lists():
    # tokens 1..7; i = 1, j = 2.  {3, 4} connect j to i; {5, 6} only touch each other (cut off from i);
    # {1, 7} holds only a retired pool.
    return {
        (1, 3): [(0, 0, True)],
        (2, 4): [(1, 0, True), (0, 5, False)],
        (3, 4): [(2, 1, True)],
        (5, 6): [(0, 1, True)],
        (1, 7): [(0, 2, False)],
        (2, 7): [(0, 3, True)],
    }


def test_token_set_and_pools():
    allowed = np.ones(7, bool)
    T, pools = so.row_subgraph(lists(), 2, 1, allowed)
    assert T == [1, 2, 3, 4, 7]   # 7 joins through j: {2, 7} is active
    # {1, 7}'s retired pool lies inside T and is listed; {5, 6} is cut off from i and is not
    assert sorted(pools) == sorted([(0, 0), (1, 0), (0, 5), (2, 1), (0, 2), (0, 3)])


def test_cut_off_and_unreachable():
    allowed = np.array([1, 1, 1, 0, 1, 1, 1], bool)   # 4 not allowed: j is cut off from i
    T, pools = so.row_subgraph(lists(), 2, 1, allowed)
    assert T == [1, 3]
    assert pools == [(0, 0)]
    T, _ = so.row_subgraph(lists(), 2, 1, np.zeros(7, bool))
    assert T == [1]


def test_warp_sum_shape():
    x = np.random.default_rng(0).standard_normal(100) * 1e3
    s = so.warp_sum(x)
    assert abs(s - np.sum(x)) <= 1e-9 * np.sum(np.abs(x))
    assert so.warp_sum([]) == 0.0
    assert so.warp_sum([1.5]) == 1.5


@pytest.mark.parametrize("seed", range(6))
def test_weighted_stop_bounds(seed):
    rng = np.random.default_rng(seed)
    n, j, delta, rtol = 12, 1, 5.0, 1e-9
    nu = np.exp(rng.uniform(-3, 3, n))
    lower = np.full(n, so.SQRT_EPS)
    lower[0] = 1 + so.SQRT_EPS
    nu = np.maximum(nu, 1.5 * lower)
    on = rng.random(n) < 0.2
    nu[on] = lower[on]
    # gradients whose weighted projected size is just under rtol: the bounds hold
    g = rng.uniform(-1, 1, n) * rtol * delta * nu[j] / nu * 0.999
    g[on] = np.abs(g[on]) * 1e6   # on the bound and pushing out: clipped, any size
    m, ok = so.stop_bounds(nu, g, lower, delta, j, rtol)
    assert m <= rtol and ok
    # one token's imbalance valued at its price above rtol·δ·ν_j: the stop does not hold
    k = int(np.flatnonzero(~on)[0])
    g[k] = 2 * rtol * delta * nu[j] / nu[k]
    m, ok = so.stop_bounds(nu, g, lower, delta, j, rtol)
    assert m > rtol and not ok


def test_scipy_swap_route_over_a_rows_pools_certifies():
    """route!'s host path (scipy L-BFGS-B) with Swap(i, j, δ) over one row's pools, each evaluation from
    the 50-digit pool responses: the result certifies under Swap's box, and its stop, read as the
    weighted rule, gives the bounds stop_bounds states."""
    from scipy.optimize import minimize

    import order_certificate as oc
    import solve_certificate as sc

    # tokens 1..4; the row sells j = 2 for i = 1 through B = {3, 4}, with pools between 3 and 4
    pools = [oc.product([900.0, 1000.0], 0.997, [1, 2]), oc.product([500.0, 520.0], 0.997, [1, 3]),
             oc.product([800.0, 790.0], 0.997, [2, 3]), oc.product([700.0, 650.0], 0.997, [3, 4]),
             oc.product([600.0, 640.0], 0.997, [2, 4]), oc.product([400.0, 380.0], 1.0, [1, 4], active=False)]
    lists = {}
    for k, p in enumerate(pools):
        a, b = sorted(p.Ai)
        lists.setdefault((a, b), []).append((0, k, p.active))
    T, listed = so.row_subgraph(lists, 2, 1, np.ones(4, bool))
    assert T == [1, 2, 3, 4] and sorted(k for _, k in listed) == list(range(6))
    n, i, j, delta = 4, 1, 2, 25.0
    lin = np.zeros(n)
    lin[j - 1] = delta
    box = sc.basket(i, lin)
    sweep = sc.oracle_sweep(pools, n)
    res = minimize(lambda x: float(box.lin @ x) + sweep(x)[1], np.maximum(np.ones(n), box.lower),
                   jac=lambda x: box.lin + sweep(x)[0], method="L-BFGS-B", bounds=[(lo, None) for lo in box.lower],
                   options=dict(maxcor=5, ftol=0.0, gtol=1e-9, maxiter=2000))
    x = res.x
    D, L = sc.oracle_trades(pools, x)
    psi = sweep(x)[0]
    rtol = 1e-6
    m, ok = so.stop_bounds(x, box.lin + psi, box.lower, delta, j - 1, rtol)
    assert ok, m
    pgtol = float(np.max(m * delta * x[j - 1] / x)) * (1 + 1e-9) + 1e-12
    out = sc.certify(pools, box, x, D, L, pgtol=pgtol, rule="lbfgsb")
    assert out["gap"] <= out["bound"] + out["allowance"]
    assert abs(-psi[j - 1] - delta) <= rtol * delta       # the row paid δ
    assert psi[i - 1] > 0.0                                # and received i


class _Stub:
    n_tokens = 6


@pytest.mark.parametrize("args, match", [
    (([1, 2], [3], [1.0, 1.0], np.ones(6, bool)), "one entry per row"),
    (([1], [3], [1.0], None), "allowed"),
    (([1], [3], [1.0], np.ones(5, bool)), "6 entries"),
])
def test_python_argument_errors(args, match):
    import cfmmrouter_b200 as cr
    with pytest.raises(ValueError, match=match):
        cr.DevicePools._subgraph(_Stub(), False, *args, None, None)
    with pytest.raises(ValueError, match="limit must have"):
        cr.DevicePools._subgraph(_Stub(), True, [1], [3], [1.0], np.ones(6, bool), [1.0, 2.0], None)
