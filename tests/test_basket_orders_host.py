"""Host checks of basket_oracle: a basket row's token set, listed tokens and pool list on hand-built pair
lists (a positive entry outside T, a zero-amount entry outside T, retired pools), the bounds the stop
m_r <= rtol gives, scipy L-BFGS-B with BasketLiquidation over one row's pools under the 50-digit
certificate, the examples/liquidate.jl market against the host route(), and the Python argument
errors.  No GPU."""
import numpy as np
import pytest

import basket_oracle as bo


def lists():
    # tokens 1..8; i = 1.  {3, 4} connect 2 to 1; {5, 6} only touch each other (cut off from 1);
    # {1, 7} holds only a retired pool; 8 touches nothing.
    return {
        (1, 3): [(0, 0, True)],
        (2, 4): [(1, 0, True), (0, 5, False)],
        (3, 4): [(2, 1, True)],
        (5, 6): [(0, 1, True)],
        (1, 7): [(0, 2, False)],
        (2, 7): [(0, 3, True)],
        (2, 5): [(0, 4, False)],
    }


def test_token_set_listed_tokens_and_pools():
    allowed = np.zeros(8, bool)
    allowed[[2, 3]] = True                       # B = {3, 4}
    T, pools, unreach = bo.row_basket(lists(), [7, 2], [1.0, 2.0], 1, allowed)
    # 2 joins through 4 and 3; 7 through its active pool with 2; the basket keeps the caller's order
    assert T == [1, 7, 2, 3, 4] and not unreach
    # {1, 7}'s retired pool lies inside T and is listed; {2, 5}'s is outside T
    assert sorted(pools) == sorted([(0, 0), (1, 0), (0, 5), (2, 1), (0, 2), (0, 3)])
    # 5 reaches T only through a retired pool: with a positive amount the row is unreachable; with
    # amount 0 it is dropped from the listed tokens
    T, _, unreach = bo.row_basket(lists(), [2, 5], [1.0, 3.0], 1, allowed)
    assert T == [1, 2, 3, 4] and unreach
    T, _, unreach = bo.row_basket(lists(), [2, 5], [1.0, 0.0], 1, allowed)
    assert T == [1, 2, 3, 4] and not unreach
    # an allowed token in the basket is a basket token, not an intermediate
    T, _, _ = bo.row_basket(lists(), [3], [1.0], 1, np.ones(8, bool))
    assert T[:2] == [1, 3] and 8 not in T and 5 not in T


def test_one_entry_basket_is_the_subgraph_row():
    import subgraph_oracle as so
    rng = np.random.default_rng(2)
    for _ in range(20):
        allowed = rng.random(8) < 0.5
        j, i = rng.choice(np.arange(1, 9), size=2, replace=False)
        T, pools, unreach = bo.row_basket(lists(), [int(j)], [1.0], int(i), allowed)
        T2, pools2 = so.row_subgraph(lists(), int(j), int(i), allowed)
        assert T == T2 and pools == pools2 and unreach == (int(j) not in T2)


def test_basket_value_order():
    # the first term alone, then the others in basket order
    assert bo.basket_value([3.0], [0.1]) == float(np.float64(3.0) * np.float64(0.1))
    v = bo.basket_value([1e16, 1.0, -1e16], [1.0, 1.0, 1.0])
    assert v == (1e16 + 1.0) - 1e16


@pytest.mark.parametrize("seed", range(6))
def test_weighted_stop_bounds(seed):
    rng = np.random.default_rng(seed)
    n, K, rtol = 14, 4, 1e-9
    nu = np.exp(rng.uniform(-3, 3, n))
    lower = np.full(n, bo.SQRT_EPS)
    lower[0] = 1 + bo.SQRT_EPS
    nu = np.maximum(nu, 1.5 * lower)
    on = rng.random(n) < 0.2
    on[:K + 1] = False
    nu[on] = lower[on]
    delta = rng.uniform(0.5, 20, K)
    V = bo.basket_value(delta, nu[1:K + 1])
    g = rng.uniform(-1, 1, n) * rtol * V / nu * 0.999
    g[on] = np.abs(g[on]) * 1e6   # on the bound and pushing out: clipped, any size
    m, ok = bo.stop_bounds(nu, g, lower, V, rtol)
    assert m <= rtol and ok
    k = int(np.flatnonzero(~on)[-1])
    g[k] = 2 * rtol * V / nu[k]
    m, ok = bo.stop_bounds(nu, g, lower, V, rtol)
    assert m > rtol and not ok


def test_scipy_basket_route_over_a_rows_pools_certifies():
    """route!'s host path with BasketLiquidation(i, Δin) over one basket row's pools, from 50-digit pool
    responses: the result certifies under the basket's box, and its stop, read as the weighted rule,
    gives the header's bounds (each basket token paid within rtol·V/ν_k, the gap within |T|·rtol·V)."""
    import order_certificate as oc
    import solve_certificate as sc

    # tokens 1..5; the row sells 2, 3 and 5 for 1 through B = {4}
    pools = [oc.product([900.0, 1000.0], 0.997, [1, 2]), oc.product([500.0, 520.0], 0.997, [1, 3]),
             oc.product([800.0, 790.0], 0.997, [2, 3]), oc.product([700.0, 650.0], 0.997, [3, 4]),
             oc.product([600.0, 640.0], 0.997, [2, 4]), oc.product([300.0, 310.0], 0.997, [4, 5]),
             oc.product([400.0, 380.0], 1.0, [1, 4], active=False)]
    lst = {}
    for k, p in enumerate(pools):
        a, b = sorted(p.Ai)
        lst.setdefault((a, b), []).append((0, k, p.active))
    basket, amounts = [2, 3, 5], [25.0, 10.0, 4.0]
    T, listed, unreach = bo.row_basket(lst, basket, amounts, 1, np.array([0, 0, 0, 1, 0], bool))
    assert T == [1, 2, 3, 5, 4] and not unreach and sorted(k for _, k in listed) == list(range(7))
    n = 5
    delta_in = np.zeros(n)
    delta_in[np.array(basket) - 1] = amounts
    x, psi, box = bo.scipy_basket(pools, n, 1, delta_in)
    D, L = sc.oracle_trades(pools, x)
    rtol = 1e-6
    V = bo.basket_value(amounts, x[np.array(basket) - 1])
    m, ok = bo.stop_bounds(x, box.lin + psi, box.lower, V, rtol)
    assert ok, m
    pgtol = float(np.max(m * V / x)) * (1 + 1e-9) + 1e-12
    out = sc.certify(pools, box, x, D, L, pgtol=pgtol, rule="lbfgsb")
    assert out["gap"] <= out["bound"] + out["allowance"]
    assert out["gap"] <= n * rtol * V + out["allowance"] + n * sc.SQRT_EPS * np.max(np.abs(box.lin + psi))
    for t, d in zip(basket, amounts):
        assert abs(-psi[t - 1] - d) <= rtol * V / x[t - 1] * (1 + 1e-9)   # every basket token paid
    assert psi[0] > 0.0                                                   # and token 1 received


@pytest.mark.parametrize("i, delta_in", [(1, [0.0, 10.0, 100.0]), (2, [10.0, 0.0, 0.0])])
def test_liquidate_example_agrees_with_host_route(cr, i, delta_in):
    """examples/liquidate.jl: three ProductTwoCoin pools, the basket [0, 10, 100] into token 1 and the
    one-entry basket [10, 0, 0] into token 2.  The basket row's restatement and the host route() (its
    sweeps on the CPU oracle) both certify, and their dual values agree within the two gaps."""
    import order_certificate as oc
    import solve_certificate as sc
    from test_host_logic import OraclePools

    spec = [([1e3, 1e4], [1, 2]), ([1e3, 1e2], [2, 3]), ([1e3, 2e4], [1, 3])]
    cert = [oc.product(R, 0.997, A) for R, A in spec]
    n = 3
    x, psi, box = bo.scipy_basket(cert, n, i, delta_in)
    D, L = sc.oracle_trades(cert, x)
    a = sc.certify(cert, box, x, D, L, check_stop=False)
    r = cr.Router(cr.BasketLiquidation(i, delta_in), [cr.ProductTwoCoin(R, 0.997, A) for R, A in spec], n,
                  _pools_factory=OraclePools)
    cr.route(r, pgtol=1e-10, factr=1e1)
    b = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
    for res in (a, b):
        assert abs(res["gap"]) <= 1e-6 * abs(res["g50"]) + res["allowance"], res
    slack = abs(a["gap"]) + a["allowance"] + abs(b["gap"]) + b["allowance"] + 1e-9 * abs(a["g50"])
    assert abs(a["g50"] - b["g50"]) <= slack, (a, b)
    net = cr.netflows(r)
    assert net[i - 1] > 0 and abs(net[i - 1] - psi[i - 1]) <= 1e-6 * net[i - 1]
    basket = [t for t in range(n) if delta_in[t] > 0]
    assert np.all(np.abs(net[basket] + np.asarray(delta_in)[basket]) <= 1e-6 * np.asarray(delta_in)[basket])


class _Stub:
    n_tokens = 6
    _world = 1


@pytest.mark.parametrize("args, match", [
    (([1, 2], [0, 1], [3], [1.0], np.ones(6, bool)), "basket_off must have 3"),
    (([1], [0, 2], [3], [1.0], np.ones(6, bool)), "need basket_off"),
    (([1], [0, 1], [3], [1.0], None), "allowed"),
    (([1], [0, 1], [3], [1.0], np.ones(5, bool)), "6 entries"),
])
def test_python_argument_errors(cr, args, match):
    with pytest.raises(ValueError, match=match):
        cr.DevicePools._basket(_Stub(), False, *args, None, None)
    with pytest.raises(ValueError, match="limit must have"):
        cr.DevicePools._basket(_Stub(), True, [1], [0, 1], [3], [1.0], np.ones(6, bool), [1.0, 2.0], None)


def test_router_basket_argument_errors(cr):
    args = cr.Router._basket_args
    tout, off, toks, amts, _ = args(_Stub(), [1, 2], [{2: 1.0, 3: 2.0}, ([4], [0.5])], np.ones(6, bool), None, "q")
    assert off.tolist() == [0, 2, 3] and toks.tolist() == [2, 3, 4] and amts.tolist() == [1.0, 2.0, 0.5]
    with pytest.raises(ValueError, match="one entry per row"):
        args(_Stub(), [1], [{2: 1.0}, {3: 1.0}], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="one amount per token"):
        args(_Stub(), [1], [([2, 3], [1.0])], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="limits must have"):
        args(_Stub(), [1], [{2: 1.0}], np.ones(6, bool), [1.0, 2.0], "q")
    with pytest.raises(ValueError, match="allowed"):
        args(_Stub(), [1], [{2: 1.0}], None, None, "q")
    s = _Stub()
    s._world = 2
    with pytest.raises(NotImplementedError):
        args(s, [1], [{2: 1.0}], np.ones(6, bool), None, "q")
