"""Host checks of buy rows (cfmm_quote_basket_swap_orders, include/cfmm_b200.h) and of BasketSwap: the
objective's value, gradient, box and linear term (BasketLiquidation without bought tokens, the exact-out
subgraph box with one bought token and nothing sold); the host route() with BasketSwap over one buy row's
pools under the 50-digit certificate; the local order and what the stop with its per-bought-entry term
promises on random vectors; and the Python argument errors.  No GPU."""
import numpy as np
import pytest

import basket_oracle as bo
import basket_swap_oracle as bs
import solve_certificate as sc
import subgraph_exact_out_oracle as seo


def test_basket_swap_objective(cr):
    n, i = 5, 2
    d_in = np.array([3.0, 0.0, 0.0, 1.5, 0.0])
    # no bought token: BasketLiquidation, box included
    a, b = cr.BasketSwap(i, d_in, np.zeros(n)), cr.BasketLiquidation(i, d_in)
    for fn in ("lower_limit", "upper_limit", "linear_term"):
        assert np.array_equal(getattr(a, fn)(), getattr(b, fn)())
    for v in (np.full(n, 2.0), np.array([1.0, 0.5, 1.0, 1.0, 1.0])):
        assert a.f(v) == b.f(v)
        ga, gb = np.zeros(n), np.zeros(n)
        a.grad(ga, v)
        b.grad(gb, v)
        assert np.array_equal(ga, gb)
    # bought tokens: ν_i fixed at 1, lin = Δin − Δout with lin_i = 0
    d_out = np.array([0.0, 0.0, 4.0, 0.0, 2.0])
    s = cr.BasketSwap(i, d_in, d_out)
    lin = s.linear_term()
    assert np.array_equal(lin, [3.0, 0.0, -4.0, 1.5, -2.0])
    lo, hi = s.lower_limit(), s.upper_limit()
    assert lo[i - 1] == hi[i - 1] == 1.0
    assert np.all(lo[np.arange(n) != i - 1] == sc.SQRT_EPS) and np.all(np.isinf(hi[np.arange(n) != i - 1]))
    v = np.array([0.5, 1.0, 2.0, 0.25, 3.0])
    assert s.f(v) == pytest.approx(float(lin @ v))
    g = np.zeros(n)
    s.grad(g, v)
    assert np.array_equal(g, lin)
    v[i - 1] = 1.5
    assert s.f(v) == np.inf
    s.grad(g, v)
    assert np.all(np.isinf(g))
    with pytest.raises(ValueError):
        cr.BasketSwap(0, d_in, d_out)
    with pytest.raises(ValueError):
        cr.BasketSwap(1, d_in, d_out[:3])


def test_one_buy_no_sells_is_the_exact_out_box(cr):
    """BasketSwap(j, 0, y′ at i) is the exact-out subgraph row's box (buy y of i, pay in j)."""
    n, i, j, y, rtol = 6, 4, 2, 7.25, 1e-4
    yp = np.zeros(n)
    yp[i - 1] = seo.y_prime(y, rtol)
    s = cr.BasketSwap(j, np.zeros(n), yp)
    want = seo.box(n, i, j, y, rtol)
    assert np.array_equal(s.linear_term(), want.lin)
    assert np.array_equal(s.lower_limit(), want.lower) and np.array_equal(s.upper_limit(), want.upper)
    got = bs.box(n, j, np.zeros(n), np.eye(n)[i - 1] * y, rtol)
    assert np.array_equal(got.lin, want.lin) and np.array_equal(got.ref, want.ref)


def lists():
    # tokens 1..7; i = 1
    return {(1, 2): [(0, 0, True)], (1, 3): [(0, 1, True)], (2, 3): [(0, 2, True)], (3, 4): [(0, 3, True)],
            (4, 5): [(0, 4, True)], (6, 7): [(0, 5, True)], (2, 5): [(0, 6, False)]}


def test_local_order():
    allowed = np.zeros(7, bool)
    allowed[[3, 5]] = True                                   # B = {4, 6}
    T, pools, unreach = bs.row_order(lists(), [3, 5, 2], [1.0, 2.0, 3.0], [False, True, True], 1, allowed)
    assert T == [5, 2, 1, 3, 4] and not unreach               # bought in caller order, i, sold, B ∩ T
    assert sorted(k for _, k in pools) == [0, 1, 2, 3, 4, 6]
    # a bought token outside T: unreachable with y > 0, dropped with y = 0
    T, _, unreach = bs.row_order(lists(), [2, 7], [1.0, 2.0], [False, True], 1, allowed)
    assert unreach
    T, _, unreach = bs.row_order(lists(), [2, 7], [1.0, 0.0], [False, True], 1, allowed)
    assert not unreach and T == [1, 2]                       # 3 and 5 are not allowed
    # one bought entry and nothing sold: the exact-out row's order (i, j, B ∩ T), here with j = 1
    T, _, _ = bs.row_order(lists(), [2], [1.0], [True], 1, allowed)
    assert T == [2, 1]


@pytest.mark.parametrize("seed", range(4))
def test_stop_with_buy_term_implies_bought_at_least_y(seed):
    """On random (ν, Ψ) that meet m_r <= rtol, every bought entry with y_l > 0 has Ψ_l >= y_l, and the
    other stated bounds hold; without the buy term a large sale would let Ψ_l fall short of y_l."""
    rng = np.random.default_rng(seed)
    rtol = 1e-4
    n_hit = 0
    for _ in range(400):
        nb, ns, nB = int(rng.integers(1, 4)), int(rng.integers(0, 4)), int(rng.integers(0, 4))
        n = nb + 1 + ns + nB
        amt = np.zeros(n)
        amt[:nb] = rng.uniform(0.5, 10.0, nb)
        amt[nb + 1:nb + 1 + ns] = 10.0 ** rng.uniform(0, 6, ns)
        lin = amt.copy()
        lin[:nb] = [-seo.y_prime(y, rtol) for y in amt[:nb]]
        nu = 10.0 ** rng.uniform(-2, 2, n)
        nu[nb] = 1.0
        nu[rng.random(n) < 0.15] = sc.SQRT_EPS
        nu[nb] = 1.0
        slots = [k for k in range(n) if (k < nb or nb < k <= nb + ns)]
        V = bs.local_sum(amt, nu, slots)
        psi = -lin + rng.uniform(-1, 1, n) * rtol * V / nu * rng.choice([1e-3, 0.5, 1.0, 3.0], n)
        psi[:nb] = -lin[:nb] + rng.uniform(-1, 1, nb) * rtol * amt[:nb] * rng.choice([0.5, 1.0, 2.0], nb)
        m, ok = bs.stop_bounds(nu, lin + psi, nb, amt, slots, nb, rtol)
        if m <= rtol:
            n_hit += 1
            assert ok
            assert np.all(psi[:nb] >= amt[:nb])
    assert n_hit >= 20
    # the second term is what holds the bought entry: one sale far larger than the buy
    nu = np.array([1.0, 1.0, 1.0])
    amt = np.array([1.0, 0.0, 1e6])
    lin = np.array([-seo.y_prime(1.0, rtol), 0.0, 1e6])
    psi = -lin.copy()
    psi[0] = 1.0 - 0.5                                     # short by 0.5 = 5e-7 of V
    m_all, _ = bs.merit(nu, lin + psi, 1, amt, [0, 2], 1)
    assert 0.5 / 1e6 < rtol < m_all


def test_route_with_basket_swap_over_a_rows_pools_certifies(cr):
    """The host route() (its sweeps on the CPU oracle) with BasketSwap(i, Δin, y′) over one buy row's
    pools: the result certifies under the raw box with the header's gap bound, and every bought token
    receives at least y."""
    import order_certificate as oc
    from test_host_logic import OraclePools

    spec = [([900.0, 1000.0], [1, 2]), ([500.0, 520.0], [1, 3]), ([800.0, 790.0], [2, 3]),
            ([700.0, 650.0], [3, 4]), ([600.0, 640.0], [2, 4]), ([300.0, 310.0], [4, 5])]
    cert = [oc.product(R, 0.997, A) for R, A in spec]
    n, i, rtol = 5, 1, 1e-4
    d_in, y = np.zeros(n), np.zeros(n)
    d_in[[1, 4]] = [25.0, 4.0]                               # sell 2 and 5
    y[2] = 6.0                                               # buy 3
    box = bs.box(n, i, d_in, y, rtol)
    yp = np.zeros(n)
    yp[2] = seo.y_prime(y[2], rtol)
    r = cr.Router(cr.BasketSwap(i, d_in, yp), [cr.ProductTwoCoin(R, 0.997, A) for R, A in spec], n,
                  _pools_factory=OraclePools)
    assert np.array_equal(r.objective.linear_term(), box.lin)
    cr.route(r, pgtol=1e-11, factr=1e1)
    res = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
    net = cr.netflows(r)
    V = float(d_in @ r.v + y @ r.v)
    assert abs(res["gap"]) <= n * rtol * V + res["allowance"], res
    assert net[2] >= y[2]
    assert np.all(np.abs(net[[1, 4]] + d_in[[1, 4]]) <= rtol * V / r.v[[1, 4]])   # the sold tokens paid


class _Stub:
    n_tokens = 6
    _world = 1


def test_python_argument_errors(cr):
    basket = cr.DevicePools._basket
    args = ([1], [0, 2], [3, 4], [1.0, 2.0], np.ones(6, bool))
    with pytest.raises(ValueError, match="kind must have 2"):
        basket(_Stub(), False, *args, None, None, [0, 1, 1])
    with pytest.raises(ValueError, match="0 .sold. or 1 .bought."):
        basket(_Stub(), False, *args, None, None, [0, 2])
    for lim in ([np.nan], [np.inf]):
        with pytest.raises(ValueError, match="NaN or \\+inf"):
            basket(_Stub(), True, *args, lim, None, [0, 1])
    with pytest.raises(ValueError, match="limit must have"):
        basket(_Stub(), True, *args, [1.0, 2.0], None, 1)
    sw = cr.Router._swap_basket_args
    _Stub._basket_args = cr.Router._basket_args
    tout, off, toks, amts, kind, _, n_sell = sw(_Stub(), [1, 2], [{2: 1.0}, ([], [])], [{3: 2.0, 4: 0.5}, {5: 1.0}],
                                                np.ones(6, bool), [-np.inf, 0.0], "q")
    assert off.tolist() == [0, 3, 4] and toks.tolist() == [2, 3, 4, 5] and kind.tolist() == [0, 1, 1, 1]
    assert amts.tolist() == [1.0, 2.0, 0.5, 1.0] and n_sell == [1, 0]
    with pytest.raises(ValueError, match="one entry per row"):
        sw(_Stub(), [1], [{2: 1.0}], [{3: 1.0}, {4: 1.0}], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="one amount per token"):
        sw(_Stub(), [1], [([2, 3], [1.0])], [{4: 1.0}], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="allowed"):
        sw(_Stub(), [1], [{2: 1.0}], [{3: 1.0}], None, None, "q")
    s = _Stub()
    s._world = 2
    with pytest.raises(NotImplementedError):
        sw(s, [1], [{2: 1.0}], [{3: 1.0}], np.ones(6, bool), None, "q")
    # sold and bought per row from paid = −Ψ
    out = type("O", (), {})()
    out.paid, out.basket_off = np.array([1.0, -2.5, -0.5, -1.0]), np.array([0, 3, 4])
    sold, bought = cr.Router._sold_bought(out, [1, 0])
    assert [x.tolist() for x in sold] == [[1.0], []] and [x.tolist() for x in bought] == [[2.5, 0.5], [1.0]]
