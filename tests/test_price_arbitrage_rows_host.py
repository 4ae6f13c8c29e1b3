"""Host checks of inventory arbitrage rows (cfmm_quote_price_arbitrage_rows, include/cfmm_b200.h): the
objective LinearHoldings (its conjugate, gradient and box, and its special cases LinearNonnegative,
BasketLiquidation and LimitBasket), the row's token set and pool list, the one-pool closed form, the host
route() with LinearHoldings over small random markets under the fill promise and the 50-digit
certificate, and the Python argument errors.  No GPU."""
import numpy as np
import pytest

import price_arb_rows_oracle as ia
import solve_certificate as sc

SQRT_EPS = float(np.sqrt(np.finfo(float).eps))


@pytest.mark.parametrize("seed", range(4))
def test_conjugate_gradient_and_box(cr, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 12))
    c = np.where(rng.random(n) < 0.2, 0.0, rng.uniform(0.1, 10.0, n))
    h = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(0.0, 5.0, n))
    o = cr.LinearHoldings(c, h)
    assert np.array_equal(o.lower_limit(), c + 1e-8) and np.all(np.isinf(o.upper_limit()))
    assert np.array_equal(o.linear_term(), h)
    nu = c + rng.uniform(0.0, 3.0, n)
    # f = sup_{Ψ >= −h} (c − ν)ᵀΨ = hᵀ(ν − c) on ν >= c
    assert o.f(nu) == pytest.approx(float(h @ (nu - c)), rel=1e-12, abs=1e-12)
    assert o.f(nu) == float(np.dot(h, nu)) - o._const()
    g = np.zeros(n)
    o.grad(g, nu)
    assert np.array_equal(g, h)
    # a finite difference of f along a direction that stays in the box
    d = rng.uniform(0.0, 1.0, n)
    assert (o.f(nu + 1e-3 * d) - o.f(nu)) / 1e-3 == pytest.approx(float(h @ d), rel=1e-6, abs=1e-9)
    below = nu.copy()
    below[0] = c[0] - 1.0
    assert o.f(below) == np.inf
    o.grad(g, below)
    assert np.all(np.isinf(g))


def test_special_cases(cr):
    c = np.array([2.0, 0.5, 1.5, 3.0])
    # h = 0: LinearNonnegative(c), box bit for bit, f = 0
    o, ln = cr.LinearHoldings(c, np.zeros(4)), cr.LinearNonnegative(c)
    nu = c + 0.25
    assert np.array_equal(o.lower_limit(), ln.lower_limit())
    assert np.array_equal(o.linear_term(), ln.linear_term())
    assert o.f(nu) == ln.f(nu) == 0.0
    # c = e_i, h = Δin: BasketLiquidation(i, Δin) up to the box (ν_i >= 1 + 1e-8, ν_t >= 1e-8 against
    # 1 + √eps and √eps)
    i, din = 2, np.array([3.0, 0.0, 1.0, 4.0])
    e = np.zeros(4)
    e[i - 1] = 1.0
    o, bl = cr.LinearHoldings(e, din), cr.BasketLiquidation(i, din)
    assert np.array_equal(o.linear_term(), bl.linear_term())
    nu = np.array([0.7, 1.3, 2.0, 0.1])
    assert o.f(nu) == pytest.approx(bl.f(nu), rel=1e-15)
    assert np.array_equal(o.lower_limit(), e + 1e-8)
    assert np.allclose(o.lower_limit(), bl.lower_limit(), rtol=0, atol=SQRT_EPS)
    # c = (1 at i, limit_k at each sold k), h = Δin: LimitBasket up to the box
    lim = np.array([0.4, 0.0, 2.5, 0.9])
    cc = lim.copy()
    cc[i - 1] = 1.0
    o, lb = cr.LinearHoldings(cc, din), cr.LimitBasket(i, din, lim)
    nu = np.maximum(cc, lb.lower_limit()) + np.array([0.1, 0.2, 0.3, 0.4])
    assert np.array_equal(o.linear_term(), lb.linear_term())
    assert o.f(nu) == pytest.approx(lb.f(nu), rel=1e-12, abs=1e-12)
    assert np.allclose(o.lower_limit(), lb.lower_limit(), rtol=0, atol=SQRT_EPS)
    with pytest.raises(ValueError):
        cr.LinearHoldings([1.0, -1.0], [0.0, 0.0])
    with pytest.raises(ValueError):
        cr.LinearHoldings([1.0, 1.0], [0.0, np.nan])
    with pytest.raises(ValueError):
        cr.LinearHoldings([1.0, 1.0], [0.0])


def test_row_order_keeps_zero_prices_and_sorts_the_list():
    lists = {(1, 2): [(0, 0, True), (2, 3, False)], (2, 3): [(1, 1, False)], (5, 6): [(0, 5, True)],
             (3, 5): [(0, 7, True)], (1, 4): [(0, 9, True)]}
    T, pools = ia.row_order(lists, [6, 3, 1, 2, 5])
    assert T == [1, 2, 3, 5, 6]
    assert sorted(pools) == sorted([(0, 0), (2, 3), (1, 1), (0, 5), (0, 7)])
    # a retired pair alone does not make a token part of T
    T, _ = ia.row_order(lists, [3, 2])
    assert T == []
    assert ia.local([6, 3, 1], [60.0, 30.0, 10.0], [1, 3, 6]).tolist() == [10.0, 30.0, 60.0]
    # hᵀc over the held tokens only, the first term alone
    assert ia.hc([0.0, 2.0, 3.0], [5.0, 7.0, 11.0]) == 2.0 * 7.0 + 3.0 * 11.0
    assert ia.hc([0.0, 0.0], [1.0, 1.0]) == 0.0


def _route(cr, spec, n, c, h, gamma=0.997):
    from test_host_logic import OraclePools
    r = cr.Router(cr.LinearHoldings(c, h), [cr.ProductTwoCoin(R, gamma, A) for R, A in spec], n,
                  _pools_factory=OraclePools)
    cr.route(r, pgtol=1e-11, factr=1e1)
    return r, cr.netflows(r)


@pytest.mark.parametrize("h", [0.0, 1.0, 5.0, 1e6])
def test_one_pool_closed_form(cr, h):
    """A tree of one pool at prices c: the row sells min(h, x*) of the held token a, x* find_arb!'s
    amount at ν = c; with h = 0 nothing trades."""
    R, ca, cb = (1000.0, 1000.0), 1.0, 1.02
    r, net = _route(cr, [(list(R), [1, 2])], 2, np.array([ca, cb]), np.array([h, 0.0]))
    want = ia.product_sold(R, 0.997, ca, cb, h)
    assert -net[0] == pytest.approx(want, rel=1e-5, abs=1e-6)
    assert net[1] >= -1e-9


@pytest.mark.parametrize("seed", range(4))
def test_route_meets_the_fill_promise_and_certifies(cr, seed):
    import order_certificate as oc
    rng = np.random.default_rng(seed)
    n = 6
    edges = [(1, 2), (1, 3), (2, 3), (3, 4), (2, 4), (4, 5), (5, 6)]
    spec = [(list(rng.uniform(300.0, 1000.0, 2)), list(e)) for e in edges]
    nu0 = rng.uniform(0.8, 1.2, n)
    c = np.where(rng.random(n) < 0.2, 0.0, nu0 * rng.uniform(0.97, 1.03, n))
    c[0] = max(c[0], 0.5)
    h = np.where(rng.random(n) < 0.5, rng.uniform(0.0, 20.0, n), 0.0)
    r, net = _route(cr, spec, n, c, h)
    cert = [oc.product(R, 0.997, A) for R, A in spec]
    res = sc.certify(cert, ia.cert_box(c, h), r.v, r.Δs, r.Λs, check_stop=False)
    P = ia.pbar(r.v, net, h, c)
    assert P >= -1e-9
    e = ia.eps(P, 1e-6, 1e-9)
    assert np.all(net >= ia.fill_floor(r.v, h, e, ia.cbar(c)) - 1e-6)
    assert P - ia.profit(c, net) <= ia.gap_bound(r.v, net, h, c, e) + abs(res["gap"]) + res["allowance"] + 1e-6


class _Stub:
    n_tokens = 6
    _world = 1


def test_python_argument_errors(cr):
    f = cr.DevicePools._price_arb_rows
    off, tok, pr = [0, 2, 3], [1, 2, 4], [1.0, 0.0, 2.0]
    with pytest.raises(ValueError, match="allow_off"):
        f(_Stub(), False, [1, 2], tok, pr, None, None, None)
    with pytest.raises(ValueError, match="allow_off"):
        f(_Stub(), False, [0, 2, 1], tok, pr, None, None, None)
    with pytest.raises(ValueError, match="1 to 258"):
        f(_Stub(), False, [0, 3, 3], tok, pr, None, None, None)
    with pytest.raises(ValueError, match="one entry per listed token"):
        f(_Stub(), False, off, tok, pr[:2], None, None, None)
    for bad in (-1.0, np.nan, np.inf):
        with pytest.raises(ValueError, match="price is negative"):
            f(_Stub(), False, off, tok, [1.0, bad, 1.0], None, None, None)
        with pytest.raises(ValueError, match="holding is negative"):
            f(_Stub(), False, off, tok, pr, [0.0, bad, 0.0], None, None)
        with pytest.raises(ValueError, match="min_profit"):
            f(_Stub(), True, off, tok, pr, None, [bad, 0.0], None)
        with pytest.raises(ValueError, match="atol"):
            f(_Stub(), False, off, tok, pr, None, None, {"atol": bad})
    with pytest.raises(ValueError, match="no positive price"):
        f(_Stub(), False, off, tok, [1.0, 1.0, 0.0], None, None, None)
    with pytest.raises(ValueError, match="holding needs"):
        f(_Stub(), False, off, tok, pr, [0.0], None, None)
    # the Router's lists
    stub = _Stub()
    stub.v = np.zeros(6)
    g = cr.Router._inventory_args
    with pytest.raises(ValueError, match="one list of 1-based tokens per row"):
        g(stub, [1, 2], [[1.0, 1.0]], None, "quote_inventory_arbitrage")
    with pytest.raises(ValueError, match="outside 1..6"):
        g(stub, [[1, 7]], [[1.0, 1.0]], None, "quote_inventory_arbitrage")
    with pytest.raises(ValueError, match="listed twice"):
        g(stub, [[1, 1]], [[1.0, 1.0]], None, "quote_inventory_arbitrage")
    with pytest.raises(ValueError, match="prices needs one list per row"):
        g(stub, [[1, 2]], [[1.0]], None, "quote_inventory_arbitrage")
    with pytest.raises(ValueError, match="holdings needs one list per row"):
        g(stub, [[1, 2]], [[1.0, 1.0]], [[1.0]], "quote_inventory_arbitrage")
    off, tok, pr, h = g(stub, [[4, 1], [2]], [[1.0, 2.0], [3.0]], [[0.5, 0.0], [1.0]], "q")
    assert off.tolist() == [0, 2, 3] and tok.tolist() == [4, 1, 2]
    assert pr.tolist() == [1.0, 2.0, 3.0] and h.tolist() == [0.5, 0.0, 1.0]
    stub._world = 2
    with pytest.raises(NotImplementedError):
        g(stub, [[1, 2]], [[1.0, 1.0]], None, "quote_inventory_arbitrage")
