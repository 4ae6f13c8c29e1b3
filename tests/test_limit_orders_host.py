"""Host checks of limit_order_oracle and LimitBasket: a limit row's reachability and dropped entries on
hand-built pair lists, its box and the start's clamp, the surplus's operation order, LimitBasket through
the host route() under the 50-digit certificate (the dual value is the surplus; a partially filled
entry sits on its limit), zero limits giving BasketLiquidation exactly, and the Python argument errors.
No GPU."""
import numpy as np
import pytest

import limit_order_oracle as lo
from test_basket_orders_host import _Stub, lists


def test_reachability_and_dropped_entries():
    allowed = np.zeros(8, bool)
    allowed[[2, 3]] = True                       # B = {3, 4}
    # 5 reaches T only through a retired pool: at limit 0 a positive amount makes the row unreachable
    # (the basket rule); at a positive limit the entry is dropped and the row still solves
    T, _, unreach, dropped, solve = lo.row_limit(lists(), [2, 5], [1.0, 3.0], [0.5, 0.0], 1, allowed)
    assert T == [1, 2, 3, 4] and unreach and dropped == [False, False] and not solve
    T, _, unreach, dropped, solve = lo.row_limit(lists(), [2, 5], [1.0, 3.0], [0.5, 0.2], 1, allowed)
    assert T == [1, 2, 3, 4] and not unreach and dropped == [False, True] and solve
    # only a dropped entry has an amount: the row fills with zeros and runs no solve
    T, _, unreach, dropped, solve = lo.row_limit(lists(), [2, 5], [0.0, 3.0], [0.5, 0.2], 1, allowed)
    assert not unreach and dropped == [False, True] and not solve
    # the token set and pools do not depend on the amounts or the limits
    for lim in ([0.0, 0.0], [2.0, 7.0]):
        T2, pools2, _, _, _ = lo.row_limit(lists(), [7, 2], [1.0, 2.0], lim, 1, allowed)
        T1, pools1, _ = lo.row_basket(lists(), [7, 2], [1.0, 2.0], 1, allowed)
        assert T2 == T1 == [1, 7, 2, 3, 4] and pools2 == pools1


def test_box_and_start_clamp():
    T = [1, 7, 2, 3, 4]
    low = lo.box(T, [7, 2, 5], [0.25, 0.0, 3.0])
    assert low[0] == 1.0 + lo.SQRT_EPS and low[1] == 0.25 and low[2] == lo.SQRT_EPS
    assert np.all(low[3:] == lo.SQRT_EPS)
    # a limit below √eps keeps √eps; fmax is one IEEE operation
    assert lo.box(T, [7], [1e-12])[1] == lo.SQRT_EPS
    # zero limits: Swap's box bit for bit
    zero = lo.box(T, [7, 2], [0.0, 0.0])
    assert np.array_equal(zero, np.r_[1.0 + lo.SQRT_EPS, np.full(4, lo.SQRT_EPS)])
    # the start: breadth-first prices below an entry's limit are raised to it, others kept
    x = np.array([1.0, 0.1, 0.5, 0.0, 2.0])
    assert lo.start_clamp(x, low).tolist() == [1.0 + lo.SQRT_EPS, 0.25, 0.5, lo.SQRT_EPS, 2.0]


def test_surplus_operation_order():
    # received first, then a multiply and a subtract per entry, in entry order
    assert lo.surplus(10.0, [2.0, 3.0], [0.5, 1.5]) == (10.0 - 0.5 * 2.0) - 1.5 * 3.0
    a, b = 0.1, 3.0000000000000004
    want = np.float64(1.0) - np.float64(a) * np.float64(b)
    assert lo.surplus(1.0, [b], [a]) == float(want)
    # the order matters in fp64: 1e16 first, then 1, then −1e16 worth
    assert lo.surplus(1e16, [-1.0, 1e16], [1.0, 1.0]) == (1e16 + 1.0) - 1e16
    assert lo.surplus(5.0, [], []) == 5.0


def test_zero_limits_are_basket_liquidation(cr):
    rng = np.random.default_rng(3)
    for _ in range(5):
        n = 9
        d = rng.uniform(0, 10, n)
        i = int(rng.integers(1, n + 1))
        a, b = cr.LimitBasket(i, d, np.zeros(n)), cr.BasketLiquidation(i, d)
        assert np.array_equal(a.lower_limit(), b.lower_limit())
        assert np.array_equal(a.linear_term(), b.linear_term())
        assert np.array_equal(a.upper_limit(), b.upper_limit())
        v = b.lower_limit() + rng.uniform(0, 2, n)
        assert a.f(v) == pytest.approx(b.f(v), rel=1e-15)
    c = np.array([0.0, 0.5, 1e-12, 2.0])
    lb = cr.LimitBasket(1, [0.0, 1.0, 2.0, 3.0], c)
    assert lb.lower_limit().tolist() == [1.0 + lo.SQRT_EPS, 0.5, lo.SQRT_EPS, 2.0]
    assert lb.linear_term().tolist() == [0.0, 1.0, 2.0, 3.0]
    assert lb.f(lb.lower_limit()) == pytest.approx(2.0 * (lo.SQRT_EPS - 1e-12), rel=1e-6)
    assert lb.f(np.array([1.0, 0.5, 1.0, 2.0])) == np.inf
    with pytest.raises(ValueError):
        cr.LimitBasket(1, [1.0, 2.0], [0.0, -1.0])
    with pytest.raises(ValueError):
        cr.LimitBasket(1, [1.0, 2.0], [0.0])
    with pytest.raises(ValueError):
        cr.LimitBasket(3, [1.0, 2.0], [0.0, 0.0])


POOLS = [([900.0, 1000.0], [1, 2]), ([500.0, 520.0], [1, 3]), ([800.0, 790.0], [2, 3]),
         ([700.0, 650.0], [3, 4]), ([600.0, 640.0], [2, 4]), ([300.0, 310.0], [4, 5])]


@pytest.mark.parametrize("limits", [[0.0, 0.0, 0.0], [0.85, 0.5, 0.0], [0.8, 0.97, 0.9], [2.0, 2.0, 2.0]])
def test_limit_basket_through_host_route_certifies(cr, limits):
    """LimitBasket(1, Δin, c) over six ProductTwoCoin pools through the host route() (its sweeps on the
    CPU oracle): the result certifies at 50 digits under the limit box with ℓ̂ = c at the entries, so
    the certified gap bounds how far the surplus Ψ_1 + Σ c_k·Ψ_k is below the optimum; the surplus is
    at least minus that gap (trading nothing is feasible); and an entry sold partially has ν_k on its
    limit, one sold in full has ν_k above it."""
    import order_certificate as oc
    import solve_certificate as sc
    from test_host_logic import OraclePools

    n = 5
    basket, amounts = [2, 3, 5], [25.0, 10.0, 4.0]
    d, c = np.zeros(n), np.zeros(n)
    d[np.array(basket) - 1] = amounts
    c[np.array(basket) - 1] = limits
    obj = cr.LimitBasket(1, d, c)
    r = cr.Router(obj, [cr.ProductTwoCoin(R, 0.997, A) for R, A in POOLS], n, _pools_factory=OraclePools)
    cr.route(r, pgtol=1e-10, factr=1e1)
    cert = [oc.product(R, 0.997, A) for R, A in POOLS]
    ref = c.copy()
    ref[0] = 1.0
    box = sc.Box(obj.linear_term(), obj.lower_limit(), ref=ref)
    res = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
    tol = 1e-6 * max(1.0, abs(res["g50"])) + res["allowance"]
    assert abs(res["gap"]) <= tol, res
    net = cr.netflows(r)
    S = lo.surplus(net[0], [-net[t - 1] for t in basket], limits)
    # the dual value (constant included) is the surplus at the optimum
    assert abs(res["g50"] - float(d @ c) - S) <= tol
    assert S >= -tol
    for t, a, lim in zip(basket, amounts, limits):
        paid = -net[t - 1]
        assert paid <= a * (1 + 1e-6)
        low = obj.lower_limit()[t - 1]
        if paid < a * (1 - 1e-4):            # partially filled (or bought): ν_k on its limit
            assert r.v[t - 1] <= low * (1 + 1e-6), (t, r.v[t - 1], low)
        if r.v[t - 1] > low * (1 + 1e-4):    # above its limit: sold in full
            assert abs(paid - a) <= 1e-5 * a
    if limits == [0.0, 0.0, 0.0]:
        for t, a in zip(basket, amounts):
            assert abs(-net[t - 1] - a) <= 1e-6 * a
    if limits == [2.0, 2.0, 2.0]:
        # every entry on its limit, so the row may also receive an entry token: the pools deliver token
        # 3 for less than 2 of the others, and the surplus counts it at its limit
        assert all(r.v[t - 1] <= 2.0 * (1 + 1e-6) for t in basket) and net[2] > 0.0


def test_python_argument_errors(cr):
    ok = ([1], [0, 1], [3], [1.0], [0.5], np.ones(6, bool))
    f = cr.DevicePools._limit
    for args, match in [
        (([1, 2], [0, 1], [3], [1.0], [0.5], np.ones(6, bool)), "basket_off must have 3"),
        (([1], [0, 1], [3], [1.0], [0.5, 1.0], np.ones(6, bool)), "need basket_off"),
        (([1], [0, 1], [3], [1.0], [-0.5], np.ones(6, bool)), "limit price"),
        (([1], [0, 1], [3], [1.0], [np.nan], np.ones(6, bool)), "limit price"),
        (([1], [0, 1], [3], [1.0], [np.inf], np.ones(6, bool)), "limit price"),
        (([1], [0, 1], [3], [1.0], [0.5], None), "allowed"),
        (([1], [0, 1], [3], [1.0], [0.5], np.ones(5, bool)), "6 entries"),
    ]:
        with pytest.raises(ValueError, match=match):
            f(_Stub(), False, *args, None, None)
    with pytest.raises(ValueError, match="limit must have"):
        f(_Stub(), True, *ok, [1.0, 2.0], None)
    class _RStub(_Stub):
        _basket_args = cr.Router._basket_args

    args = cr.Router._limit_args
    tout, off, toks, amts, lims, _ = args(_RStub(), [1, 2], [{2: (1.0, 0.5), 3: (2.0, 0.0)}, ([4], [0.5], [3.0])],
                                          np.ones(6, bool), None, "q")
    assert off.tolist() == [0, 2, 3] and toks.tolist() == [2, 3, 4] and amts.tolist() == [1.0, 2.0, 0.5]
    assert lims.tolist() == [0.5, 0.0, 3.0]
    with pytest.raises(ValueError, match="one entry per row"):
        args(_RStub(), [1], [{2: (1.0, 0.0)}, {3: (1.0, 0.0)}], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="one limit per token"):
        args(_RStub(), [1], [([2, 3], [1.0, 1.0], [0.5])], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="amount, limit"):
        args(_RStub(), [1], [{2: (1.0,)}], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="tokens, amounts, limits"):
        args(_RStub(), [1], [([2], [1.0])], np.ones(6, bool), None, "q")
    with pytest.raises(ValueError, match="limits must have"):
        args(_RStub(), [1], [{2: (1.0, 0.0)}], np.ones(6, bool), [1.0, 2.0], "q")
    s = _RStub()
    s._world = 2
    with pytest.raises(NotImplementedError):
        args(s, [1], [{2: (1.0, 0.0)}], np.ones(6, bool), None, "q")
