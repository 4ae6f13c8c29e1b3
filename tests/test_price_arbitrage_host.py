"""Host checks of price arbitrage rows (cfmm_quote_price_arbitrage, include/cfmm_b200.h): the row's box
and start (LinearNonnegative's lower limit, bit for bit), its stop and what the stop promises, and its
profit's operation order, on random vectors; its token set and pool list; the host route() with
LinearNonnegative(c) over one row's pools under the 50-digit certificate with the header's gap bound; and
the Python argument errors.  No GPU."""
import numpy as np
import pytest

import price_arb_oracle as pa
import solve_certificate as sc


@pytest.mark.parametrize("seed", range(5))
def test_box_start_merit_and_profit_order(cr, seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 40))
    c = rng.uniform(0.01, 100.0, n)
    lo = pa.box(c)
    # the box is LinearNonnegative's lower limit, bit for bit, and the start is that bound
    assert np.array_equal(lo, cr.LinearNonnegative(c).lower_limit())
    assert np.all(lo > c)
    # the profit: the first term alone, then the terms in local order
    psi = rng.normal(0.0, 10.0, n)
    want = c[0] * psi[0]
    for t in range(1, n):
        want = want + c[t] * psi[t]
    assert pa.profit(c, psi) == want
    if n > 2:
        assert pa.profit(c[::-1], psi[::-1]) == pytest.approx(want, rel=1e-9, abs=1e-9)
    # the stop: a token on its bound with Ψ > 0 is clipped; the max over the others scaled by 1/g
    nu = np.where(rng.random(n) < 0.3, lo, lo * rng.uniform(1.0, 2.0, n))
    g = float(abs(rng.normal(5.0, 1.0))) + 1e-3
    pg = np.where((nu <= lo) & (psi > 0), 0.0, psi)
    m = pa.merit(nu, psi, lo, g)
    assert m == (np.max(nu * np.abs(pg)) / g if np.any(pg) else 0.0)
    # what a stop at rtol promises: Ψ_t >= −rtol·g/ν_t, and g − cᵀΨ within the header's bound when
    # g = νᵀΨ (π positively homogeneous)
    rtol = 1e-4
    pos = rng.random(n) < 0.5
    nu2 = np.where(pos, lo, lo * rng.uniform(1.0, 1.5, n))
    psi2 = np.where(pos, rng.uniform(0.0, 1.0, n), -rng.uniform(0.0, 1.0, n) * rtol * g / nu2)
    g2 = float(nu2 @ psi2)
    if g2 > 0:
        pg2 = np.where((nu2 <= lo) & (psi2 > 0), 0.0, psi2)
        assert np.all(nu2 * np.abs(pg2) <= rtol * g * (1 + 1e-12))
        assert np.all(psi2 >= -rtol * g / nu2 * (1 + 1e-12))
        assert g2 - float(c @ psi2) <= pa.gap_bound(nu2, psi2, c, rtol, max(g, g2)) * (1 + 1e-9) + 1e-12


def test_merit_edges():
    lo = pa.box([1.0, 2.0])
    # nothing trades: m_r = 0, whatever g
    assert pa.merit(lo, np.zeros(2), lo, 0.0) == 0.0
    # on the bound with Ψ > 0: clipped
    assert pa.merit(lo, np.array([1.0, 0.0]), lo, 0.0) == 0.0
    # an imbalance with g <= 0 never stops the row
    assert pa.merit(lo, np.array([-1.0, 0.0]), lo, 0.0) == np.inf
    assert pa.profit([], []) == 0.0


def test_row_order():
    # tokens 1..6; allowed {1, 2, 3, 5, 6}; pairs (1, 2) active, (2, 3) retired only, (5, 6) active,
    # (3, 5) active, (1, 4) active (4 not allowed)
    lists = {(1, 2): [(0, 0, True), (2, 3, False)], (2, 3): [(1, 1, False)], (5, 6): [(0, 5, True)],
             (3, 5): [(0, 7, True)], (1, 4): [(0, 9, True)]}
    allowed = np.array([1, 1, 1, 0, 1, 1], bool)
    T, pools = pa.row_order(lists, allowed, [1.0, 2.0, 3.0, 4.0, 5.0])
    assert T == [1, 2, 3, 5, 6]
    assert sorted(pools) == sorted([(0, 0), (2, 3), (1, 1), (0, 5), (0, 7)])
    # a price of 0 takes a token out: 3 keeps (3, 5); 2 and 1 drop with 2's price
    T, pools = pa.row_order(lists, allowed, [1.0, 0.0, 3.0, 4.0, 0.0])
    assert T == [3, 5] and pools == [(0, 7)]
    # the retired pair alone does not make a token part of T
    T, _ = pa.row_order(lists, allowed, [0.0, 2.0, 3.0, 0.0, 0.0])
    assert T == []


def test_route_with_linear_nonnegative_over_a_rows_pools_certifies(cr):
    """The host route() (its sweeps on the CPU oracle) with LinearNonnegative(c) over one row's pools:
    the result certifies at 50 digits with the header's gap bound, no token's net is below −1e-4, and
    g = νᵀΨ is the profit within that gap."""
    import order_certificate as oc
    from test_host_logic import OraclePools

    spec = [([900.0, 1000.0], [1, 2]), ([500.0, 520.0], [1, 3]), ([800.0, 700.0], [2, 3]),
            ([700.0, 650.0], [3, 4]), ([600.0, 680.0], [2, 4]), ([300.0, 310.0], [4, 5])]
    cert = [oc.product(R, 0.997, A) for R, A in spec]
    n, rtol = 5, 1e-4
    c = np.array([1.0, 1.02, 0.97, 1.1, 0.9])
    r = cr.Router(cr.LinearNonnegative(c), [cr.ProductTwoCoin(R, 0.997, A) for R, A in spec], n,
                  _pools_factory=OraclePools)
    cr.route(r, pgtol=1e-11, factr=1e1)
    box = sc.linear_nonnegative(c)
    assert np.array_equal(box.lower, pa.box(c))
    res = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
    net = cr.netflows(r)
    g = float(res["g50"])
    assert g > 0.0
    assert abs(res["gap"]) <= pa.gap_bound(r.v, net, c, rtol, g) + res["allowance"], res
    assert np.all(net >= -1e-4)  # test/arb.jl's tolerance
    assert abs(g - pa.profit(c, net)) <= abs(res["gap"]) + res["allowance"] + 1e-9 * g


class _Stub:
    n_tokens = 6
    _world = 1


def test_python_argument_errors(cr):
    pa_ = cr.DevicePools._price_arb
    allowed = np.array([1, 1, 0, 1, 0, 0], bool)
    with pytest.raises(ValueError, match="allowed .* is required"):
        pa_(_Stub(), False, [[1.0, 1.0, 1.0]], None, None, None)
    with pytest.raises(ValueError, match="6 entries"):
        pa_(_Stub(), False, [[1.0, 1.0, 1.0]], allowed[:5], None, None)
    with pytest.raises(ValueError, match=r"\[q, 3\]"):
        pa_(_Stub(), False, [[1.0, 1.0]], allowed, None, None)
    with pytest.raises(ValueError, match=r"\[q, 3\]"):
        pa_(_Stub(), False, [1.0, 1.0, 1.0], allowed, None, None)
    for bad in (-1.0, np.nan, np.inf):
        with pytest.raises(ValueError, match="negative, NaN or Inf"):
            pa_(_Stub(), False, [[1.0, bad, 1.0]], allowed, None, None)
    with pytest.raises(ValueError, match="no positive price"):
        pa_(_Stub(), False, [[1.0, 1.0, 1.0], [0.0, 0.0, 0.0]], allowed, None, None)
    for bad in (-1.0, np.nan, np.inf):
        with pytest.raises(ValueError, match="min_profit"):
            pa_(_Stub(), True, [[1.0, 1.0, 1.0]], allowed, [bad], None)
    with pytest.raises(ValueError, match="more than 258"):
        s = _Stub()
        s.n_tokens = 300
        pa_(s, False, np.ones((1, 300)), np.ones(300, bool), None, None)
    with pytest.raises(ValueError):
        pa_(_Stub(), False, [[1.0, 1.0, 1.0]], allowed, None, {"max_iter": "x"})
    # the Router: a mask is required, one GPU only, a 1-D price vector is one row
    args = cr.Router._price_arb_args
    with pytest.raises(ValueError, match="allowed"):
        args(_Stub(), [1.0, 2.0, 3.0], None, "q")
    assert args(_Stub(), [1.0, 2.0, 3.0], allowed, "q").shape == (1, 3)
    s = _Stub()
    s._world = 2
    with pytest.raises(NotImplementedError):
        args(s, [[1.0, 2.0, 3.0]], allowed, "q")
