"""Host checks of the exact-out rows of subgraph orders (include/cfmm_b200.h,
cfmm_quote_subgraph_swap_orders): the dual over one row's pools restated with scipy's L-BFGS-B from
the 50-digit pool responses and certified on its raw box (ν_j fixed at 1, ℓ̂_i = 0); an exact-out row
asking for what an exact-in row received pays what that row tendered; the capacity pre-check on
ProductTwoCoin, GeometricMeanTwoCoin and UniV3 pools (one whose last tick is empty); and the Python
argument errors of the kind argument.  No GPU."""
import math

import numpy as np
import pytest

import order_certificate as oc
import solve_certificate as sc
import subgraph_exact_out_oracle as xo
import subgraph_oracle as so

RTOL = 1e-6


def row_pools():
    # tokens 1..4; the row buys i = 1 and pays in j = 2 through B = {3, 4}, with pools between 3 and 4
    return [oc.product([900.0, 1000.0], 0.997, [1, 2]), oc.product([500.0, 520.0], 0.997, [1, 3]),
            oc.product([800.0, 790.0], 0.997, [2, 3]), oc.product([700.0, 650.0], 0.997, [3, 4]),
            oc.product([600.0, 640.0], 0.997, [2, 4]), oc.product([400.0, 380.0], 1.0, [1, 4], active=False)]


def solve(pools, box, n, gtol=1e-11):
    from scipy.optimize import minimize
    sweep = sc.oracle_sweep(pools, n)
    bounds = [(lo, None if not np.isfinite(up) else up) for lo, up in zip(box.lower, box.upper)]
    res = minimize(lambda x: float(box.lin @ x) + sweep(x)[1], np.maximum(np.ones(n), box.lower),
                   jac=lambda x: box.lin + sweep(x)[0], method="L-BFGS-B", bounds=bounds,
                   options=dict(maxcor=5, ftol=0.0, gtol=gtol, maxiter=3000))
    return res.x, sweep(res.x)[0]


def exact_out(pools, n, i, j, y):
    """The certified exact-out solve: (ν, Ψ, certificate)."""
    box = xo.box(n, i, j, y, RTOL)
    x, psi = solve(pools, box, n)
    assert x[j - 1] == 1.0
    m, ok = xo.stop_bounds(x, box.lin + psi, box.lower, y, i - 1, j - 1, RTOL)
    assert ok, m
    free = np.arange(n) != j - 1
    pgtol = float(np.max(m * y * x[i - 1] / x[free])) * (1 + 1e-9) + 1e-12
    D, L = sc.oracle_trades(pools, x)
    cert = sc.certify(pools, box, x, D, L, pgtol=pgtol, rule="lbfgsb")
    return x, psi, cert


def test_scipy_exact_out_over_a_rows_pools_certifies():
    pools = row_pools()
    lists = {}
    for k, p in enumerate(pools):
        a, b = sorted(p.Ai)
        lists.setdefault((a, b), []).append((0, k, p.active))
    T, listed = so.row_subgraph(lists, 2, 1, np.ones(4, bool))
    assert T == [1, 2, 3, 4] and sorted(k for _, k in listed) == list(range(6))
    n, i, j, y = 4, 1, 2, 25.0
    x, psi, cert = exact_out(pools, n, i, j, y)
    assert cert["gap"] <= cert["bound"] + cert["allowance"]
    # the fill promise: received in [y, y·(1 + 2·rtol)] with ν_i off its bound, a positive payment,
    # and every intermediate within the stop's bound
    assert x[i - 1] > xo.SQRT_EPS
    assert y <= psi[i - 1] <= y * (1 + 2 * RTOL) * (1 + 1e-12), psi[i - 1]
    assert -psi[j - 1] > 0.0
    for b in (3, 4):
        assert psi[b - 1] >= -RTOL * y * x[i - 1] / x[b - 1] * (1 + 1e-9)
    # the gap bound of the header: |T|·rtol·y·ν_i plus the box's terms
    assert cert["gap"] <= len(T) * RTOL * y * x[i - 1] + cert["allowance"] + 1e-9 * y


def test_round_trip_exact_in_then_exact_out_pays_the_tender():
    pools = row_pools()
    n, i, j, delta = 4, 1, 2, 40.0
    lin = np.zeros(n)
    lin[j - 1] = delta
    box_in = sc.basket(i, lin)
    x_in, psi_in = solve(pools, box_in, n)
    m, ok = so.stop_bounds(x_in, box_in.lin + psi_in, box_in.lower, delta, j - 1, RTOL)
    assert ok, m
    received = float(psi_in[i - 1])
    assert received > 0.0
    x, psi, _ = exact_out(pools, n, i, j, received)
    paid = -float(psi[j - 1])
    # exact-in tendered δ within rtol·δ; exact-out buys at most 2·rtol·y more than y, each unit at
    # the marginal price ν_i/ν_j (ν_j = 1 here)
    bound = RTOL * delta + 2 * RTOL * received * x[i - 1] + 1e-9 * delta
    assert abs(paid - delta) <= bound, (paid, delta, bound)


def ladder():
    # lower ticks descending; tick 4 spans (0, 0.5] and is empty
    return [4.0, 2.0, 1.0, 0.5], [100.0, 200.0, 150.0, 0.0]


@pytest.mark.parametrize("side", [0, 1])
def test_capacity_per_pool_type(side):
    lt, lq = ladder()
    u = oc.univ3(1.5, lt, lq, 0.997, [1, 2])
    c_u = xo.pool_capacity("univ3", side, price=1.5, lt=lt, lq=lq, g=0.997)
    # the fp64 walk to the end of the ladder is the 50-digit depth of the pool, up to rounding
    want = float(oc.depth(u, 1 - side)[1])
    assert c_u > 0.0 and abs(c_u - want) <= 1e-12 * want, (c_u, want)
    # the empty last tick pays nothing: with liquidity there, only the walk down (paying token 2)
    # gains the tick's sqrt(k·0.5)
    c_full = xo.pool_capacity("univ3", side, price=1.5, lt=lt, lq=lq[:3] + [50.0], g=0.997)
    if side == 0:
        assert c_full == c_u
    else:
        assert abs(c_full - c_u - math.sqrt(50.0 * 0.5)) <= 1e-12 * c_full, (c_full, c_u)
    # two-coin pools: the reserve of the side paid out
    P = oc.product([900.0, 1000.0], 0.997, [1, 2])
    G = oc.geomean([300.0, 700.0], 0.99, [0.3, 0.7], [1, 2])
    assert xo.pool_capacity("product", side, R=P.R) == P.R[side]
    assert xo.pool_capacity("geomean", side, R=G.R) == G.R[side]
    # no price pays out more than the capacity: the optimal response at ν_out/ν_in = 1e12 (a UniV3
    # walk then reaches the end of its ladder; a two-coin pool never pays out its whole reserve)
    for p, c in ((u, c_u), (P, P.R[side]), (G, G.R[side])):
        nu = [oc._m(1.0), oc._m(1.0)]
        nu[side] = oc._m(1e12)
        _, L, _, _ = oc.response(p, nu)
        got = float(L[side])
        assert 0.0 < got <= c * (1 + 1e-12) and (p.kind == "univ3" or got < c), (p.kind, got, c)


def test_capacity_rule_on_a_row():
    lt, lq = ladder()
    # the row's pools in pool order: two pools holding i on side 0 and 1, one that does not, a retired one
    terms = [xo.pool_capacity("product", 0, R=(900.0, 1000.0)),
             xo.pool_capacity("univ3", 1, price=1.5, lt=lt, lq=lq, g=0.997),
             0.0,   # a pool between two other tokens
             0.0,   # a retired pool holding i
             xo.pool_capacity("geomean", 0, R=(300.0, 700.0))]
    C = xo.capacity(terms)
    assert abs(C - math.fsum(terms)) <= 4 * np.finfo(float).eps * C
    assert xo.unreachable(C, terms) and xo.unreachable(2 * C, terms)
    assert not xo.unreachable(math.nextafter(C, 0.0), terms)
    assert xo.unreachable(1.0, terms, j_in_T=False)
    # the kernel's order: 300 pools, thread l adds pools l, l + 256 (then the butterfly and the warps)
    many = [float(k % 7) + 0.1 for k in range(300)]
    assert abs(xo.capacity(many) - math.fsum(many)) <= 300 * np.finfo(float).eps * math.fsum(many)


def test_y_prime_rounds_up():
    from fractions import Fraction
    for y in (1.0, 3.0, 25.0, 0.1, 1e300 / 3, 7e-300):
        for rtol in (1e-4, 1e-6, 3e-5):
            v = xo.y_prime(y, rtol)
            exact = Fraction(y) * Fraction(rtol) + Fraction(y)
            assert Fraction(v) >= exact and Fraction(math.nextafter(v, 0.0)) < exact


class _Stub:
    n_tokens = 6


@pytest.mark.parametrize("kind, limit, match", [
    ([0, 1, 0], None, "kind must have 2 entries"),
    ([0, 2], None, "kind must be 0"),
    ([1, 255], None, "kind must be 0"),
    ([0, 1], [float("inf"), 1.0], "exact-in limit"),
    (0, [1.0, float("inf")], "exact-in limit"),
    ([1, 1], [1.0, float("nan")], "NaN"),
    ([0, 1], [float("nan"), 1.0], "NaN"),
])
def test_python_argument_errors(kind, limit, match):
    import cfmmrouter_b200 as cr
    args = ([1, 2], [3, 4], [1.0, 1.0], np.ones(6, bool))
    execute = limit is not None
    with pytest.raises(ValueError, match=match):
        cr.DevicePools._subgraph(_Stub(), execute, *args, limit, None, kind)


def test_python_kind_forms():
    import cfmmrouter_b200 as cr
    rk = cr.router._row_kind
    assert rk(None, 3, None, "x") is None
    assert rk(1, 3, None, "x").tolist() == [1, 1, 1] and rk(1, 3, None, "x").dtype == np.uint8
    assert rk([0, 1, 0], 3, None, "x").tolist() == [0, 1, 0]
    # exact-out limits may be +inf (no cap on the payment)
    assert rk([1, 0], 2, np.array([np.inf, 2.0]), "x").tolist() == [1, 0]
