"""The 50-digit certificate of order_certificate.py, without a GPU.

The reference itself is checked against closed forms (π of a fee-free ProductTwoCoin pool), a
brute-force grid (the UniV3 walk, with zero-liquidity gaps and an empty last tick) and a 50-digit
root of the derivative (GeometricMeanTwoCoin π).  Then the host mirrors of split and routed orders (split_oracle.py,
route_oracle.py), the oracle of the bit-exact GPU tests, are certified on deep pairs and hub sets."""
import mpmath as mp
import numpy as np
import pytest

import oracle_lib
import order_certificate as oc
import route_oracle as ro
import split_oracle as so
from test_split_orders_host import random_pair_pools


def cert_pool(p):
    if isinstance(p, so.Univ3):
        return oc.univ3(p.price, p.lt, p.lq, p.g, p.Ai, p.active)
    if isinstance(p, so.GeoMean):
        return oc.geomean(p.R, p.g, p.w, p.Ai, p.active)
    return oc.product(p.R, p.g, p.Ai, p.active)


def certify(direct, hubs, j, i, kind, amount, res, nested=True):
    row = oc.Row([cert_pool(p) for p in direct],
                 [(h, [cert_pool(p) for p in A], [cert_pool(p) for p in B]) for h, A, B in hubs], j, i)
    out = dict(res)
    out.setdefault("hub_price", [])
    out.setdefault("hub_surplus", [])
    return oc.certify_row(row, kind, amount, out, nested=nested)


# ---- the reference ---------------------------------------------------------------------------
def test_product_pi_closed_form():
    rng = np.random.default_rng(1)
    for _ in range(50):
        R = 10.0 ** rng.uniform(-3, 9, size=2)
        nu = [mp.mpf(float(x)) for x in 10.0 ** rng.uniform(-2, 2, size=2)]
        with mp.workdps(50):
            pi = oc.response(oc.product(R, 1.0, [1, 2]), nu)[2]
            want = (mp.sqrt(nu[0] * R[0]) - mp.sqrt(nu[1] * R[1])) ** 2
            assert abs(pi - want) <= mp.mpf(10) ** -40 * (nu[0] * R[0] + nu[1] * R[1])
            # with a fee: the first-order condition holds, and the forward trade pays the flows
            p = oc.product(R, 0.997, [1, 2])
            D, L, v, _ = oc.response(p, nu)
            a = 0 if D[0] > 0 else 1
            if D[a] > 0:
                assert abs(oc.forward(p, a, D[a]) - L[1 - a]) <= mp.mpf(10) ** -40 * R[1 - a]
                h = D[a] * mp.mpf(10) ** -20
                slope = (oc.forward(p, a, D[a] + h) - oc.forward(p, a, D[a] - h)) / (2 * h)
                assert abs(slope * nu[1 - a] - nu[a]) <= mp.mpf(10) ** -15 * nu[a]


def grid_walk(price, lt, lq, a, target, steps=20000):
    """The UniV3 flows from price to target on a fine geometric grid of prices, each step at the
    liquidity of the tick it starts in."""
    lt = np.asarray(lt, float)
    ps = np.geomspace(price, target, steps + 1)
    xin = yout = 0.0
    for p0, p1 in zip(ps[:-1], ps[1:]):
        mid = np.sqrt(p0 * p1)
        k = float(lq[int(np.sum(lt >= mid)) - 1]) if mid <= lt[0] else 0.0
        if a == 0:
            xin += np.sqrt(k / p1) - np.sqrt(k / p0)
            yout += np.sqrt(k * p0) - np.sqrt(k * p1)
        else:
            xin += np.sqrt(k * p1) - np.sqrt(k * p0)
            yout += np.sqrt(k / p0) - np.sqrt(k / p1)
    return xin, yout


@pytest.mark.parametrize("lq", [[1.0, 2.0, 1.5, 0.7], [1.0, 0.0, 3.0, 2.0], [2.0, 1.0, 0.0, 0.0]],
                         ids=["dense", "gap", "empty-last"])
def test_univ3_walk_against_grid(lq):
    lt = [30.0, 20.0, 10.0, 5.0]
    p = oc.univ3(15.0, lt, lq, 0.997, [1, 2])
    for target in (14.0, 9.0, 4.0, 1.0, 16.0, 25.0, 29.0):
        a = 0 if target < 15.0 else 1
        with mp.workdps(50):
            g = mp.mpf(0.997)
            nu = [mp.mpf(target) * g, mp.mpf(1)] if a == 0 else [mp.mpf(target) / g, mp.mpf(1)]
            D, L, v, _ = oc.response(p, nu)
        x, y = grid_walk(15.0, lt, lq, a, target)
        # (the grid straddles each tick boundary with one step: up to about 1e-4 of the flow)
        assert abs(float(D[a]) * 0.997 - x) <= 1e-3 * x and abs(float(L[1 - a]) - y) <= 1e-3 * y
        # the forward trade of the tender pays the same flows
        assert abs(oc.forward(p, a, D[a]) - L[1 - a]) <= mp.mpf(10) ** -40 * (1 + L[1 - a])
    # the depth: an empty last tick caps what token 0 buys; the top of the ladder caps token 1
    x0, y0 = oc.depth(p, 0)
    assert (x0 == mp.inf) == (lq[-1] > 0)
    x1, y1 = oc.depth(p, 1)
    assert x1 < mp.inf and abs(float(y1) - grid_walk(15.0, lt, lq, 1, 30.0)[1]) <= 1e-4 * float(y1)


def test_univ3_walk_matches_the_oracle_forward_trade():
    """forward() against the CPU oracle's forward_trade (a double walk): a few ulp of the scale."""
    o = oracle_lib.load()
    lt, lq = [30.0, 20.0, 10.0, 5.0], [1.0, 0.0, 3.0, 2.0]
    p = oc.univ3(15.0, lt, lq, 0.997, [1, 2])
    for x in np.geomspace(1e-6, 1e3, 30):
        for a in (0, 1):
            T = [x, 0.0] if a == 0 else [0.0, x]
            got = o.univ3_forward_trade(15.0, lt, lq, 0.997, T)
            assert abs(oc.forward(p, a, mp.mpf(float(x))) - got) <= 64 * oc.EPS * 20


def test_geomean_pi_against_findroot():
    rng = np.random.default_rng(2)
    for _ in range(20):
        R = 10.0 ** rng.uniform(-2, 6, size=2)
        w = [0.05, 0.95] if rng.random() < 0.5 else list(rng.uniform(0.2, 0.8, size=2))
        p = oc.geomean(R, 0.997, w, [1, 2])
        with mp.workdps(50):
            nu = [mp.mpf(float(x)) for x in (w[0] / R[0], w[1] / R[1])]
            nu[0] *= mp.mpf(float(rng.choice([0.5, 2.0])))
            D, L, v, _ = oc.response(p, nu)
            a = 0 if D[0] > 0 else 1
            assert D[a] > 0
            f = lambda x: nu[1 - a] * oc.forward(p, a, x) - nu[a] * x
            df = lambda x: (f(x * (1 + mp.mpf(10) ** -20)) - f(x * (1 - mp.mpf(10) ** -20))) / (x * 2 * mp.mpf(10) ** -20)
            # the derivative's root, by bisection from a bracket 0.1 % either side of the closed form
            lo, hi = D[a] * mp.mpf(0.999), D[a] * mp.mpf(1.001)
            assert df(lo) > 0 > df(hi)
            for _ in range(90):
                mid = (lo + hi) / 2
                lo, hi = (mid, hi) if df(mid) > 0 else (lo, mid)
            x = (lo + hi) / 2
            assert abs(x - D[a]) <= mp.mpf(10) ** -20 * D[a]
            assert abs(f(D[a]) - v) <= mp.mpf(10) ** -35 * (nu[0] * R[0] + nu[1] * R[1])
            assert f(D[a] * mp.mpf(0.999)) < v and f(D[a] * mp.mpf(1.001)) < v


# ---- the mirrors, certified ------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 31, 33, 65])
def test_split_mirror_certified(n):
    rng = np.random.default_rng(100 + n)
    for k in range(6 if n < 60 else 3):
        pools = random_pair_pools(rng, n, types=((0, 1, 2), (0,), (2,), (1,))[k % 4])
        for q in pools[::7]:
            q.active = n == 1
        tin, tout = (1, 2) if k % 2 else (2, 1)
        kind = k // 2 % 2
        amount = float(10.0 ** rng.uniform(-6, 2)) * max(1, n // 8)
        res = so.split_row(pools, tin, tout, kind, amount)
        assert res["status"] == so.FILLED
        c = certify(pools, [], tin, tout, kind, amount, res)
        assert c["gap"] <= c["allowance"]


def test_routed_mirror_certified():
    rng = np.random.default_rng(6)
    for k in range(10):
        types = ((0,), (2,), (0, 2), (1,), (0, 1, 2))[k % 5]
        direct = random_pair_pools(rng, int(rng.integers(0, 4)), types, a=1, b=2)
        hubs = [(h, random_pair_pools(rng, int(rng.integers(0, 3)), types, a=1, b=h),
                 random_pair_pools(rng, int(rng.integers(0, 3)), types, a=h, b=2)) for h in range(3, 3 + 1 + k % 3)]
        kind = k % 2
        amount = float(10.0 ** rng.uniform(-3, 1.5))
        res = ro.route_row(direct, hubs, 1, 2, kind, amount)
        certify(direct, hubs, 1, 2, kind, amount, res, nested=k < 6)


def test_routed_mirror_seven_hubs_certified():
    """Seven hubs, one with more than 32 pools over its two lists, one with pools on one side only."""
    rng = np.random.default_rng(8)
    direct = random_pair_pools(rng, 2, (0,), a=1, b=2)
    hubs = [(3, random_pair_pools(rng, 14, (0, 2), a=1, b=3), random_pair_pools(rng, 21, (0, 2), a=3, b=2)),
            (4, random_pair_pools(rng, 1, (0,), a=1, b=4), [])]
    hubs += [(h, random_pair_pools(rng, 1, (0,), a=1, b=h), random_pair_pools(rng, 1, (2,), a=h, b=2))
             for h in range(5, 10)]
    for kind, amount in ((0, 3.0), (1, 2.0)):
        res = ro.route_row(direct, hubs, 1, 2, kind, amount)
        assert res["status"] == ro.FILLED
        certify(direct, hubs, 1, 2, kind, amount, res, nested=kind == 0)


def test_unreachable_rows_against_the_depth():
    u = so.Univ3(1.0, [1.2, 1.0, 0.8], [10.0, 20.0, 0.0], 0.997, [1, 2])
    p = oc.univ3(1.0, [1.2, 1.0, 0.8], [10.0, 20.0, 0.0], 0.997, [1, 2])
    for tin, tout in ((1, 2), (2, 1)):
        a = p.Ai.index(tin)
        xin, yout = (float(v) for v in oc.depth(p, a))
        for kind, cap in ((1, yout), (0, xin)):
            for f, want in ((1 - 1e-9, so.FILLED), (1 + 1e-9, so.UNREACHABLE)):
                res = so.split_row([u], tin, tout, kind, cap * f)
                assert res["status"] == want, (tin, kind, f)
                certify([u], [], tin, tout, kind, cap * f, res)
    # a wrong status is caught
    res = so.split_row([u], 1, 2, 1, yout * 0.5)
    with pytest.raises(AssertionError):
        certify([u], [], 1, 2, 1, yout * 0.5, dict(res, status=so.UNREACHABLE, D=res["D"] * 0, L=res["L"] * 0))


def test_certificate_catches_a_one_percent_misallocation():
    """Legs moved between two pools (accounting intact) fail the optimality check."""
    rng = np.random.default_rng(4)
    pools = random_pair_pools(rng, 4, (0,))
    res = so.split_row(pools, 1, 2, 0, 5.0)
    certify(pools, [], 1, 2, 0, 5.0, res)
    D, L = res["D"].copy(), res["L"].copy()
    k = [n for n in range(4) if D[n, pools[n].Ai.index(1)] > 0][:1]
    assert k
    n = k[0]
    x = pools[n].Ai.index(1)
    D[n, x] *= 0.99
    L[n, 1 - x] = float(oc.forward(cert_pool(pools[n]), x, mp.mpf(float(D[n, x]))))
    bad = dict(res, D=D, L=L, paid=float(sum(D[m, pools[m].Ai.index(1)] for m in range(4))),
               received=float(sum(L[m, pools[m].Ai.index(2)] for m in range(4))))
    with pytest.raises(AssertionError):
        certify(pools, [], 1, 2, 0, 5.0, bad)


def test_geomean_closed_form_overflow_is_pinned():
    """The reference's geom_arb_δ forms γ·m·η·R₁·R₂^η before its 1/(η+1)-th root: at extreme price
    ratios it overflows to an infinite tender though the optimum of the trading set is finite.  The
    mirror keeps that parity (a row deep enough to reach such prices reports paid = inf)."""
    o = oracle_lib.load()
    R, w, g = np.array([1e9, 1e9]), np.array([0.05, 0.95]), 0.997
    v = np.array([1.0, 1e-200])  # token 1 nearly worthless: sell it
    D, L = o.geomean_arb(R, w, g, v)
    assert D[1] == np.inf and L[0] <= R[0]
    p = oc.geomean(R, g, w, [1, 2])
    with mp.workdps(50):
        d, l, _, _ = oc.response(p, [mp.mpf(1), mp.mpf(1e-200)])
    assert mp.isfinite(d[1]) and d[1] > 0 and l[0] <= R[0]
