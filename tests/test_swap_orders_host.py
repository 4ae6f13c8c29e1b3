"""Exact-output quotes and order rows with limits (cfmm_quote_swaps_exact_out /
cfmm_execute_swap_orders) on the host, without a GPU.

The mirror in swap_order_oracle.py is checked for the crossing property the header promises,
ProductTwoCoin monotonicity, agreement with a 50-digit inverse, the evaluation bound and the
in-order replay with limits.  The Router methods are checked through an oracle-backed stand-in
for DevicePools, as in test_swaps_host.py."""
import mpmath as mp
import numpy as np
import pytest

import swap_order_oracle as oo
from test_swaps_host import SwapPools, market

EPS = np.finfo(np.float64).eps
DBL_MAX = np.finfo(np.float64).max
MAX_EVALS = 1 + 63 + 62


def pred(x):
    return float(np.nextafter(x, 0.0))


def check_crossing(pool, y, tok1):
    """x* of the mirror satisfies the header's crossing property; returns (x*, evaluations)."""
    x, n = oo.exact_out(pool, y, tok1)
    assert n <= MAX_EVALS
    if x == oo.INF:
        assert pool.f(DBL_MAX, tok1) < y
    else:
        assert pool.f(x, tok1) >= y, (y, x)
        assert x == 0.0 or pool.f(pred(x), tok1) < y, (y, x)
    return x, n


def random_univ3(rng, ticks=None):
    t = int(rng.integers(1, 17)) if ticks is None else ticks
    cp = float(np.exp(rng.uniform(-2, 2)))
    lt = cp * float(np.exp(rng.uniform(0.05, 1.0))) * np.cumprod(
        np.concatenate([[1.0], rng.uniform(0.5, 0.95, size=t - 1)]))
    lq = rng.uniform(0, 50, size=t)
    lq[rng.random(t) < 0.25] = 0.0
    g = float(rng.choice([1.0, 0.997, 0.9995]))
    return oo.Univ3Pool(cp, lt, lq, g)


# ---- ordinals ------------------------------------------------------------------------------
def test_ordinals():
    assert oo.ordinal(0.0) == 0 and oo.ordinal(DBL_MAX) == oo.ORD_MAX
    assert oo.from_ordinal(1) == np.nextafter(0.0, 1.0) and oo.from_ordinal(oo.ORD_MAX) == DBL_MAX
    rng = np.random.default_rng(1)
    xs = np.sort(np.concatenate([10.0 ** rng.uniform(-300, 300, size=500), [5e-324, 1.0, 2.0, DBL_MAX]]))
    o = [oo.ordinal(x) for x in xs]
    assert o == sorted(o)
    for x in xs[:-1]:
        assert oo.from_ordinal(oo.ordinal(x)) == x
        assert oo.from_ordinal(oo.ordinal(x) + 1) == np.nextafter(x, np.inf)
    assert oo.start_ordinal(float("nan")) == 1 and oo.start_ordinal(-3.0) == 1 and oo.start_ordinal(0.0) == 1
    assert oo.start_ordinal(float("inf")) == oo.ORD_MAX and oo.start_ordinal(2.0) == oo.ordinal(2.0)


def test_crossing_search_on_a_step_function():
    # f(x) = floor(x): the least x with f >= y is y itself; from any estimate, within the bound
    for y in (1.0, 3.0, 1e10, 2.0 ** 60):
        for e in (0.0, 1e-300, y / 3, y, 3 * y, 1e300, float("inf"), float("nan")):
            o, n = oo.crossing(np.floor, y, e)
            assert oo.from_ordinal(o) == y and n <= MAX_EVALS, (y, e, n)
    o, n = oo.crossing(lambda x: 0.0, 1.0, 1.0)  # never reaches: unreachable
    assert o == -1 and n <= 64


# ---- crossing property ---------------------------------------------------------------------
def test_product_crossing_random_and_adversarial():
    rng = np.random.default_rng(2)
    for k in range(400):
        scale = 2.0 ** rng.choice([-100, 0, 0, 0, 100]) if k % 4 == 0 else 1.0
        R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=2)) * scale
        pool = oo.ProductPool(R, rng.choice([1.0, 0.997, 0.99]))
        tok1 = bool(k % 2)
        r_out = R[1] if tok1 else R[0]
        for y in (r_out * 10.0 ** rng.uniform(-12, -0.001), r_out * 1e-300, 5e-324, r_out, pred(r_out),
                  float(np.nextafter(r_out, np.inf))):
            x, n = check_crossing(pool, y, tok1)
            if y > r_out:
                assert x == oo.INF
    # y = 0 costs nothing
    assert oo.exact_out(oo.ProductPool([3.0, 4.0], 0.997), 0.0, True) == (0.0, 0)


def test_univ3_crossing_random_and_adversarial():
    rng = np.random.default_rng(3)
    unreachable = 0
    for k in range(150):
        pool = random_univ3(rng)
        tok1 = bool(k % 2)
        cap = pool.f(DBL_MAX, tok1)  # everything the walk can give
        ys = [cap * 10.0 ** rng.uniform(-9, 0), cap, pred(cap), float(np.nextafter(cap, np.inf)), 1e-300]
        # y at the output capacity of each tick the walk passes: the partial sums of R_out
        n, cur = len(pool.lt), oo.current_tick(pool.lt, pool.price)
        acc = 0.0
        for idx in (range(cur, n + 1) if tok1 else range(cur, 0, -1)):
            _, _, _, R1, R2 = oo.univ3_tick(pool.price, cur, pool.lt, pool.lq, idx)
            acc = acc + float(R2 if tok1 else R1)
            if acc > 0:
                ys += [acc, pred(acc)]
        for y in ys:
            if y > 0:
                x, _ = check_crossing(pool, y, tok1)
                unreachable += x == oo.INF
    assert unreachable > 10


def test_univ3_empty_ticks_and_reference_pool():
    # test/cfmms.jl:117-120: ticks (30, 20, 10, 5], liquidities (1, 2, 1.5, 0) -- an empty last tick
    pool = oo.Univ3Pool(15.0, [30.0, 20, 10, 5], [1.0, 2.0, 1.5, 0.0], 0.997)
    for tok1 in (True, False):
        cap = pool.f(DBL_MAX, tok1)
        for y in np.concatenate([np.geomspace(1e-9, 1, 40) * cap, [cap, pred(cap)]]):
            x, _ = check_crossing(pool, y, tok1)
            assert x < oo.INF
        assert oo.exact_out(pool, float(np.nextafter(cap, np.inf)), tok1)[0] == oo.INF
    # a ladder of empty ticks only reaches nothing
    empty = oo.Univ3Pool(2.0, [4.0, 3.0, 1.0], [0.0, 0.0, 0.0], 1.0)
    assert oo.exact_out(empty, 1e-300, True)[0] == oo.INF and oo.exact_out(empty, 1.0, False)[0] == oo.INF


def test_geomean_crossing():
    rng = np.random.default_rng(4)
    for k in range(300):
        R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=2))
        w1 = float(rng.choice([0.04, 0.3, 0.5, 0.96]))
        pool = oo.GeoMeanPool(R, rng.choice([1.0, 0.997]), [w1, 1 - w1])
        tok1 = bool(k % 2)
        r_out = R[1] if tok1 else R[0]
        for y in (r_out * 10.0 ** rng.uniform(-12, -0.001), r_out * 1e-200, pred(r_out)):
            check_crossing(pool, y, tok1)


# ---- monotonicity -------------------------------------------------------------------------
def test_product_monotone_on_dense_grids():
    rng = np.random.default_rng(5)
    for _ in range(40):
        R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=2)) * 2.0 ** rng.choice([-100, 0, 100])
        pool = oo.ProductPool(R, rng.choice([1.0, 0.997]))
        for tok1 in (True, False):
            r_in = R[0] if tok1 else R[1]
            xs = [oo.from_ordinal(oo.ordinal(r_in * 10.0 ** rng.uniform(-14, 4)) + j) for j in range(300)]
            xs += list(r_in * np.geomspace(1e-16, 1e16, 300))
            fx = [pool.f(x, tok1) for x in sorted(xs)]
            assert all(a <= b for a, b in zip(fx, fx[1:]))
    # so x* is the least tender that reaches y: no smaller tender on a dense grid reaches it
    pool = oo.ProductPool([123.0, 456.0], 0.997)
    x, _ = oo.exact_out(pool, 7.0, True)
    o = oo.ordinal(x)
    assert all(pool.f(oo.from_ordinal(o - j), True) < 7.0 for j in range(1, 2000))


# ---- agreement with a 50-digit inverse -----------------------------------------------------
def _mp_inverse(kind, r_in, r_out, g, y, eta=None):
    """The exact tender receiving y (or +inf past R_out)."""
    y = mp.mpf(y)
    if y >= r_out:
        return mp.inf
    if kind == "product":
        d = r_in * r_out / (r_out - y) - r_in
    else:
        d = r_in * ((1 - y / r_out) ** (-1 / eta) - 1)
    return d / g


@pytest.mark.parametrize("kind", ["product", "geomean"])
def test_inverse_against_mpmath(kind):
    """x* lies between the exact inverses of y ∓ B, B = the forward bound plus eps/2·R_out for the
    rounding of γ·x: 4·eps·R_out for ProductTwoCoin, (4 + 2η)·eps·R_out for GeometricMean."""
    rng = np.random.default_rng(6)
    with mp.workdps(50):
        for k in range(300):
            R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=2))
            g = float(rng.choice([1.0, 0.997]))
            tok1 = bool(k % 2)
            i, o = (0, 1) if tok1 else (1, 0)
            if kind == "product":
                pool, eta, fwd = oo.ProductPool(R, g), None, 4.0
            else:
                w1 = float(rng.choice([0.04, 0.3, 0.5, 0.96]))
                pool = oo.GeoMeanPool(R, g, [w1, 1 - w1])
                eta = mp.mpf(pool.w[i]) / mp.mpf(pool.w[o])
                fwd = 4 + 2 * float(eta)
            r_in, r_out, gm = mp.mpf(R[i]), mp.mpf(R[o]), mp.mpf(g)
            y = float(R[o] * 10.0 ** rng.uniform(-10, -0.01))
            x, _ = oo.exact_out(pool, y, tok1)
            B = (fwd + 0.5) * EPS * R[o]
            assert x >= _mp_inverse(kind, r_in, r_out, gm, y - B, eta), (k, x)
            assert pred(x) <= _mp_inverse(kind, r_in, r_out, gm, y + B, eta), (k, x)


# ---- evaluation count ----------------------------------------------------------------------
def test_evaluation_count():
    """Within 1 + 63 + 62 always.  For ProductTwoCoin the count follows the plateaus of f: R_in + δ
    rounds to a multiple of ulp(R_in), so f is constant over about R_in/x* consecutive tenders and
    the gallop and the bisection each take about log2(R_in/x*) steps when x* << R_in."""
    rng = np.random.default_rng(7)
    counts = []
    for k in range(300):
        R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=2))
        pool = oo.ProductPool(R, 0.997)
        x, n = oo.exact_out(pool, R[1] * 10.0 ** rng.uniform(-12, -0.01), True)
        assert n <= 2 * max(0.0, np.log2(R[0] / x)) + 12, (R, x, n)
        counts.append(n)
    for k in range(100):
        pool = random_univ3(rng)
        cap = pool.f(DBL_MAX, True)
        if cap > 0:
            counts.append(oo.exact_out(pool, cap * 10.0 ** rng.uniform(-6, -0.001), True)[1])
    assert max(counts) <= MAX_EVALS


# ---- in-order replay with limits -----------------------------------------------------------
def test_replay_limits_and_reverts():
    pools = [oo.ProductPool([1000.0, 2000.0], 0.997), oo.Univ3Pool(15.0, [30.0, 20, 10, 5], [1.0, 2.0, 1.5, 0.0], 0.997)]
    # the first exact-out row's x* and the exact-in quote of 5
    x0, _ = oo.exact_out(oo.ProductPool([1000.0, 2000.0], 0.997), 50.0, True)
    l5 = oo.ProductPool([1000.0, 2000.0], 0.997).f(5.0, True)
    kind = [oo.EXACT_OUT, oo.EXACT_OUT, oo.EXACT_IN, oo.EXACT_IN, oo.EXACT_OUT, oo.EXACT_OUT]
    amount = [(0.0, 50.0), (0.0, 50.0), (5.0, 0.0), (0.0, 0.0), (0.0, 3000.0), (0.0, 0.0)]
    limit = [pred(x0), x0, 0.0, 0.0, oo.INF, 0.0]
    paid, rec, st, _ = oo.replay_orders(pools, [0] * 6, kind, amount, limit)
    # one ulp below x* reverts, x* itself fills against the unchanged state
    assert st.tolist() == [oo.LIMIT, oo.FILLED, oo.FILLED, oo.FILLED, oo.UNREACHABLE, oo.FILLED]
    assert paid[0].tolist() == [0.0, 0.0] and rec[0].tolist() == [0.0, 0.0]
    assert paid[1].tolist() == [x0, 0.0] and rec[1, 1] >= 50.0 and rec[1, 0] == 0.0
    assert rec[2, 1] < l5  # the exact-in row sees the filled exact-out row before it
    assert paid[3].tolist() == [0.0, 0.0] and paid[5].tolist() == [0.0, 0.0]
    # an exact-in limit equal to what arrives fills; one ulp more reverts
    a = oo.ProductPool([1000.0, 2000.0], 0.997)
    got = a.f(5.0, False)
    for lim, want in ((got, oo.FILLED), (float(np.nextafter(got, np.inf)), oo.LIMIT)):
        st = oo.replay_orders([oo.ProductPool([1000.0, 2000.0], 0.997)], [0], [0], [(0.0, 5.0)], [lim])[2]
        assert st.tolist() == [want]
    # a (0, 0) exact-in row with a positive minimum reverts; retired pools revert every row
    assert oo.replay_orders(pools, [0], [0], [(0.0, 0.0)], [1.0])[2].tolist() == [oo.LIMIT]
    _, _, st, _ = oo.replay_orders(pools, [1, 1], [0, 1], [(1.0, 0.0), (0.0, 0.0)], retired={1})
    assert st.tolist() == [oo.RETIRED, oo.RETIRED]


def test_replay_filled_rows_equal_exact_in_replay():
    """The filled rows of a batch leave the state, and receive what, the same tenders as exact-in
    rows without limits give."""
    rng = np.random.default_rng(8)
    for make in (lambda: oo.ProductPool([300.0, 700.0], 0.997),
                 lambda: oo.Univ3Pool(15.0, [30.0, 20, 10, 5], [1.0, 2.0, 1.5, 0.0], 0.997)):
        q = 60
        kind = rng.integers(0, 2, size=q)
        side = rng.integers(0, 2, size=q)
        amount = np.zeros((q, 2))
        amount[np.arange(q), side] = 10.0 ** rng.uniform(-3, 0.5, size=q)
        limit = np.where(kind == 1, 10.0 ** rng.uniform(-3, 1, size=q), 10.0 ** rng.uniform(-4, 0, size=q))
        a = make()
        paid, rec, st, _ = oo.replay_orders([a], np.zeros(q, dtype=int), kind, amount, limit)
        assert {0, 1} <= set(st.tolist())
        b = make()
        filled = np.flatnonzero(st == oo.FILLED)
        paid2, rec2, st2, _ = oo.replay_orders([b], np.zeros(len(filled), dtype=int), np.zeros(len(filled)),
                                               paid[filled])
        assert np.array_equal(rec2, rec[filled]) and not st2.any()
        assert np.array_equal(getattr(a, "R", None), getattr(b, "R", None)) and getattr(a, "price", 0) == getattr(b, "price", 0)


# ---- the Router, through an oracle-backed stand-in -----------------------------------------
class OrderPools(SwapPools):
    """SwapPools with the exact-output quote and the order rows of the mirror."""

    def _pool(self, t, i):
        if t == 0:
            return oo.ProductPool(self.R[0][i], self.g[0][i])
        if t == 1:
            return oo.GeoMeanPool(self.R[1][i], self.g[1][i], self.w[i])
        return oo.Univ3Pool(self.cp[i], *self.ticks[i], self.g[2][i])

    def quote_swaps_exact_out(self, t, pools, want):
        return np.array([oo.quote_exact_out(self._pool(t, i), y) for i, y in zip(pools, want)]).reshape(-1, 2)

    def execute_swap_orders(self, t, pools, kind, amount, limit=None):
        objs = {i: self._pool(t, i) for i in set(int(i) for i in pools)}
        paid, rec, st, _ = oo.replay_orders(objs, [int(i) for i in pools], kind, amount, limit)
        for i, p in objs.items():
            if t == 2:
                self.cp[i] = p.price
            else:
                self.R[t][i] = p.R
        return paid, rec, st


def test_router_orders_map_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=OrderPools)
    ref = OrderPools(n)
    r2 = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=lambda *a: ref)
    rng = np.random.default_rng(9)
    q = 40
    ids = rng.integers(0, len(pools), size=q)
    W = np.zeros((q, 2))
    W[np.arange(q), rng.integers(0, 2, size=q)] = rng.uniform(0.1, 30, size=q)
    W[::9] = 0.0

    def loc(i):
        t = [0, 1, 2][[cr.ProductTwoCoin, cr.GeometricMeanTwoCoin, cr.UniV3].index(type(pools[i]))]
        return t, r2._type_lists[t].index(i)
    x = r.quote_swaps_exact_out(ids, W)
    for j, i in enumerate(ids):  # caller's order, each row on the current state
        t, k = loc(i)
        assert np.array_equal(x[j], ref.quote_swaps_exact_out(t, [k], W[j:j + 1])[0])
    assert np.isinf(x).any() and (x[::9] == 0).all()
    kind = rng.integers(0, 2, size=q)
    amount = np.where(kind[:, None] == 1, W, W[:, ::-1] * 0.5)
    limit = np.where(kind == 1, rng.uniform(0, 40, size=q), rng.uniform(0, 2, size=q))
    before = [c.R.copy() if hasattr(c, "R") else c.current_price for c in pools]
    paid, rec, st = r.execute_swap_orders(ids, kind, amount, limit)
    for j, i in enumerate(ids):  # replayed one row at a time, in order
        t, k = loc(i)
        p1, r1, s1 = ref.execute_swap_orders(t, [k], kind[j:j + 1], amount[j:j + 1], limit[j:j + 1])
        assert np.array_equal(p1[0], paid[j]) and np.array_equal(r1[0], rec[j]) and s1[0] == st[j]
    assert {0, 1} <= set(st.tolist())
    filled = set(ids[(st == 0) & (paid.max(axis=1) > 0)].tolist())
    for i, c in enumerate(pools):
        t, k = loc(i)
        if t == 2:
            assert c.current_price == ref.cp[k]
            assert c.current_tick == int(np.sum(c.lower_ticks >= c.current_price))
            changed = c.current_price != before[i]
        else:
            assert np.array_equal(c.R, ref.R[t][k])
            changed = not np.array_equal(c.R, before[i])
        assert changed <= (i in filled)


def test_router_order_argument_checks(cr):
    n = 6
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=OrderPools)
    with pytest.raises(ValueError):
        r.quote_swaps_exact_out([0, 1], [[0.0, 1.0]])
    with pytest.raises(ValueError):
        r.execute_swap_orders([0, 1], [0], [[1.0, 0.0], [1.0, 0.0]])
    with pytest.raises(ValueError):
        r.execute_swap_orders([0], [0], [[1.0, 0.0]], limits=[0.0, 1.0])
    with pytest.raises(IndexError):
        r.quote_swaps_exact_out([15], [[0.0, 1.0]])
    with pytest.raises(IndexError):
        r.execute_swap_orders([-1], [1], [[0.0, 1.0]])
    assert r.quote_swaps_exact_out([], np.zeros((0, 2))).shape == (0, 2)
    paid, rec, st = r.execute_swap_orders([], [], np.zeros((0, 2)))
    assert paid.shape == rec.shape == (0, 2) and st.shape == (0,)
    r._world = 2  # a multi-GPU Router
    with pytest.raises(NotImplementedError):
        r.quote_swaps_exact_out([0], [[0.0, 1.0]])
    with pytest.raises(NotImplementedError):
        r.execute_swap_orders([0], [1], [[0.0, 1.0]])
