"""Orders split across the pools of their token pair (cfmm_quote_split_orders /
cfmm_execute_split_orders) on the host, without a GPU.

The mirror in split_oracle.py is checked against the closed form for identical ProductTwoCoin
pools, against route() (scipy L-BFGS-B over the oracle's sweeps) with the reference's Swap objective
on the pair's pools, for the bracket the search promises, for its evaluation bound and for the
in-order replay with limits.  The Router methods are checked through an oracle-backed stand-in for
DevicePools, as in test_paths_host.py."""
import numpy as np
import pytest

import split_oracle as so
from swap_order_oracle import from_ordinal, ordinal
from test_paths_host import PathPools
from test_swap_orders_host import random_univ3
from test_swaps_host import market

EPS = np.finfo(np.float64).eps


def random_pair_pools(rng, n, types=(0, 1, 2), a=1, b=2):
    """n pools on the pair {a, b}, random orientation and type, prices spread around 1."""
    pools = []
    for k in range(n):
        t = types[k % len(types)]
        Ai = [a, b] if rng.random() < 0.5 else [b, a]
        if t == 0:
            pools.append(so.Product(np.exp(rng.uniform(2, 8)) * np.exp(rng.uniform(-0.3, 0.3, size=2)),
                                    rng.choice([0.997, 0.9995, 1.0]), Ai))
        elif t == 1:
            pools.append(so.GeoMean(np.exp(rng.uniform(2, 8, size=2)), 0.997, rng.uniform(0.3, 0.7, size=2), Ai))
        else:
            u = random_univ3(rng)
            pools.append(so.Univ3(u.price, u.lt, u.lq, u.g, Ai))
    return pools


def bracket(pools, row, tin, tout, kind, amount):
    """The header's bracket: exact-in N(s*) <= δ < N(pred s*), exact-out O(s*) >= y > O(succ s*)."""
    o = ordinal(row["price"])
    if kind == so.EXACT_IN:
        assert row["paid"] <= amount
        N = so.evaluate(pools, tout, tin, from_ordinal(o - 1))[0]
        assert not (N <= amount)
    else:
        assert row["received"] >= amount
        O = so.evaluate(pools, tout, tin, from_ordinal(o + 1))[1]
        assert O < amount


# ---- the mirror ----------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 7, 40])
def test_identical_product_pools_closed_form(n):
    for R, g, d in [(1000.0, 0.997, 5.0), (3.5e6, 0.9995, 1.2e4), (50.0, 1.0, 49.0)]:
        pools = [so.Product([R, R], g, [1, 2] if k % 2 else [2, 1]) for k in range(n)]
        row = so.split_row(pools, 1, 2, so.EXACT_IN, d)
        assert row["status"] == so.FILLED
        for k, p in enumerate(pools):  # (one ulp of s moves a leg by about eps·(R + γδ/n)/2γ)
            j = 0 if p.Ai[0] == 1 else 1
            assert abs(row["D"][k, j] - d / n) <= 1e-12 * (R + d / n)
        # paid is within one step of s below δ; each pool then receives the closed form at paid/n
        assert 0.0 <= d - row["paid"] <= 4 * n * EPS * (R + d / n) / g
        exact = n * (R - R * R / (R + g * row["paid"] / n))
        assert abs(row["received"] - exact) <= 1e-12 * exact


class SplitPools(PathPools):
    """PathPools with the pair index, the split orders of the mirror, and host sweeps (oracle
    find_arb! and folds) so that route() runs against the same pools."""

    def _objs(self):
        objs = {}
        for t in (0, 1, 2):
            for i in range(len(self.Ai[t])):
                Ai = self.Ai[t][i]
                if t == 0:
                    objs[t, i] = so.Product(self.R[0][i], self.g[0][i], Ai)
                elif t == 1:
                    objs[t, i] = so.GeoMean(self.R[1][i], self.g[1][i], self.w[i], Ai)
                else:
                    objs[t, i] = so.Univ3(self.cp[i], *self.ticks[i], self.g[2][i], Ai)
        return objs

    def _keys(self, a, b):
        return [(t, i) for t in (0, 1, 2) for i in range(len(self.Ai[t])) if set(self.Ai[t][i]) == {a, b}]

    def pair_pools(self, token_a, token_b):
        keys = [self._keys(int(a), int(b)) for a, b in zip(token_a, token_b)]
        off = np.concatenate([[0], np.cumsum([len(k) for k in keys])]).astype(np.int64)
        flat = [k for ks in keys for k in ks]
        return (off, np.array([t for t, _ in flat], dtype=np.int32), np.array([i for _, i in flat], dtype=np.int64),
                np.ones(len(flat), bool))

    def _split(self, execute, tin, tout, kind, amount, limit):
        objs = self._objs()
        fn = so.replay_split if execute else so.quote_split
        rows = fn(lambda a, b: [objs[k] for k in self._keys(a, b)], tin, tout, kind, amount,
                  *((limit,) if execute else ()))
        if execute:
            for (t, i), p in objs.items():
                if t == 2:
                    self.cp[i] = p.price
                else:
                    self.R[t][i] = p.R
        return tuple(np.array([r[k] for r in rows], dtype=np.uint8 if k == "status" else float).reshape(-1)
                     for k in ("paid", "received", "price", "status"))

    def quote_split_orders(self, tin, tout, kind, amount):
        return self._split(False, tin, tout, kind, amount, None)

    def execute_split_orders(self, tin, tout, kind, amount, limit=None):
        return self._split(True, tin, tout, kind, amount, limit)

    def sweep(self, v, materialize=False):
        objs = self._objs()
        D, L = np.zeros((len(objs), 2)), np.zeros((len(objs), 2))
        psi, acc = np.zeros(self.n_tokens), 0.0
        for k, key in enumerate(sorted(objs)):
            p = objs[key]
            va = np.asarray(v)[np.array(p.Ai) - 1]
            D[k], L[k] = p.legs(va)
            psi[np.array(p.Ai) - 1] += L[k] - D[k]
            acc += float(np.dot(L[k] - D[k], va))
        self._trades = (D, L)
        return psi, acc

    def trades(self):
        return self._trades


def feasible(c, D, L, tol=1e-6):
    """check_primal_feasibility of the reference's tests (test/arb.jl:5-16) on one pool's legs:
    no negative leg beyond tol, and the invariant does not drop beyond sqrt(eps)."""
    R = c.R + c.gamma * D - L
    return np.all(D >= -tol) and np.all(L >= -tol) and R[0] * R[1] >= c.R[0] * c.R[1] - np.sqrt(EPS)


def test_matches_route_on_the_pair(cr):
    """The split equals route! with Swap(i, j, δ, 2) over the pair's pools (L-BFGS-B tolerance)."""
    rng = np.random.default_rng(11)
    for trial in range(6):
        n = int(rng.integers(1, 6))
        pools = []
        for _ in range(n):
            Ai = [1, 2] if rng.random() < 0.5 else [2, 1]
            pools.append(cr.ProductTwoCoin(rng.uniform(100, 1000) * np.exp(rng.uniform(-0.05, 0.05, size=2)),
                                           0.997, Ai))
        delta = float(rng.uniform(1, 50))
        r = cr.Router(cr.Swap(1, 2, delta, 2), pools, 2, _pools_factory=SplitPools)
        cr.route(r, pgtol=1e-10, factr=1e1)
        psi = cr.netflows(r)
        mirror = [so.Product(c.R, c.gamma, c.Ai) for c in pools]
        row = so.split_row(mirror, 2, 1, so.EXACT_IN, delta)
        assert row["status"] == so.FILLED
        # (route!'s L-BFGS-B stops within about 1e-6 of the optimum; the split is exact to one step of s)
        assert abs(row["received"] - psi[0]) <= 1e-5 * psi[0], (trial, row["received"], psi[0])
        assert abs(row["paid"] + psi[1]) <= 1e-5 * delta
        assert abs(row["price"] - r.v[1] / r.v[0]) <= 1e-5 * row["price"]
        for k, c in enumerate(pools):
            assert feasible(c, row["D"][k], row["L"][k])


def test_bracket_and_evaluation_bound():
    rng = np.random.default_rng(3)
    seen = {so.FILLED: 0, so.UNREACHABLE: 0}
    for k in range(120):
        pools = random_pair_pools(rng, int(rng.integers(1, 9)), types=((0, 1, 2), (0,), (2,))[k % 3])
        tin, tout = (1, 2) if k % 2 else (2, 1)
        kind = int(rng.integers(0, 2))
        amount = float(10.0 ** rng.uniform(-4, 3)) if k % 11 else float(10.0 ** rng.uniform(5, 300))
        row = so.split_row(pools, tin, tout, kind, amount)
        assert row["evals"] <= so.MAX_EVALS
        seen[row["status"]] += 1
        if row["status"] == so.FILLED and k % 3:  # (GeometricMean: monotone only to a few ulp)
            bracket(pools, row, tin, tout, kind, amount)
    assert seen[so.FILLED] > 60 and seen[so.UNREACHABLE] > 0


def test_zero_amount_and_no_active_pool():
    pools = [so.Product([100.0, 200.0], 0.997, [1, 2]), so.Product([100.0, 100.0], 0.997, [2, 1])]
    row = so.split_row(pools, 1, 2, so.EXACT_IN, 0.0)
    assert row["status"] == so.FILLED and row["evals"] == 0 and not row["D"].any() and row["received"] == 0.0
    for p in pools:
        p.active = False
    assert so.split_row(pools, 1, 2, so.EXACT_OUT, 1.0)["status"] == so.UNREACHABLE
    assert so.split_row([], 1, 2, so.EXACT_IN, 1.0)["status"] == so.UNREACHABLE


def test_univ3_with_an_empty_last_tick_is_unreachable_past_its_depth():
    u = so.Univ3(1.0, [1.2, 1.0, 0.8], [10.0, 20.0, 0.0], 0.997, [1, 2])
    ok = so.split_row([u], 1, 2, so.EXACT_IN, 0.3)  # (tick 2 absorbs about 0.53)
    assert ok["status"] == so.FILLED
    assert so.split_row([u], 1, 2, so.EXACT_IN, 1e6)["status"] == so.UNREACHABLE
    assert so.split_row([u], 1, 2, so.EXACT_OUT, 1e6)["status"] == so.UNREACHABLE


def test_replay_limits_and_reverts():
    rng = np.random.default_rng(8)
    # one price, several depths and fees: no arbitrage between the pools, so paid > 0
    base = [so.Product(np.full(2, np.exp(rng.uniform(3, 8))), rng.choice([0.997, 0.9995]),
                       [1, 2] if k % 2 else [2, 1]) for k in range(5)]
    clone = lambda ps: [so.Univ3(p.price, p.lt, p.lq, p.g, p.Ai) if isinstance(p, so.Univ3)
                        else so.Product(p.R, p.g, p.Ai) for p in ps]
    q = so.split_row(clone(base), 1, 2, so.EXACT_IN, 3.0)
    # an equal limit fills, one ulp tighter reverts, and the next row sees the state without it
    a = clone(base)
    r0 = so.split_row(a, 1, 2, so.EXACT_IN, 3.0, limit=q["received"], execute=True)
    assert r0["status"] == so.FILLED and r0["received"] == q["received"]
    b = clone(base)
    r1 = so.split_row(b, 1, 2, so.EXACT_IN, 3.0, limit=float(np.nextafter(q["received"], np.inf)), execute=True)
    assert r1["status"] == so.LIMIT and r1["paid"] == 0.0 and not r1["D"].any()
    r2 = so.split_row(b, 1, 2, so.EXACT_IN, 3.0, execute=True)
    assert r2["received"] == q["received"]
    # exact-out: the maximum paid
    q2 = so.split_row(clone(base), 2, 1, so.EXACT_OUT, 2.0)
    c = clone(base)
    assert so.split_row(c, 2, 1, so.EXACT_OUT, 2.0, limit=q2["paid"], execute=True)["status"] == so.FILLED
    c = clone(base)
    lim = float(np.nextafter(q2["paid"], 0.0))
    assert so.split_row(c, 2, 1, so.EXACT_OUT, 2.0, limit=lim, execute=True)["status"] == so.LIMIT
    # a filled row moves the pools, so the same row again gets less
    assert so.split_row(a, 1, 2, so.EXACT_IN, 3.0)["received"] < q["received"]


# ---- the Router, through an oracle-backed stand-in -----------------------------------------
def test_router_split_map_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=SplitPools)
    for a in range(1, n + 1):
        for b in range(1, n + 1):
            if a != b:
                want = [i for t in (0, 1, 2) for i in r._type_lists[t] if set(pools[i].Ai) == {a, b}]
                assert r.pair_pools(a, b).tolist() == want
    pairs = [(int(c.Ai[0]), int(c.Ai[1])) for c in pools[:8]]
    tin = np.array([p[0] for p in pairs] + [p[1] for p in pairs])
    tout = np.array([p[1] for p in pairs] + [p[0] for p in pairs])
    q = len(tin)
    kinds = np.arange(q) % 2
    amounts = np.full(q, 0.5)
    paid, got, price, st = r.quote_split_orders(tin, tout, kinds, amounts)
    for j in range(q):  # each row quoted on its own gives the same
        one = r.quote_split_orders(tin[j:j + 1], tout[j:j + 1], kinds[j:j + 1], amounts[j:j + 1])
        assert [x[0] for x in one] == [paid[j], got[j], price[j], st[j]]
    before = [c.R.copy() if hasattr(c, "R") else c.current_price for c in pools]
    limits = np.where(kinds == 1, paid * 1.001, got * 0.999)
    limits[3] = got[3] * 2.0 if kinds[3] == 0 else paid[3] * 0.5  # reverts
    paid, got, price, st = r.execute_split_orders(tin, tout, kinds, amounts, limits)
    assert st[3] == so.LIMIT and so.FILLED in st.tolist()
    touched = {i for j in np.flatnonzero(st == so.FILLED) for i in r.pair_pools(tin[j], tout[j])}
    state = r._pools
    for i, c in enumerate(pools):
        t = [cr.ProductTwoCoin, cr.GeometricMeanTwoCoin, cr.UniV3].index(type(c))
        k = r._type_lists[t].index(i)
        if t == 2:
            assert c.current_price == state.cp[k]
            changed = c.current_price != before[i]
        else:
            assert np.array_equal(c.R, state.R[t][k])
            changed = not np.array_equal(c.R, before[i])
        assert changed <= (i in touched)


def test_router_split_argument_checks(cr):
    n = 6
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=SplitPools)
    with pytest.raises(ValueError):
        r.quote_split_orders([1, 2], [2], [0, 0], [1.0, 1.0])
    with pytest.raises(ValueError):
        r.execute_split_orders([1], [2], [0], [1.0], limits=[0.0, 1.0])
    out = r.quote_split_orders([], [], [], [])
    assert all(x.shape == (0,) for x in out)
    r._world = 2  # a multi-GPU Router
    for call in (lambda: r.quote_split_orders([1], [2], [0], [1.0]),
                 lambda: r.execute_split_orders([1], [2], [0], [1.0]),
                 lambda: r.pair_pools(1, 2)):
        with pytest.raises(NotImplementedError):
            call()
