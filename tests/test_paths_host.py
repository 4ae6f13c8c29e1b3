"""Multi-hop swap paths (cfmm_quote_paths / cfmm_execute_paths) on the host, without a GPU.

The mirror in path_oracle.py is checked against the single-row order replay of
swap_order_oracle.py, for the crossing property of every exact-out hop, for the pass-on of a
negative intermediate output, and for the status precedence.  The Router methods are checked
through an oracle-backed stand-in for DevicePools, as in test_swap_orders_host.py."""
import numpy as np
import pytest

import path_oracle as po
import swap_order_oracle as oo
from test_swap_orders_host import OrderPools, pred, random_univ3
from test_swaps_host import market

DBL_MAX = np.finfo(np.float64).max


def random_pool(rng, k):
    if k % 3 == 0:
        return oo.ProductPool(np.exp(rng.uniform(0, 8, size=2)), rng.choice([0.997, 1.0]))
    if k % 3 == 1:
        return oo.GeoMeanPool(np.exp(rng.uniform(0, 8, size=2)), 0.997, rng.uniform(0.2, 0.8, size=2))
    return random_univ3(rng)


def clone(p):
    if isinstance(p, oo.Univ3Pool):
        return oo.Univ3Pool(p.price, p.lt, p.lq, p.g)
    if isinstance(p, oo.GeoMeanPool):
        return oo.GeoMeanPool(p.R, p.g, p.w)
    return oo.ProductPool(p.R, p.g)


# ---- the mirror ----------------------------------------------------------------------------
def test_one_hop_path_is_an_order_row():
    rng = np.random.default_rng(1)
    for k in range(300):
        base = random_pool(rng, k)
        tok1 = bool(rng.integers(0, 2))
        kind = int(rng.integers(0, 2))
        amt = float(10.0 ** rng.uniform(-6, 2.5)) if k % 17 else 0.0
        lim = float(10.0 ** rng.uniform(-6, 3)) if k % 3 else None
        a, b = clone(base), clone(base)
        x, lam, st = po.quote_path([a], [tok1], kind, amt, lim, execute=True)
        side = 0 if tok1 else 1  # the tendered side
        row = [0.0, 0.0]
        row[side if kind == oo.EXACT_IN else 1 - side] = amt
        paid, rec, st2, _ = oo.replay_orders([b], [0], [kind], [row], None if lim is None else [lim])
        assert st == st2[0]
        assert x[0] == paid[0].max() and lam[0] == rec[0, 1 - side]
        assert getattr(a, "R", a.__dict__.get("price")).tolist() == getattr(b, "R", b.__dict__.get("price")).tolist()


def test_exact_out_hops_cross_and_keep_a_surplus():
    rng = np.random.default_rng(2)
    seen = 0
    for k in range(200):
        n = int(rng.integers(1, 9))
        pools = [random_pool(rng, int(rng.integers(0, 3)) if k % 2 else 0) for _ in range(n)]
        tok1 = list(rng.integers(0, 2, size=n).astype(bool))
        y = float(10.0 ** rng.uniform(-4, 1))
        x, lam, st = po.quote_path(pools, tok1, oo.EXACT_OUT, y)
        if st != po.FILLED:
            assert st == po.UNREACHABLE and not x.any() and not lam.any()
            continue
        seen += 1
        want = np.concatenate([x[1:], [y]])  # y_h: what hop h must deliver
        for h in range(n):
            assert lam[h] >= want[h] and lam[h] - want[h] >= 0.0
            assert x[h] == 0.0 or pools[h].f(pred(x[h]), tok1[h]) < want[h]
            assert x[h] == oo.exact_out(pools[h], want[h], tok1[h])[0]
    assert seen > 50


def test_negative_intermediate_is_passed_on_as_zero():
    def p1():
        return oo.ProductPool([0.692853898234414, 766.1105947727434], 0.997)

    def p2():
        return oo.ProductPool([5.0, 7.0], 0.997)
    x1 = 1.188266364553944e-19
    assert p1().f(x1, True) < 0.0
    x, lam, st = po.quote_path([p1(), p2()], [True, True], oo.EXACT_IN, x1)
    assert st == po.FILLED and lam[0] < 0.0 and x[1] == 0.0 and lam[1] == 0.0
    # execute: the second hop receives 0, which meets the default minimum, and does not move
    b = p2()
    x, lam, st = po.quote_path([p1(), b], [True, False], oo.EXACT_IN, x1, execute=True)
    assert st == po.FILLED and x[1] == 0.0 and lam[1] == 0.0 and b.R.tolist() == [5.0, 7.0]
    # a negative final output misses the default minimum
    _, lam, st = po.quote_path([p1()], [True], oo.EXACT_IN, x1)
    assert st == po.FILLED and lam[0] < 0.0
    _, _, st = po.quote_path([p1()], [True], oo.EXACT_IN, x1, execute=True)
    assert st == po.LIMIT


def test_status_precedence():
    pools = [oo.ProductPool([10.0, 10.0], 1.0), oo.ProductPool([10.0, 10.0], 1.0)]
    big = 100.0  # more than the last pool holds: unreachable
    # retired beats unreachable and limit
    x, lam, st = po.quote_path(pools, [True, True], oo.EXACT_OUT, big, limit=0.0, retired=True, execute=True)
    assert st == po.RETIRED and not x.any() and not lam.any()
    # unreachable beats limit
    _, _, st = po.quote_path(pools, [True, True], oo.EXACT_OUT, big, limit=0.0, execute=True)
    assert st == po.UNREACHABLE
    # the limit applies to execute only; an equal limit fills, one ulp beyond reverts
    x, lam, st = po.quote_path(pools, [True, True], oo.EXACT_OUT, 1.0, limit=0.0)
    assert st == po.FILLED and x[0] > 0
    for kind, amt, at, beyond in ((oo.EXACT_OUT, 1.0, lambda x, l: x[0], lambda v: pred(v)),
                                  (oo.EXACT_IN, 1.0, lambda x, l: l[-1], lambda v: np.nextafter(v, np.inf))):
        x, lam, _ = po.quote_path(pools, [True, False], kind, amt)
        v = at(x, lam)
        a = [clone(p) for p in pools]
        assert po.quote_path(a, [True, False], kind, amt, limit=beyond(v), execute=True)[2] == po.LIMIT
        assert [p.R.tolist() for p in a] == [p.R.tolist() for p in pools]
        x2, lam2, st = po.quote_path(a, [True, False], kind, amt, limit=v, execute=True)
        assert st == po.FILLED and x2.tolist() == x.tolist() and lam2.tolist() == lam.tolist()
    # exact-out amount 0: all zeros, filled
    x, lam, st = po.quote_path(pools, [True, True], oo.EXACT_OUT, 0.0, limit=0.0, execute=True)
    assert st == po.FILLED and not x.any() and not lam.any()


def test_replay_sees_earlier_filled_paths_only():
    rng = np.random.default_rng(4)
    pools = {i: random_pool(rng, i) for i in range(6)}
    hop_off = [0, 2, 4, 5]
    hops = [0, 1, 1, 2, 0]
    tok1 = [True, False, True, True, False]
    kind, amount = [0, 1, 0], [3.0, 0.5, 2.0]
    # the first path reverts (impossible minimum): the second and third see the state before it
    ref = {i: clone(p) for i, p in pools.items()}
    t, r, st = po.replay_paths(pools, hop_off, hops, tok1, kind, amount, limit=[1e300, np.inf, 0.0])
    assert st.tolist() == [po.LIMIT, po.FILLED, po.FILLED] and not t[:2].any() and not r[:2].any()
    t2, r2, st2 = po.replay_paths(ref, [0, 2, 3], hops[2:], tok1[2:], kind[1:], amount[1:])
    assert np.array_equal(t[2:], t2) and np.array_equal(r[2:], r2) and np.array_equal(st[1:], st2)
    for i in pools:
        assert np.array_equal(getattr(pools[i], "R", None), getattr(ref[i], "R", None))
        assert getattr(pools[i], "price", 0) == getattr(ref[i], "price", 0)


# ---- the Router, through an oracle-backed stand-in -----------------------------------------
class PathPools(OrderPools):
    """OrderPools with the paths of the mirror; keeps each type's ingest token pairs."""

    def __init__(self, n_tokens, device=0):
        super().__init__(n_tokens, device)
        self.Ai = {0: np.zeros((0, 2), int), 1: np.zeros((0, 2), int), 2: np.zeros((0, 2), int)}

    def add_product(self, R, gamma, Ai):
        super().add_product(R, gamma, Ai)
        self.Ai[0] = np.array(Ai).reshape(-1, 2)

    def add_geomean(self, R, gamma, Ai, w):
        super().add_geomean(R, gamma, Ai, w)
        self.Ai[1] = np.array(Ai).reshape(-1, 2)

    def add_univ3(self, cp, gamma, Ai, off, lt, lq):
        super().add_univ3(cp, gamma, Ai, off, lt, lq)
        self.Ai[2] = np.array(Ai).reshape(-1, 2)

    def _paths(self, hop_off, hop_type, hop_pool, token_in, kind, amount, limit, execute):
        keys = [(int(t), int(i)) for t, i in zip(hop_type, hop_pool)]
        objs = {k: self._pool(*k) for k in set(keys)}
        tok1 = []
        for j in range(len(hop_off) - 1):
            s = keys[hop_off[j]:hop_off[j + 1]]
            sides = po.hop_sides([self.Ai[t][i] for t, i in s], token_in[j])
            assert sides is not None
            tok1 += sides
        fn = po.replay_paths if execute else po.quote_paths
        args = (objs, hop_off, keys, tok1, kind, amount) + ((limit,) if execute else ())
        out = fn(*args)
        if execute:
            for (t, i), p in objs.items():
                if t == 2:
                    self.cp[i] = p.price
                else:
                    self.R[t][i] = p.R
        return out

    def quote_paths(self, hop_off, hop_type, hop_pool, token_in, kind, amount):
        return self._paths(hop_off, hop_type, hop_pool, token_in, kind, amount, None, False)

    def execute_paths(self, hop_off, hop_type, hop_pool, token_in, kind, amount, limit=None):
        return self._paths(hop_off, hop_type, hop_pool, token_in, kind, amount, limit, True)


def random_walks(pools, rng, q, max_hops=4):
    """q paths as lists of list positions: random walks on the token graph, distinct pools."""
    paths, starts = [], []
    by_token = {}
    for i, c in enumerate(pools):
        for t in c.Ai:
            by_token.setdefault(int(t), []).append(i)
    while len(paths) < q:
        t0 = int(rng.choice(sorted(by_token)))
        t, path = t0, []
        for _ in range(int(rng.integers(1, max_hops + 1))):
            nxt = [i for i in by_token[t] if i not in path]
            if not nxt:
                break
            i = int(rng.choice(nxt))
            path.append(i)
            a, b = (int(v) for v in pools[i].Ai)
            t = b if t == a else a
        if path:
            paths.append(path)
            starts.append(t0)
    return paths, starts


def test_router_paths_map_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=PathPools)
    rng = np.random.default_rng(5)
    q = 30
    paths, starts = random_walks(pools, rng, q)
    kinds = rng.integers(0, 2, size=q)
    amounts = 10.0 ** rng.uniform(-2, 1, size=q)
    paid, got, st, ht, hr = r.quote_paths(paths, starts, kinds, amounts)
    off = np.concatenate([[0], np.cumsum([len(p) for p in paths])])
    assert len(ht) == off[-1] and np.array_equal(paid[st == 0], ht[off[:-1]][st == 0])
    assert np.array_equal(got, hr[off[1:] - 1])
    # each path quoted on its own, one at a time, gives the same
    for j in range(q):
        p1, g1, s1, _, _ = r.quote_paths([paths[j]], [starts[j]], [kinds[j]], [amounts[j]])
        assert p1[0] == paid[j] and g1[0] == got[j] and s1[0] == st[j]
    before = [c.R.copy() if hasattr(c, "R") else c.current_price for c in pools]
    limits = np.where(kinds == 1, paid * 10.0 ** rng.uniform(-0.01, 0.02, size=q),
                      got * 10.0 ** rng.uniform(-0.02, 0.01, size=q))
    paid, got, st, ht, hr = r.execute_paths(paths, starts, kinds, amounts, limits)
    assert {0, 1} <= set(st.tolist())
    filled = {i for j in np.flatnonzero(st == 0) for i in paths[j]}
    state = r._pools
    for i, c in enumerate(pools):
        t = [cr.ProductTwoCoin, cr.GeometricMeanTwoCoin, cr.UniV3].index(type(c))
        k = r._type_lists[t].index(i)
        if t == 2:
            assert c.current_price == state.cp[k]
            assert c.current_tick == int(np.sum(c.lower_ticks >= c.current_price))
            changed = c.current_price != before[i]
        else:
            assert np.array_equal(c.R, state.R[t][k])
            changed = not np.array_equal(c.R, before[i])
        assert changed <= (i in filled)


def test_router_path_argument_checks(cr):
    n = 6
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=PathPools)
    with pytest.raises(ValueError):
        r.quote_paths([[0], [1]], [1], [0, 0], [1.0, 1.0])
    with pytest.raises(ValueError):
        r.execute_paths([[0]], [1], [0], [1.0], limits=[0.0, 1.0])
    with pytest.raises(IndexError):
        r.quote_paths([[15]], [1], [0], [1.0])
    with pytest.raises(IndexError):
        r.execute_paths([[0, -1]], [1], [0], [1.0])
    paid, got, st, ht, hr = r.quote_paths([], [], [], [])
    assert paid.shape == got.shape == st.shape == ht.shape == hr.shape == (0,)
    r._world = 2  # a multi-GPU Router
    with pytest.raises(NotImplementedError):
        r.quote_paths([[0]], [1], [0], [1.0])
    with pytest.raises(NotImplementedError):
        r.execute_paths([[0]], [1], [0], [1.0])
