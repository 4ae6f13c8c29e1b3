"""Orders routed over their pair and two-hop routes through hub tokens (cfmm_quote_routed_orders /
cfmm_execute_routed_orders) on the host, without a GPU.

The mirror in route_oracle.py is checked against split orders' mirror (no hubs, or hubs that hold no
pools: bit for bit), against the two-hop path composition of path_oracle.py (one {j, h} and one
{h, i} pool), against route() (scipy L-BFGS-B over the oracle's sweeps) with the reference's Swap
objective on exactly the row's pools, for its hub surplus and evaluation bounds, and for the
in-order replay with limits.  The Router methods are checked through an oracle-backed stand-in for
DevicePools."""
import numpy as np
import pytest

import path_oracle as po
import route_oracle as ro
import split_oracle as so
import swap_order_oracle as oo
from swap_order_oracle import from_ordinal, ordinal
from test_split_orders_host import SplitPools, feasible, random_pair_pools
from test_swaps_host import market

EPS = np.finfo(np.float64).eps


def clone(ps):
    out = []
    for p in ps:
        if isinstance(p, so.Univ3):
            c = so.Univ3(p.price, p.lt, p.lq, p.g, p.Ai)
        elif isinstance(p, so.GeoMean):
            c = so.GeoMean(p.R, p.g, p.w, p.Ai)
        else:
            c = so.Product(p.R, p.g, p.Ai)
        c.active = p.active
        out.append(c)
    return out


def same_row(a, b):
    for k in ("paid", "received", "price", "status"):
        assert a[k] == b[k] or (np.isnan(a[k]) and np.isnan(b[k])), k
    assert np.array_equal(a["D"][:len(b["D"])], b["D"]) and np.array_equal(a["L"][:len(b["L"])], b["L"])


# ---- no hubs: split orders' bits ---------------------------------------------------------------
def test_no_hubs_and_empty_hubs_equal_the_split():
    rng = np.random.default_rng(21)
    for k in range(60):
        pools = random_pair_pools(rng, int(rng.integers(1, 7)), types=((0, 1, 2), (0,), (2,))[k % 3])
        if k % 7 == 0:
            pools[0].active = False
        tin, tout = (1, 2) if k % 2 else (2, 1)
        kind = int(rng.integers(0, 2))
        amount = float(10.0 ** rng.uniform(-4, 3)) if k % 11 else float(10.0 ** rng.uniform(5, 300))
        ref = so.split_row(clone(pools), tin, tout, kind, amount)
        same_row(ro.route_row(clone(pools), [], tin, tout, kind, amount), ref)
        # hubs 3 and 4 hold no pools of the row (t_h = DBL_MIN, no legs)
        row = ro.route_row(clone(pools), [(3, [], []), (4, [], [])], tin, tout, kind, amount)
        same_row(row, ref)
        assert row["hub_surplus"] == [0.0, 0.0]
        if row["status"] == so.FILLED and amount > 0.0:
            assert row["hub_price"] == [so.DBL_MIN, so.DBL_MIN]
        # the same row executed changes the pools as the split does
        a, b = clone(pools), clone(pools)
        so.split_row(a, tin, tout, kind, amount, execute=True)
        ro.route_row(b, [(5, [], [])], tin, tout, kind, amount, execute=True)
        for x, y in zip(a, b):
            assert (x.price == y.price) if isinstance(x, so.Univ3) else np.array_equal(x.R, y.R)


# ---- one {j, h} pool and one {h, i} pool: the two-hop path ---------------------------------------
def test_single_two_hop_route_is_the_path():
    """Exact-in δ of j through pool A = {j, h} and pool B = {h, i}, no direct pool.  The route takes
    paid = N(s*) <= δ of j and passes A's output of h to B less the surplus H(t*) >= 0.  So the path
    of cfmm_quote_paths with tender δ receives at most what the route receives plus the value of what
    the route leaves unspent, which is below one ordinal of s and one of t:
        path(δ) − received <= s*·(N(pred s*) − N(s*)) + t*·(H(t*) − H(pred t*)) + ε,
    since j is worth s* of i at the margin and h worth t*; and received <= path(δ) + ε.  ε is the
    rounding of the two formulas (find_arb!'s legs against the swap's output), each a difference of
    reserves-sized terms: a few ulp of A's reserves in h, worth t*, plus a few of B's in i."""
    rng = np.random.default_rng(4)
    j, h, i = 2, 3, 1
    for trial in range(40):
        RA = np.exp(rng.uniform(3, 8)) * np.exp(rng.uniform(-0.2, 0.2, size=2))
        RB = np.exp(rng.uniform(3, 8)) * np.exp(rng.uniform(-0.2, 0.2, size=2))
        gA, gB = rng.choice([0.997, 0.9995]), rng.choice([0.997, 0.9995])
        A = so.Product(RA, gA, [j, h] if trial % 2 else [h, j])
        B = so.Product(RB, gB, [h, i] if trial % 3 else [i, h])
        delta = float(min(RA) * 10.0 ** rng.uniform(-4, -0.5))
        row = ro.route_row([], [(h, [A], [B])], j, i, ro.EXACT_IN, delta)
        assert row["status"] == ro.FILLED
        s, t = row["price"], row["hub_price"][0]
        # path(δ) through the same two pools
        pa = oo.ProductPool(A.R, A.g)
        pb = oo.ProductPool(B.R, B.g)
        x, lam, st = po.quote_path([pa, pb], po.hop_sides([A.Ai, B.Ai], j), ro.EXACT_IN, delta)
        path = lam[-1]
        dN = ro.hub_sums([A], [B], j, h, i, from_ordinal(ordinal(s) - 1), t)[0] - row["paid"]
        Hm = ro.hub_sums([A], [B], j, h, i, s, from_ordinal(ordinal(t) - 1))[2] if t > so.DBL_MIN else 0.0
        dH = row["hub_surplus"][0] - Hm
        assert row["hub_surplus"][0] >= 0.0 and dN >= 0.0 and dH >= 0.0
        rounding = 16 * EPS * (t * max(RA) + max(RB))
        bound = s * dN + t * dH + rounding
        assert path - row["received"] <= bound, (trial, path, row["received"], bound)
        assert row["received"] - path <= rounding, trial


# ---- route() on exactly the row's pools ----------------------------------------------------------
def hub_market(rng, hubs, direct=1, per_side=2):
    """ProductTwoCoin pools on i = 1, j = 2 and hubs 3 … : `direct` pools of {1, 2} and per_side pools
    of each {2, h} and {h, 1}, prices near a common ν, random orientation."""
    nu = {1: 1.0, 2: float(np.exp(rng.uniform(-0.5, 0.5)))}
    for h in hubs:
        nu[h] = float(np.exp(rng.uniform(-1, 1)))
    spec = [(2, 1)] * direct + [p for h in hubs for p in [(2, h)] * per_side + [(h, 1)] * per_side]
    pools = []
    for a, b in spec:
        Ai = [a, b] if rng.random() < 0.5 else [b, a]
        depth = rng.uniform(200, 2000)
        R = np.array([depth / nu[Ai[0]], depth / nu[Ai[1]]]) * np.exp(rng.uniform(-0.03, 0.03, size=2))
        pools.append((Ai, R))
    return pools


@pytest.mark.parametrize("objective", ["swap", "basket"])
def test_matches_route_on_the_row_pools(cr, objective):
    rng = np.random.default_rng(17 if objective == "swap" else 18)
    for trial in range(4):
        hubs = [3, 4, 5][:1 + trial % 3]
        spec = hub_market(rng, hubs, direct=trial % 2)
        n = 2 + len(hubs)
        cs = [cr.ProductTwoCoin(R, 0.997, Ai) for Ai, R in spec]
        delta = float(rng.uniform(1, 20))
        obj = cr.Swap(1, 2, delta, n) if objective == "swap" else cr.BasketLiquidation(1, [0.0, delta] + [0.0] * len(hubs))
        r = cr.Router(obj, cs, n, _pools_factory=SplitPools)
        cr.route(r, pgtol=1e-10, factr=1e1)
        psi = cr.netflows(r)
        mirror = {k: so.Product(c.R, c.gamma, c.Ai) for k, c in enumerate(cs)}
        of = lambda a, b: [k for k, c in enumerate(cs) if set(c.Ai) == {a, b}]
        order = of(2, 1) + [k for h in hubs for k in of(2, h) + of(h, 1)]
        row = ro.route_row([mirror[k] for k in of(2, 1)], [(h, [mirror[k] for k in of(2, h)],
                                                            [mirror[k] for k in of(h, 1)]) for h in hubs],
                           2, 1, ro.EXACT_IN, delta)
        assert row["status"] == ro.FILLED
        assert abs(row["received"] - psi[0]) <= 1e-5 * psi[0], (trial, row["received"], psi[0])
        assert abs(row["paid"] + psi[1]) <= 1e-5 * delta
        assert np.all(np.abs(psi[2:]) <= 1e-5 * delta), psi
        assert all(x >= 0.0 and x <= 1e-6 * delta for x in row["hub_surplus"])
        for pos, k in enumerate(order):
            assert feasible(cs[k], row["D"][pos], row["L"][pos])


# ---- hub surplus and evaluation bounds on random sets ----------------------------------------
def random_row(rng, nh, types):
    j, i = 1, 2
    direct = random_pair_pools(rng, int(rng.integers(0, 4)), types, a=j, b=i)
    hubs = []
    for h in range(3, 3 + nh):
        hubs.append((h, random_pair_pools(rng, int(rng.integers(0, 3)), types, a=j, b=h),
                     random_pair_pools(rng, int(rng.integers(0, 3)), types, a=h, b=i)))
    return direct, hubs


def test_hub_surplus_and_evaluation_bound():
    rng = np.random.default_rng(6)
    seen = {ro.FILLED: 0, ro.UNREACHABLE: 0}
    for k in range(36):
        types = ((0,), (2,), (0, 2))[k % 3]
        direct, hubs = random_row(rng, 1 + k % 3, types)
        kind = int(rng.integers(0, 2))
        amount = float(10.0 ** rng.uniform(-3, 1.5)) if k % 9 else 1e200
        tin, tout = 1, 2
        row = ro.route_row(direct, hubs, tin, tout, kind, amount)
        seen[row["status"]] = seen.get(row["status"], 0) + 1
        assert row["outer"] <= ro.MAX_OUTER
        assert all(x <= ro.MAX_INNER for x in row["inner"])
        if row["status"] == ro.FILLED:
            assert all(x >= 0.0 for x in row["hub_surplus"]), k
            if kind == ro.EXACT_IN:
                assert row["paid"] <= amount
            else:
                assert row["received"] >= amount
    assert seen[ro.FILLED] > 15 and seen[ro.UNREACHABLE] > 0


def test_univ3_ladders_cross_ticks():
    """UniV3 hub pools with orders deep enough to cross ticks: surplus >= 0 and the bound hold."""
    rng = np.random.default_rng(12)
    crossed = 0
    for k in range(10):
        direct, hubs = random_row(rng, 2, (2,))
        before = {id(p): p.price for _, A, B in hubs for p in A + B}
        row = ro.route_row(direct, hubs, 1, 2, ro.EXACT_IN, float(10.0 ** rng.uniform(0, 2.5)), execute=True)
        assert row["outer"] <= ro.MAX_OUTER and all(x <= ro.MAX_INNER for x in row["inner"])
        if row["status"] == ro.FILLED:
            assert all(x >= 0.0 for x in row["hub_surplus"])
            for _, A, B in hubs:
                for p in A + B:
                    lt = p.lt
                    crossed += int(np.sum(lt >= before[id(p)]) != np.sum(lt >= p.price))
    assert crossed > 0


# ---- limits and batch order --------------------------------------------------------------------
def test_replay_limits_and_reverts():
    rng = np.random.default_rng(8)
    spec = hub_market(rng, [3, 4], direct=1)
    base = [so.Product(R, 0.997, Ai) for Ai, R in spec]
    of = lambda ps, a, b: [p for p in ps if set(p.Ai) == {a, b}]
    hubs = lambda ps: [(h, of(ps, 2, h), of(ps, h, 1)) for h in (3, 4)]
    q = ro.route_row(of(clone(base), 2, 1), hubs(clone(base)), 2, 1, ro.EXACT_IN, 3.0)
    a = clone(base)
    r0 = ro.route_row(of(a, 2, 1), hubs(a), 2, 1, ro.EXACT_IN, 3.0, limit=q["received"], execute=True)
    assert r0["status"] == ro.FILLED and r0["received"] == q["received"]
    b = clone(base)
    r1 = ro.route_row(of(b, 2, 1), hubs(b), 2, 1, ro.EXACT_IN, 3.0,
                      limit=float(np.nextafter(q["received"], np.inf)), execute=True)
    assert r1["status"] == ro.LIMIT and r1["paid"] == 0.0 and not r1["D"].any() and r1["price"] == q["price"]
    assert all(np.array_equal(x.R, y.R) for x, y in zip(b, base))
    # exact-out: the maximum paid
    q2 = ro.route_row(of(clone(base), 2, 1), hubs(clone(base)), 2, 1, ro.EXACT_OUT, 2.0)
    c = clone(base)
    assert ro.route_row(of(c, 2, 1), hubs(c), 2, 1, ro.EXACT_OUT, 2.0, limit=q2["paid"], execute=True)["status"] == 0
    c = clone(base)
    lim = float(np.nextafter(q2["paid"], 0.0))
    assert ro.route_row(of(c, 2, 1), hubs(c), 2, 1, ro.EXACT_OUT, 2.0, limit=lim, execute=True)["status"] == ro.LIMIT
    # a filled row moves the pools, so the same row again gets less
    assert ro.route_row(of(a, 2, 1), hubs(a), 2, 1, ro.EXACT_IN, 3.0)["received"] < q["received"]
    # replay_routed runs the rows in batch order on the state the earlier ones left
    d = clone(base)
    pairs = lambda x, y: of(d, x, y)
    rows = ro.replay_routed(pairs, [2, 2, 1], [1, 1, 2], [0, 0, 1], [3.0, 3.0, 1.0], [0, 2, 2, 2], [3, 4], [0.0, 0.0, 1e9])
    e = clone(base)
    one = [ro.route_row(of(e, 2, 1), hubs(e), 2, 1, 0, 3.0, execute=True),
           ro.route_row(of(e, 2, 1), [], 2, 1, 0, 3.0, execute=True),
           ro.route_row(of(e, 1, 2), [], 1, 2, 1, 1.0, limit=1e9, execute=True)]
    for x, y in zip(rows, one):
        same_row(x, y)
    assert all(np.array_equal(x.R, y.R) for x, y in zip(d, e))


# ---- the Router, through an oracle-backed stand-in -----------------------------------------
class RoutePools(SplitPools):
    """SplitPools with the routed orders of the mirror."""

    def _routed(self, execute, tin, tout, kind, amount, hub_off, hubs, limit):
        objs = self._objs()
        pairs = lambda a, b: [objs[k] for k in self._keys(a, b)]
        if execute:
            rows = ro.replay_routed(pairs, tin, tout, kind, amount, hub_off, hubs, limit)
            for (t, i), p in objs.items():
                if t == 2:
                    self.cp[i] = p.price
                else:
                    self.R[t][i] = p.R
        else:
            rows = ro.quote_routed(pairs, tin, tout, kind, amount, hub_off, hubs)
        out = tuple(np.array([r[k] for r in rows], dtype=np.uint8 if k == "status" else float).reshape(-1)
                    for k in ("paid", "received", "price", "status"))
        return out + (np.array([x for r in rows for x in r["hub_price"]]),
                      np.array([x for r in rows for x in r["hub_surplus"]]))

    def quote_routed_orders(self, tin, tout, kind, amount, hub_off, hubs):
        return self._routed(False, tin, tout, kind, amount, hub_off, hubs, None)

    def execute_routed_orders(self, tin, tout, kind, amount, hub_off, hubs, limit=None):
        return self._routed(True, tin, tout, kind, amount, hub_off, hubs, limit)


def test_router_routed_hubs_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=RoutePools)
    tin, tout = np.array([1, 2, 3, 4]), np.array([2, 3, 1, 5])
    kinds, amounts = np.array([0, 1, 0, 1]), np.full(4, 0.3)
    per_row = [[h for h in (6, 5, 4) if h not in (a, b)] for a, b in zip(tin, tout)]
    with pytest.raises(ValueError):
        r.quote_routed_orders(tin, tout, kinds, amounts, [[6]])  # one list per row needs q lists
    out = r.quote_routed_orders(tin, tout, kinds, amounts, per_row)
    for j in range(4):  # each row on its own gives the same
        one = r.quote_routed_orders(tin[j:j + 1], tout[j:j + 1], kinds[j:j + 1], amounts[j:j + 1], per_row[j])
        assert [x[0] for x in one] == [out[k][j] for k in range(4)]
    # no hubs: split orders
    assert all(np.array_equal(x, y) for x, y in zip(r.quote_routed_orders(tin, tout, kinds, amounts, []),
                                                    r.quote_split_orders(tin, tout, kinds, amounts)))
    before = [c.R.copy() if hasattr(c, "R") else c.current_price for c in pools]
    paid, got, price, st = r.execute_routed_orders(tin, tout, kinds, amounts, per_row)
    assert ro.FILLED in st.tolist()
    touched = set()
    for j in np.flatnonzero(st == ro.FILLED):
        touched |= set(r.pair_pools(tin[j], tout[j]).tolist())
        for h in per_row[j]:
            touched |= set(r.pair_pools(tin[j], h).tolist()) | set(r.pair_pools(h, tout[j]).tolist())
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
    r._world = 2  # a multi-GPU Router
    for call in (lambda: r.quote_routed_orders([1], [2], [0], [1.0], [3]),
                 lambda: r.execute_routed_orders([1], [2], [0], [1.0], [3])):
        with pytest.raises(NotImplementedError):
            call()
