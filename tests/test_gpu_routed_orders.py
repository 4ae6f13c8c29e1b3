"""cfmm_quote_routed_orders / cfmm_execute_routed_orders (include/cfmm_b200.h) on the device.

A hub-structured pool set: hub tokens 1, 2, 3 each paired with every other token by one or two
pools, and sparse direct pools between the other tokens, as a main set and appended pools per type,
some retired.  Quotes and executes are checked bit for bit against the host mirror (route_oracle.py)
on ProductTwoCoin, UniV3 and mixed sets; rows without hubs against cfmm_quote_split_orders /
cfmm_execute_split_orders; every type, GeometricMeanTwoCoin included, against a fresh context
holding only the row's pools (a materialising cfmm_sweep at the row's ν, cfmm_apply_trades); and
the result against the split, the two-hop paths and cfmm_solve."""
import numpy as np
import pytest

import oracle_lib
import route_oracle as ro
import split_oracle as so
from test_gpu_paths import APPEND, same_state
from test_gpu_parity import make_pools
from test_gpu_split_orders import compare, expected_pairs
from test_gpu_swap_orders import univ3_host_pools

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
HUBS = (1, 2, 3)


class HubSet:
    """The attributes test_gpu_split_orders' helpers read (n, mm, mt, main, tail, Ai, g, w, m, retired,
    p, fresh, state) for a hub-structured set of the given types."""

    def __init__(self, cr, synth, types, seed, n=14, tail=0.25, retire=True):
        rng = np.random.default_rng(seed)
        self._cr, self.n = cr, n
        nu = np.exp(rng.uniform(-1, 1, size=n + 1))
        spec = [(h, x) for h in HUBS for x in range(4, n + 1) for _ in range(int(rng.integers(1, 3)))]
        spec += [tuple(rng.choice(np.arange(4, n + 1), size=2, replace=False)) for _ in range(n)]
        by = {t: [] for t in (P, G, U)}
        for a, b in spec:
            Ai = [int(a), int(b)] if rng.random() < 0.5 else [int(b), int(a)]
            by[types[int(rng.integers(0, len(types)))]].append(Ai)
        self.main, self.tail, self.Ai, self.g, self.mm, self.mt = {}, {}, {}, {}, {}, {}
        self.w = np.zeros((0, 2))
        for t in (P, G, U):
            A = np.array(by[t], dtype=np.int64).reshape(-1, 2)
            m = len(A)
            depth = rng.uniform(200, 5000, size=m)
            noise = np.exp(rng.uniform(-0.05, 0.05, size=(m, 2)))
            R = depth[:, None] / nu[A] * noise
            g = rng.choice([0.997, 0.9995, 1.0], size=m) if t == P else np.full(m, 0.997)
            if t == G:
                self.w = rng.uniform(0.3, 0.7, size=(m, 2))
                data = [R, g, A, self.w]
            elif t == U:
                cp, gu, _, off, lt, lq = synth.univ3_pools(max(m, 1), 2, seed=seed + 5, ragged=True)
                cp, off = cp[:m], off[:m + 1]
                lt, lq = lt[:off[-1]].copy(), lq[:off[-1]].copy()
                target = nu[A[:, 0]] / nu[A[:, 1]] * np.exp(rng.uniform(-0.05, 0.05, size=m))
                for i in range(m):
                    lt[off[i]:off[i + 1]] *= target[i] / cp[i]
                    lq[off[i]:off[i + 1]] *= depth[i] / 100.0
                data = [target, gu[:m], A, off, lt, lq]
            else:
                data = [R, g, A]
            self.Ai[t], self.g[t] = A, data[1]
            k = m - int(round(m * tail))
            self.mm[t], self.mt[t] = k, m - k
            if t == U:
                o1 = off[k]
                self.main[t] = (data[0][:k], data[1][:k], A[:k], off[:k + 1], lt[:o1], lq[:o1])
                self.tail[t] = (data[0][k:], data[1][k:], A[k:], off[k:] - o1, lt[o1:], lq[o1:])
            else:
                self.main[t] = tuple(x[:k] for x in data)
                self.tail[t] = tuple(x[k:] for x in data)
        self.m = {t: self.mm[t] + self.mt[t] for t in (P, G, U)}
        self.retired = set()
        if retire:
            for t in (P, G, U):
                if self.m[t] > 8:
                    self.retired |= {(t, int(i)) for i in rng.choice(self.m[t], size=3, replace=False)}
        self.p = self.fresh()

    def fresh(self):
        kw = {("product", "geomean", "univ3")[t]: self.main[t] for t in (P, G, U) if self.mm[t]}
        p = make_pools(self._cr, self.n, pre={"orient_by_degree": 1}, **kw)
        for t in (P, G, U):
            if self.mt[t]:
                getattr(p, APPEND[t])(*self.tail[t])
            if self.m[t]:
                act = np.ones(self.m[t], bool)
                act[[i for (s, i) in self.retired if s == t]] = False
                p.set_active(t, 0, act)
        return p

    def state(self, p):
        return [p.pool_state(t)[0].copy() for t in (P, G, U) if self.m[t]] + \
            (list(p.univ3_ticks()) if self.m[U] else [])


def keys_of(hs):
    return [k for t in (P, G, U) for k in [(t, i) for i in range(hs.mm[t])]] + \
        [(t, hs.mm[t] + i) for t in (P, G, U) for i in range(hs.mt[t])]


def rows(rng, hs, q, max_hubs=3):
    tin = rng.integers(4, hs.n + 1, size=q)
    tout = np.array([rng.choice([x for x in range(4, hs.n + 1) if x != a]) for a in tin])
    per = [list(rng.permutation(HUBS)[:int(rng.integers(0, max_hubs + 1))]) for _ in range(q)]
    hub_off = np.concatenate([[0], np.cumsum([len(h) for h in per])]).astype(np.int64)
    hubs = np.array([h for x in per for h in x], dtype=np.int64)
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    amount = 10.0 ** rng.uniform(-2, 2, size=q)
    amount[::13] = 0.0
    return tin.astype(np.int64), tout.astype(np.int64), kind, amount, hub_off, hubs


def mirror_pools(hs, p):
    """route_oracle's pools at the device's state, keyed (type, index), retired ones inactive."""
    out = {}
    if hs.m[P]:
        st, _ = p.pool_state(P)
        for i in range(hs.m[P]):
            out[(P, i)] = so.Product(st[i], hs.g[P][i], hs.Ai[P][i])
    if hs.m[G]:
        st, _ = p.pool_state(G)
        for i in range(hs.m[G]):
            out[(G, i)] = so.GeoMean(st[i], hs.g[G][i], hs.w[i], hs.Ai[G][i])
    if hs.m[U]:
        for i, h in enumerate(univ3_host_pools(p, hs.g[U])):
            out[(U, i)] = so.Univ3(h.price, h.lt, h.lq, h.g, hs.Ai[U][i])
    for k in hs.retired:
        out[k].active = False
    return out


def mirror_of(hs, p):
    objs = mirror_pools(hs, p)
    keys = keys_of(hs)
    return objs, (lambda a, b: [objs[k] for k in expected_pairs(hs, keys, a, b)])


def check(dev, rws, hub_off):
    paid, got, price, st, hp, hsur, (o, D, L) = dev
    compare((paid, got, price, st, (o, D, L)), rws, o)
    for r, row in enumerate(rws):
        g = slice(int(hub_off[r]), int(hub_off[r + 1]))
        assert hp[g].tolist() == row["hub_price"] and hsur[g].tolist() == row["hub_surplus"], r
        if row["status"] == so.FILLED:
            assert np.all(hsur[g] >= 0.0)


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U)], ids=["product", "univ3", "mixed"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=40 + len(request.param) + request.param[0])
    yield hs
    hs.p.close()


def test_bit_exact_against_mirror(hset):
    rng = np.random.default_rng(3)
    tin, tout, kind, amount, hub_off, hubs = rows(rng, hset, 16)
    dev = hset.p.quote_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    _, pairs = mirror_of(hset, hset.p)
    rws = ro.quote_routed(pairs, tin, tout, kind, amount, hub_off, hubs)
    assert so.FILLED in {r["status"] for r in rws}
    assert max(r["outer"] for r in rws) <= ro.MAX_OUTER
    check(dev, rws, hub_off)
    # execute on a fresh copy, in batch order, with limits around the quotes (some revert)
    p = hset.fresh()
    lim = np.where(kind == 1, dev[0] * 1.0000001 + 1e-9, dev[1] * 0.9999999)
    lim[::5] = np.where(kind[::5] == 1, 0.0, 1e300)
    out = p.execute_routed_orders(tin, tout, kind, amount, hub_off, hubs, np.maximum(lim, 0.0), legs=True)
    objs, pairs = mirror_of(hset, hset.p)
    rws = ro.replay_routed(pairs, tin, tout, kind, amount, hub_off, hubs, np.maximum(lim, 0.0))
    check(out, rws, hub_off)
    after = mirror_pools(hset, p)
    for k, o in objs.items():
        assert (after[k].price == o.price) if k[0] == U else np.array_equal(after[k].R, o.R), k
    p.close()


@pytest.fixture(scope="module")
def allset(cr, synth):
    hs = HubSet(cr, synth, (P, G, U), seed=77)
    yield hs
    hs.p.close()


def test_zero_hubs_equal_split(allset):
    rng = np.random.default_rng(5)
    tin, tout, kind, amount, _, _ = rows(rng, allset, 40)
    tin[:20] = rng.integers(1, 4, size=20)  # hub-token pairs hold pools
    tout[:20] = np.where(tout[:20] == tin[:20], 5, tout[:20])
    none = np.zeros(len(tin) + 1, dtype=np.int64)
    a = allset.p.quote_routed_orders(tin, tout, kind, amount, none, [], legs=True)
    b = allset.p.quote_split_orders(tin, tout, kind, amount, legs=True)
    assert all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4]))
    assert all(np.array_equal(x, y) for x, y in zip(a[6], b[4]))
    p, q = allset.fresh(), allset.fresh()
    a = p.execute_routed_orders(tin, tout, kind, amount, none, [], legs=True)
    b = q.execute_split_orders(tin, tout, kind, amount, legs=True)
    assert all(np.array_equal(x, y) for x, y in zip(a[:4], b[:4]))
    assert all(np.array_equal(x, y) for x, y in zip(a[6], b[4]))
    assert same_state(allset.state(p), allset.state(q))
    p.close()
    q.close()


def row_context(cr, hs, p, keys, tmap):
    """A fresh context holding the active pools keys (state of p), tokens renamed by tmap."""
    c = cr.DevicePools(len(tmap))
    by = {t: [i for (s, i) in keys if s == t] for t in (P, G, U)}
    ren = lambda t, ids: np.array([[tmap[int(x)] for x in hs.Ai[t][i]] for i in ids], dtype=np.int64)
    if by[P]:
        c.add_product(p.pool_state(P)[0][by[P]], hs.g[P][by[P]], ren(P, by[P]))
    if by[G]:
        c.add_geomean(p.pool_state(G)[0][by[G]], hs.g[G][by[G]], ren(G, by[G]), hs.w[by[G]])
    if by[U]:
        st = p.pool_state(U)[0]
        off, lt, lq = p.univ3_ticks()
        ids = by[U]
        o = np.concatenate([[0], np.cumsum([off[i + 1] - off[i] for i in ids])]).astype(np.int64)
        c.add_univ3(st[ids], hs.g[U][ids], ren(U, ids), o, np.concatenate([lt[off[i]:off[i + 1]] for i in ids]),
                    np.concatenate([lq[off[i]:off[i + 1]] for i in ids]))
    c.finalize()
    return c, [(t, i) for t in (P, G, U) for i in by[t]]


def row_keys(hs, keys, j, i, hubs):
    lists = [expected_pairs(hs, keys, j, i)]
    for h in hubs:
        lists += [expected_pairs(hs, keys, j, h), expected_pairs(hs, keys, h, i)]
    return [k for x in lists for k in x]


def test_bit_exact_against_sweep_and_apply(cr, allset):
    """Each filled row = a materialising sweep at its ν on its pools alone + cfmm_apply_trades."""
    rng = np.random.default_rng(9)
    tin, tout, kind, amount, hub_off, hubs = rows(rng, allset, 10)
    keys = keys_of(allset)
    p = allset.fresh()
    for r in range(len(tin)):
        hr = [int(h) for h in hubs[hub_off[r]:hub_off[r + 1]]]
        rk = row_keys(allset, keys, int(tin[r]), int(tout[r]), hr)
        live = [k for k in rk if k not in allset.retired]
        tmap = {int(tout[r]): 1, int(tin[r]): 2, **{h: 3 + x for x, h in enumerate(hr)}}
        if live:
            ctx, order = row_context(cr, allset, p, live, tmap)
        one = p.execute_routed_orders(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], [0, len(hr)], hr,
                                      legs=True)
        if one[3][0] != so.FILLED or amount[r] == 0.0:
            if live:
                ctx.close()
            continue
        v = np.array([1.0, one[2][0]] + one[4].tolist())
        ctx.sweep(v, materialize=True)
        D, L = ctx.trades()
        for k, key in enumerate(rk):
            if key in allset.retired:
                assert not one[6][1][k].any() and not one[6][2][k].any()
                continue
            g = order.index(key)
            assert np.array_equal(one[6][1][k], D[g]) and np.array_equal(one[6][2][k], L[g]), (r, key)
        ctx.apply_trades()
        for t in (P, G, U):
            ids = [i for (s, i) in order if s == t]
            if ids:
                assert np.array_equal(ctx.pool_state(t)[0], p.pool_state(t)[0][ids]), (r, t)
        ctx.close()
    p.close()


def test_optimal_against_split_paths_and_solve(cr, allset):
    rng = np.random.default_rng(13)
    tin, tout, kind, amount, hub_off, hubs = rows(rng, allset, 12, max_hubs=3)
    kind[:] = 0
    amount[:] = 10.0 ** rng.uniform(-1, 1.5, size=len(tin))
    p = allset.p
    paid, got, price, st, hp, _ = p.quote_routed_orders(tin, tout, kind, amount, hub_off, hubs)
    sp = p.quote_split_orders(tin, tout, kind, amount)
    keys = keys_of(allset)
    converged = 0
    tol = 1e-9  # (a neighbouring ordinal of s or t_h moves received by far less; GeometricMean's pow: a few ulp)
    for r in np.flatnonzero(st == so.FILLED):
        if sp[3][r] == so.FILLED:
            assert got[r] >= sp[1][r] * (1 - tol), r
        j, i = int(tin[r]), int(tout[r])
        for h in hubs[hub_off[r]:hub_off[r + 1]]:
            for a in expected_pairs(allset, keys, j, int(h)):
                for b in expected_pairs(allset, keys, int(h), i):
                    if a in allset.retired or b in allset.retired:
                        continue
                    out = p.quote_paths([0, 2], [a[0], b[0]], [a[1], b[1]], [j], [0], [amount[r]])
                    if out[2][0] == so.FILLED:
                        assert got[r] >= out[1][1] * (1 - tol), (r, a, b)
        # cfmm_solve with BasketLiquidation on a fresh context of the row's pools
        hr = [int(h) for h in hubs[hub_off[r]:hub_off[r + 1]]]
        live = [k for k in row_keys(allset, keys, j, i, hr) if k not in allset.retired]
        tmap = {i: 1, j: 2, **{h: 3 + x for x, h in enumerate(hr)}}
        ctx, order = row_context(cr, allset, p, live, tmap)
        d = len(tmap)
        lin = np.zeros(d)
        lin[1] = amount[r]
        lower = np.full(d, 1e-12)
        lower[0] = 1.0
        v0 = np.array([1.0, price[r]] + hp[hub_off[r]:hub_off[r + 1]].tolist())
        nu, info = ctx.solve(lower, lin=lin, v0=v0 * 1.01, pgtol=1e-10)
        D, L = ctx.trades()
        psi = np.zeros(d)
        for g, (t, k) in enumerate(order):
            for s, x in enumerate(allset.Ai[t][k]):
                psi[tmap[int(x)] - 1] += L[g, s] - D[g, s]
        # The solver's iterate meets the order's constraints (Ψ_j = −δ, Ψ_h = 0) only up to a residual,
        # worth s* and t_h* of i each at the margin.  The route does at least as well as the iterate less
        # that; where the residual is negligible the two agree within 1e-5.
        slack = price[r] * abs(psi[1] + amount[r]) + float(np.dot(hp[hub_off[r]:hub_off[r + 1]], np.abs(psi[2:])))
        assert got[r] >= psi[0] * (1 - 1e-5) - slack, (r, got[r], psi[0], slack)
        if slack <= 1e-6 * psi[0]:
            assert abs(got[r] - psi[0]) <= 1e-5 * psi[0], (r, got[r], psi[0])
            converged += 1
        ctx.close()
    assert converged >= 1


def test_batch_equals_one_call_per_row(allset):
    rng = np.random.default_rng(21)
    # a block of rows sharing a hub pair (one level each) and a wide block on distinct pairs
    q1 = 12
    tin = np.array([4] * q1 + list(range(4, 4 + 5)), dtype=np.int64)
    tout = np.array([5] * q1 + list(range(9, 9 + 5)), dtype=np.int64)
    per = [[1, 2]] * q1 + [[]] * 5
    hub_off = np.concatenate([[0], np.cumsum([len(h) for h in per])]).astype(np.int64)
    hubs = np.array([h for x in per for h in x], dtype=np.int64)
    kind = rng.integers(0, 2, size=len(tin)).astype(np.uint8)
    amount = 10.0 ** rng.uniform(-1, 1, size=len(tin))
    p, q = allset.fresh(), allset.fresh()
    out = p.execute_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    for r in range(len(tin)):
        h = hubs[hub_off[r]:hub_off[r + 1]]
        one = q.execute_routed_orders(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], [0, len(h)], h,
                                      legs=True)
        assert [x[0] for x in one[:4]] == [out[k][r] for k in range(4)], r
        assert one[4].tolist() == out[4][hub_off[r]:hub_off[r + 1]].tolist()
        o = out[6][0]
        assert np.array_equal(one[6][1], out[6][1][o[r]:o[r + 1]]) and np.array_equal(one[6][2], out[6][2][o[r]:o[r + 1]])
    assert same_state(allset.state(p), allset.state(q))
    p.close()
    q.close()


def test_compact_and_liquidity_changes(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=91)
    p = hs.p
    # compact (retired pools stay retired and keep their place in the insertion order), then change a ladder
    p.compact()
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:3]
    st = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, st[ui] * 0.9, st[ui] * 1.1, np.full(len(ui), 500.0))
    rng = np.random.default_rng(2)
    tin, tout, kind, amount, hub_off, hubs = rows(rng, hs, 10)
    dev = p.quote_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    _, pairs = mirror_of(hs, p)
    check(dev, ro.quote_routed(pairs, tin, tout, kind, amount, hub_off, hubs), hub_off)
    objs, pairs = mirror_of(hs, p)
    out = p.execute_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    check(out, ro.replay_routed(pairs, tin, tout, kind, amount, hub_off, hubs), hub_off)
    # a gradient sweep on the new state matches the oracle
    after = mirror_pools(hs, p)
    for k, o in objs.items():
        assert (after[k].price == o.price) if k[0] == U else np.array_equal(after[k].R, o.R), k
    v = np.exp(np.random.default_rng(4).uniform(-1, 1, size=hs.n))
    psi, _ = p.sweep(v, materialize=False)
    o = oracle_lib.load()
    ref = np.zeros(hs.n)
    D, L = o.sweep_product(p.pool_state(P)[0], hs.g[P], hs.Ai[P], v)
    act = np.array([(P, i) not in hs.retired for i in range(hs.m[P])])
    np.add.at(ref, hs.Ai[P][act] - 1, (L - D)[act])
    off, lt, lq = p.univ3_ticks()
    D, L = o.sweep_univ3(p.pool_state(U)[0], hs.g[U], hs.Ai[U], off, lt, lq, v)
    act = np.array([(U, i) not in hs.retired for i in range(hs.m[U])])
    np.add.at(ref, hs.Ai[U][act] - 1, (L - D)[act])
    assert np.allclose(psi, ref, rtol=1e-9, atol=1e-9 * np.max(np.abs(ref)))
    p.close()


def test_rejections_change_nothing(cr, allset):
    p = allset.fresh()
    before = allset.state(p)
    ok = dict(tin=[4], tout=[5], kind=[0], amount=[1.0], hub_off=[0, 1], hubs=[1])
    bad = [dict(hubs=[4]), dict(hubs=[5]), dict(hubs=[0]), dict(hubs=[allset.n + 1]),
           dict(hub_off=[0, 2], hubs=[1, 1]), dict(hub_off=[0, 8], hubs=[1] * 8), dict(hub_off=[1, 1], hubs=[1]),
           dict(tin=[5]), dict(tin=[0]), dict(kind=[2]), dict(amount=[np.nan]), dict(amount=[-1.0]),
           dict(amount=[np.inf])]
    for b in bad:
        a = {**ok, **b}
        with pytest.raises((cr.CFMMError, ValueError)):
            p.execute_routed_orders(a["tin"], a["tout"], a["kind"], a["amount"], a["hub_off"], a["hubs"])
    for lim in ([np.nan], [-1.0], [np.inf]):
        with pytest.raises(cr.CFMMError) as e:
            p.execute_routed_orders([4], [5], [0], [1.0], [0, 1], [1], lim)
        assert e.value.code == -1
    assert same_state(before, allset.state(p))
    p.close()


def test_router_on_device(cr, synth):
    n = 8
    rng = np.random.default_rng(1)
    cs = []
    for a in range(1, n + 1):
        for b in range(a + 1, n + 1):
            if a <= 2 or rng.random() < 0.3:
                R = rng.uniform(500, 5000) * np.exp(rng.uniform(-0.1, 0.1, size=2))
                cs.append(cr.ProductTwoCoin(R, 0.997, [a, b]))
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), cs, n)
    tin, tout = np.array([3, 4, 5]), np.array([6, 7, 8])
    kinds, amounts = np.array([0, 1, 0]), np.array([2.0, 1.0, 3.0])
    q = r.quote_routed_orders(tin, tout, kinds, amounts, [1, 2])
    d = r._pools.quote_routed_orders(tin, tout, kinds, amounts, [0, 2, 4, 6], [1, 2] * 3)
    assert all(np.array_equal(x, y) for x, y in zip(q, d[:4]))
    out = r.execute_routed_orders(tin, tout, kinds, amounts, [[1, 2], [1], [2]])
    assert np.all(out[3] == so.FILLED)
    st = r._pools.pool_state(P)[0]
    for k, c in enumerate(cs):
        assert np.array_equal(c.R, st[r._type_lists[P].index(k)])
    r._pools.close()
