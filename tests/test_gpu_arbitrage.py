"""cfmm_scan_arbitrage / cfmm_quote_arbitrage / cfmm_execute_arbitrage (include/cfmm_b200.h) on the
device, on test_gpu_routed_orders' hub-structured sets (hub tokens 1, 2, 3 paired with every other
token by one or two mispriced pools, sparse pools between the others, appended and retired pools).

The scan, quotes and executes are checked bit for bit against the host mirror (arbitrage_oracle.py)
on ProductTwoCoin, UniV3 and mixed sets, also after a compact and a UniV3 liquidity change; every
filled row of every type against a fresh context's materialising sweep and cfmm_apply_trades; every
filled row against the 50-digit certificate at δ = 0; and the cycles closed after an execute."""
import ctypes as C

import numpy as np
import pytest

import arbitrage_certificate as ac
import arbitrage_oracle as ao
import order_certificate as oc
from test_gpu_paths import same_state
from test_gpu_routed_orders import HubSet, keys_of, mirror_pools, row_context
from test_gpu_split_orders import expected_pairs

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
BASES = [1, 5]
MIN_PROFIT = [1e-3, 1e-4]
N = 9  # tokens: the mirror's nested searches run in Python


def mirror(hs, p):
    """(by_pair {(lo, hi): pools}, pairs(a, b)) of route_oracle pools at p's state, pair order."""
    objs = mirror_pools(hs, p)
    by = {}
    for k in keys_of(hs):
        a, b = sorted(int(x) for x in hs.Ai[k[0]][k[1]])
        by.setdefault((a, b), []).append(objs[k])
    return objs, by, (lambda a, b: by.get((min(a, b), max(a, b)), []))


def scan_rows(dev):
    found, rb, ro, hub_off, hubs, profit, price = dev
    return found, [dict(base=int(rb[r]), other=int(ro[r]), hubs=hubs[hub_off[r]:hub_off[r + 1]].tolist(),
                        profit=float(profit[r]), price=float(price[r])) for r in range(len(rb))]


def check_scan(hs, p, max_hubs, caps=(None,), memo=None):
    """The device's scan against the mirror's, for each cap (the mirror runs once)."""
    _, by, pairs = mirror(hs, p)
    found, rows = ao.scan(by, pairs, BASES, MIN_PROFIT, max_hubs, None, memo)
    for cap in caps:
        dev = p.scan_arbitrage(BASES, MIN_PROFIT, max_hubs, cap)
        assert scan_rows(dev) == (found, rows if cap is None else rows[:cap]), (max_hubs, cap)
    return dev


def check_quotes(dev, rows):
    profit, surplus, price, st, hp, hsur, (o, D, L) = dev
    for r, row in enumerate(rows):
        assert st[r] == row["status"] and price[r] == row["price"], r
        assert profit[r] == row["profit"] and surplus[r] == row["surplus_in"], r
        assert np.array_equal(D[o[r]:o[r + 1]], row["D"]) and np.array_equal(L[o[r]:o[r + 1]], row["L"]), r


def check_hubs(dev, rows, hub_off):
    for r, row in enumerate(rows):
        g = slice(int(hub_off[r]), int(hub_off[r + 1]))
        assert dev[4][g].tolist() == row["hub_price"] and dev[5][g].tolist() == row["hub_surplus"], r
        if row["status"] == ao.FILLED:
            assert dev[1][r] >= 0.0 and np.all(dev[5][g] >= 0.0)


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U)], ids=["product", "univ3", "mixed"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=140 + len(request.param) + request.param[0], n=N)
    yield hs
    hs.p.close()


def test_scan_bit_exact_against_mirror(hset):
    memo = {}
    for mh in (0, 1, 3, 7):
        dev = check_scan(hset, hset.p, mh, memo=memo)
        assert dev[0] >= 1, mh
        if mh == 3:
            assert len(dev[4]) > 0, "no triangle row"
    full = hset.p.scan_arbitrage(BASES, MIN_PROFIT, 3)
    dev = check_scan(hset, hset.p, 3, caps=(0, 1, full[0] - 1), memo=memo)
    assert dev[0] == full[0] and len(dev[1]) == full[0] - 1


def test_quote_and_execute_bit_exact(hset):
    found, rb, ro, hub_off, hubs, profit, _ = hset.p.scan_arbitrage(BASES, MIN_PROFIT, 3)
    extra = np.array([4, 6], dtype=np.int64)  # rows the scan need not return: (1, 4) / (2, 6) without hubs
    base = np.concatenate([rb, [1, 2]]).astype(np.int64)
    other = np.concatenate([ro, extra]).astype(np.int64)
    off = np.concatenate([hub_off, [hub_off[-1]] * 2]).astype(np.int64)
    dev = hset.p.quote_arbitrage(base, other, off, hubs, legs=True)
    _, _, pairs = mirror(hset, hset.p)
    rows = ao.quote_arbitrage(pairs, base, other, off, hubs)
    check_quotes(dev, rows)
    check_hubs(dev, rows, off)
    assert np.array_equal(dev[0][:found], profit)
    # execute on a fresh copy in batch order: minimum profits around the quotes, some of which revert
    p = hset.fresh()
    mp = dev[0] * 0.5
    mp[::4] = dev[0][::4] * 2.0 + 1.0
    out = p.execute_arbitrage(base, other, off, hubs, np.maximum(mp, 0.0), legs=True)
    objs, _, pairs = mirror(hset, hset.p)
    rows = ao.replay_arbitrage(pairs, base, other, off, hubs, np.maximum(mp, 0.0))
    check_quotes(out, rows)
    check_hubs(out, rows, off)
    assert ao.LIMIT in set(out[3].tolist()) and ao.FILLED in set(out[3].tolist())
    after = mirror_pools(hset, p)
    for k, o in objs.items():
        assert (after[k].price == o.price) if k[0] == U else np.array_equal(after[k].R, o.R), k
    p.close()


def test_compact_and_liquidity_changes(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=191, n=N)
    p = hs.p
    check_scan(hs, p, 3)  # builds the adjacency
    p.compact()
    check_scan(hs, p, 3)
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:3]
    st = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, st[ui] * 0.9, st[ui] * 1.1, np.full(len(ui), 500.0))
    # retire and restore after the adjacency exists: the rates see it, the adjacency is kept
    act = np.ones(hs.m[P], bool)
    act[[i for (s, i) in hs.retired if s == P]] = False
    act[0] = False
    p.set_active(P, 0, act)
    hs.retired.add((P, 0))
    dev = check_scan(hs, p, 7)
    _, rb, ro, hub_off, hubs, _, _ = dev
    objs, _, pairs = mirror(hs, p)
    out = p.execute_arbitrage(rb, ro, hub_off, hubs, legs=True)
    rows = ao.replay_arbitrage(pairs, rb, ro, hub_off, hubs)
    check_quotes(out, rows)
    after = mirror_pools(hs, p)
    for k, o in objs.items():
        assert (after[k].price == o.price) if k[0] == U else np.array_equal(after[k].R, o.R), k
    p.close()


@pytest.fixture(scope="module")
def allset(cr, synth):
    hs = HubSet(cr, synth, (P, G, U), seed=177, n=N)
    yield hs
    hs.p.close()


def arb_keys(hs, keys, p, x, hr):
    lists = [expected_pairs(hs, keys, x, p)]
    for y in hr:
        lists += [expected_pairs(hs, keys, x, y), expected_pairs(hs, keys, y, p)]
    return [k for l in lists for k in l]


def test_bit_exact_against_sweep_and_apply(cr, allset):
    """Each filled row, every type = a materialising sweep at (ν_p = 1, ν_x = s*, ν_y = t_y*) on its
    pools alone + cfmm_apply_trades."""
    _, rb, ro, hub_off, hubs, _, _ = allset.p.scan_arbitrage(BASES, MIN_PROFIT, 3)
    keys = keys_of(allset)
    p = allset.fresh()
    kinds, done = set(), 0
    for r in range(min(len(rb), 8)):
        hr = [int(h) for h in hubs[hub_off[r]:hub_off[r + 1]]]
        b, x = int(rb[r]), int(ro[r])
        rk = arb_keys(allset, keys, b, x, hr)
        live = [k for k in rk if k not in allset.retired]
        tmap = {b: 1, x: 2, **{h: 3 + i for i, h in enumerate(hr)}}
        ctx, order = row_context(cr, allset, p, live, tmap)
        one = p.execute_arbitrage([b], [x], [0, len(hr)], hr, legs=True)
        if one[3][0] != ao.FILLED:
            ctx.close()
            continue
        ctx.sweep(np.array([1.0, one[2][0]] + one[4].tolist()), materialize=True)
        D, L = ctx.trades()
        for k, key in enumerate(rk):
            if key in allset.retired:
                assert not one[6][1][k].any() and not one[6][2][k].any()
                continue
            g = order.index(key)
            assert np.array_equal(one[6][1][k], D[g]) and np.array_equal(one[6][2][k], L[g]), (r, key)
            kinds.add(key[0])
        ctx.apply_trades()
        for t in (P, G, U):
            ids = [i for (s, i) in order if s == t]
            if ids:
                assert np.array_equal(ctx.pool_state(t)[0], p.pool_state(t)[0][ids]), (r, t)
        ctx.close()
        done += 1
    assert done >= 4 and kinds == {P, G, U}
    p.close()


def cert_pools(hs, p):
    out = {}
    for t in (P, G, U):
        if not hs.m[t]:
            continue
        st = p.pool_state(t)[0]
        if t == U:
            off, lt, lq = p.univ3_ticks()
        for i in range(hs.m[t]):
            act, Ai = (t, i) not in hs.retired, hs.Ai[t][i]
            if t == P:
                out[(t, i)] = oc.product(st[i], hs.g[t][i], Ai, act)
            elif t == G:
                out[(t, i)] = oc.geomean(st[i], hs.g[t][i], hs.w[i], Ai, act)
            else:
                out[(t, i)] = oc.univ3(st[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], hs.g[t][i], Ai, act)
    return out


def certify(hs, p, dev, base, other, hub_off, hubs):
    """Certify every row of dev (quote or execute outputs with legs) on p's current state."""
    keys = keys_of(hs)
    objs = cert_pools(hs, p)
    lst = lambda a, b: [objs[k] for k in expected_pairs(hs, keys, a, b)]
    profit, surplus, price, st, hp, hsur, (o, D, L) = dev
    res = []
    for r in range(len(base)):
        b, x = int(base[r]), int(other[r])
        hr = [int(h) for h in hubs[hub_off[r]:hub_off[r + 1]]]
        row = oc.Row(lst(x, b), [(h, lst(x, h), lst(h, b)) for h in hr], x, b)
        g = slice(int(hub_off[r]), int(hub_off[r + 1]))
        out = dict(profit=profit[r], surplus_in=surplus[r], price=price[r], status=st[r], hub_price=hp[g],
                   hub_surplus=hsur[g], D=D[o[r]:o[r + 1]], L=L[o[r]:o[r + 1]])
        res.append(ac.certify_arbitrage(row, out, nested=r < 2))
    return res


def test_certified_and_closed(allset):
    p = allset.fresh()
    _, rb, ro, hub_off, hubs, _, _ = p.scan_arbitrage(BASES, MIN_PROFIT, 3)
    q = p.quote_arbitrage(rb, ro, hub_off, hubs, legs=True)
    c = certify(allset, p, q, rb, ro, hub_off, hubs)
    assert sum(x["gap"] is not None for x in c) >= 4
    out = p.execute_arbitrage(rb, ro, hub_off, hubs, q[0] * 0.5, legs=True)
    filled = np.flatnonzero(out[3] == ao.FILLED)
    assert len(filled) >= 4
    # re-quote: a row whose pairs no later filled row touched is closed, to within its allowance
    again = p.quote_arbitrage(rb, ro, hub_off, hubs, legs=True)
    c = certify(allset, p, again, rb, ro, hub_off, hubs)
    pairs_of = lambda r: {frozenset(x) for x in [(int(rb[r]), int(ro[r]))] +
                          [(int(ro[r]), int(h)) for h in hubs[hub_off[r]:hub_off[r + 1]]] +
                          [(int(h), int(rb[r])) for h in hubs[hub_off[r]:hub_off[r + 1]]]}
    closed = 0
    for r in filled:
        if any(pairs_of(r) & pairs_of(s) for s in filled if s > r):
            continue
        assert c[r]["gap"] is not None and abs(again[0][r]) <= c[r]["allowance"], (r, again[0][r], c[r])
        closed += 1
    assert closed >= 1
    p.close()


def test_routed_amount_zero_still_fills_with_zeros(allset):
    out = allset.p.quote_routed_orders([4, 5], [1, 2], [0, 1], [0.0, 0.0], [0, 0, 0], [], legs=True)
    assert out[3].tolist() == [0, 0] and not out[0].any() and not out[1].any() and not out[2].any()
    assert not out[6][1].any() and not out[6][2].any()


def test_rejections_change_nothing(cr, allset):
    p = allset.fresh()
    before = allset.state(p)
    n = allset.n
    for kw in [dict(base=[0]), dict(base=[n + 1]), dict(base=[1, 1], min_profit=[1.0, 1.0]),
               dict(min_profit=[0.0]), dict(min_profit=[-1.0]), dict(min_profit=[np.nan]),
               dict(min_profit=[np.inf]), dict(max_hubs=-1), dict(max_hubs=8)]:
        a = {**dict(base=[1], min_profit=[1.0], max_hubs=3), **kw}
        with pytest.raises(cr.CFMMError) as e:
            p.scan_arbitrage(a["base"], a["min_profit"], a["max_hubs"], 4)
        assert e.value.code == -1, kw
    lib, ctx = p._lib, p._ctx
    b, m, found = np.array([1], np.int64), np.array([1.0]), np.zeros(1, np.int64)
    ip, dp = C.POINTER(C.c_int64), C.POINTER(C.c_double)
    assert lib.cfmm_scan_arbitrage(ctx, 1, b.ctypes.data_as(ip), m.ctypes.data_as(dp), 3, 2,
                                   found.ctypes.data_as(ip), None, None, None, None, None, None) == -1
    ok = dict(base=[1], other=[4], hub_off=[0, 1], hubs=[2])
    for kw in [dict(other=[1]), dict(other=[0]), dict(hubs=[1]), dict(hubs=[4]), dict(hubs=[n + 1]),
               dict(hub_off=[0, 2], hubs=[2, 2]), dict(hub_off=[0, 8], hubs=[2] * 8), dict(hub_off=[1, 1])]:
        a = {**ok, **kw}
        with pytest.raises((cr.CFMMError, ValueError)):
            p.execute_arbitrage(a["base"], a["other"], a["hub_off"], a["hubs"])
    for mp in ([np.nan], [-1.0], [np.inf]):
        with pytest.raises(cr.CFMMError) as e:
            p.execute_arbitrage([1], [4], [0, 1], [2], mp)
        assert e.value.code == -1
    assert same_state(before, allset.state(p))
    p.close()


def test_router_on_device(cr):
    n = 6
    rng = np.random.default_rng(3)
    cs = []
    for a in range(1, n + 1):
        for b in range(a + 1, n + 1):
            for _ in range(2 if a == 1 else 1):
                cs.append(cr.ProductTwoCoin(rng.uniform(500, 5000) * np.exp(rng.uniform(-0.05, 0.05, size=2)),
                                            0.997, [a, b]))
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), cs, n)
    rb, ro, hubs, profit, price = r.scan_arbitrage([1, 2], 1e-6, max_hubs=2)
    assert len(rb) >= 2 and np.all(profit >= 1e-6)
    assert np.array_equal(r.quote_arbitrage(rb, ro, hubs)[0], profit)
    out = r.execute_arbitrage(rb, ro, hubs, profit * 0.0)
    assert ao.FILLED in set(out[3].tolist())
    st = r._pools.pool_state(P)[0]
    for k, c in enumerate(cs):
        assert np.array_equal(c.R, st[r._type_lists[P].index(k)])
    r._pools.close()
