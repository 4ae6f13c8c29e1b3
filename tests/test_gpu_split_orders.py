"""cfmm_pair_pools / cfmm_quote_split_orders / cfmm_execute_split_orders (include/cfmm_b200.h) on the
device.

One context holds all three pool types, each with a main set and appended pools, some retired; the
ProductTwoCoin main set is laid out with orient_by_degree = 1, so some of its pools are stored with
their tokens exchanged (test_gpu_paths.Mixed).  The pair index is checked against a numpy grouping
of the ingest token pairs before and after appends and a compact.  Quotes and executes are checked
bit for bit against the host mirror (split_oracle.py) on ProductTwoCoin and UniV3 pairs, and, for
all three types, against the existing entry points: a fresh 2-token context holding the pair's pools
in their state before a row, a materialising cfmm_sweep at ν = (1, s*), cfmm_get_trades and
cfmm_apply_trades."""
import numpy as np
import pytest

import split_oracle as so
from test_gpu_parity import make_pools
from test_gpu_paths import APPEND, Mixed, same_state
from test_gpu_swap_orders import univ3_host_pools

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2


@pytest.fixture(scope="module")
def mx(cr, synth):
    return Mixed(cr, synth, seed=31)


def global_keys(mx, with_tail=True):
    """(type, index) of every pool in global insertion order."""
    keys = [(t, i) for t in (P, G, U) for i in range(mx.mm[t])]
    if with_tail:
        keys += [(t, mx.mm[t] + i) for t in (P, G, U) for i in range(mx.mt[t])]
    return keys


def expected_pairs(mx, keys, a, b):
    return [k for k in keys if set(int(x) for x in mx.Ai[k[0]][k[1]]) == {a, b}]


def all_pairs(n):
    return [(a, b) for a in range(1, n + 1) for b in range(1, n + 1) if a != b]


def check_index(mx, p, keys, retired):
    pairs = all_pairs(mx.n)
    off, typ, idx, act = p.pair_pools([a for a, _ in pairs], [b for _, b in pairs])
    for r, (a, b) in enumerate(pairs):
        got = list(zip(typ[off[r]:off[r + 1]].tolist(), idx[off[r]:off[r + 1]].tolist()))
        assert got == expected_pairs(mx, keys, a, b), (a, b)
        assert act[off[r]:off[r + 1]].tolist() == [k not in retired for k in got]


def test_pair_index_append_compact(cr, mx):
    p = make_pools(cr, mx.n, product=mx.main[P], geomean=mx.main[G], univ3=mx.main[U], pre={"orient_by_degree": 1})
    check_index(mx, p, global_keys(mx, False), set())
    for t in (P, G, U):
        getattr(p, APPEND[t])(*mx.tail[t])
    check_index(mx, p, global_keys(mx), set())
    act = np.ones(mx.m[P], bool)
    act[3] = False
    p.set_active(P, 0, act)  # retiring does not rebuild: activity is read per call
    check_index(mx, p, global_keys(mx), {(P, 3)})
    p.compact()
    check_index(mx, p, global_keys(mx), {(P, 3)})
    with pytest.raises(cr.CFMMError):
        p.pair_pools([1], [1])
    with pytest.raises(cr.CFMMError):
        p.pair_pools([0], [2])
    p.close()


def mirror_pools(mx, p):
    """split_oracle pools at the device's state, keyed (type, index), retired ones inactive."""
    out = {}
    st, _ = p.pool_state(P)
    for i in range(mx.m[P]):
        out[(P, i)] = so.Product(st[i], mx.g[P][i], mx.Ai[P][i])
    st, _ = p.pool_state(G)
    for i in range(mx.m[G]):
        out[(G, i)] = so.GeoMean(st[i], mx.g[G][i], mx.w[i], mx.Ai[G][i])
    for i, h in enumerate(univ3_host_pools(p, mx.g[U])):
        out[(U, i)] = so.Univ3(h.price, h.lt, h.lq, h.g, mx.Ai[U][i])
    for k in mx.retired:
        out[k].active = False
    return out


def rows_on(mx, rng, q, types):
    """q rows on pairs whose pools are all of `types`, both orientations, both kinds."""
    keys = global_keys(mx)
    ok = [(a, b) for a, b in all_pairs(mx.n)
          if expected_pairs(mx, keys, a, b) and all(k[0] in types for k in expected_pairs(mx, keys, a, b))]
    pick = [ok[int(j)] for j in rng.integers(0, len(ok), size=q)]
    tin = np.array([a for a, _ in pick], np.int64)
    tout = np.array([b for _, b in pick], np.int64)
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    amount = 10.0 ** rng.uniform(-3, 1.5, size=q)
    amount[::17] = 0.0
    return tin, tout, kind, amount


def compare(dev, rows, off):
    paid, got, price, st, (o, D, L) = dev
    assert np.array_equal(o, off)
    for r, row in enumerate(rows):
        assert st[r] == row["status"], r
        assert paid[r] == row["paid"] and got[r] == row["received"] and price[r] == row["price"], r
        assert np.array_equal(D[o[r]:o[r + 1]], row["D"]) and np.array_equal(L[o[r]:o[r + 1]], row["L"]), r


@pytest.mark.parametrize("types", [(P,), (U,), (P, U)], ids=["product", "univ3", "mixed"])
def test_bit_exact_against_mirror(mx, types):
    rng = np.random.default_rng(5 + len(types) + types[0])
    tin, tout, kind, amount = rows_on(mx, rng, 60, types)
    keys = global_keys(mx)
    objs = mirror_pools(mx, mx.p)
    pairs = lambda a, b: [objs[k] for k in expected_pairs(mx, keys, a, b)]
    dev = mx.p.quote_split_orders(tin, tout, kind, amount, legs=True)
    rows = so.quote_split(pairs, tin, tout, kind, amount)
    assert {r["status"] for r in rows} >= {so.FILLED}
    assert max(r["evals"] for r in rows) <= so.MAX_EVALS
    compare(dev, rows, dev[4][0])
    # execute on a fresh copy: in batch order, with limits around the quotes
    p = mx.fresh()
    lim = np.where(kind == 1, dev[0] * 1.0000001 + 1e-9, dev[1] * 0.9999999)
    lim[::5] = np.where(kind[::5] == 1, 0.0, 1e300)  # some revert
    lim = np.maximum(lim, 0.0)
    out = p.execute_split_orders(tin, tout, kind, amount, lim, legs=True)
    objs = mirror_pools(mx, mx.p)
    rows = so.replay_split(pairs, tin, tout, kind, amount, lim)
    compare(out, rows, dev[4][0])
    after = mirror_pools(mx, p)
    for k, o in objs.items():
        if k[0] == U:
            assert after[k].price == o.price, k
        elif k[0] == P:
            assert np.array_equal(after[k].R, o.R), k
    p.close()


def two_token_context(cr, mx, p, keys, tin, tout):
    """A fresh context holding the active pools keys (state of p), token_out -> 1, token_in -> 2."""
    tmap = {int(tout): 1, int(tin): 2}
    q = cr.DevicePools(2)
    by = {t: [k for k in keys if k[0] == t] for t in (P, G, U)}
    if by[P]:
        st, _ = p.pool_state(P)
        q.add_product(st[[i for _, i in by[P]]], mx.g[P][[i for _, i in by[P]]],
                      np.array([[tmap[int(x)] for x in mx.Ai[P][i]] for _, i in by[P]]))
    if by[G]:
        st, _ = p.pool_state(G)
        ids = [i for _, i in by[G]]
        q.add_geomean(st[ids], mx.g[G][ids], np.array([[tmap[int(x)] for x in mx.Ai[G][i]] for i in ids]), mx.w[ids])
    if by[U]:
        st, _ = p.pool_state(U)
        off, lt, lq = p.univ3_ticks()
        ids = [i for _, i in by[U]]
        o = np.concatenate([[0], np.cumsum([off[i + 1] - off[i] for i in ids])]).astype(np.int64)
        q.add_univ3(st[ids], mx.g[U][ids], np.array([[tmap[int(x)] for x in mx.Ai[U][i]] for i in ids]), o,
                    np.concatenate([lt[off[i]:off[i + 1]] for i in ids]), np.concatenate([lq[off[i]:off[i + 1]] for i in ids]))
    q.finalize()
    return q, by[P] + by[G] + by[U]


def test_bit_exact_against_sweep_and_apply(cr, mx):
    """Each filled row = a materialising sweep at ν = (1, s*) on its pair's pools + cfmm_apply_trades;
    rows of one pair chain; the whole batch in one call equals the rows one call at a time."""
    rng = np.random.default_rng(9)
    tin, tout, kind, amount = rows_on(mx, rng, 24, (P, G, U))
    # concentrate on a few pairs so that rows chain
    tin[12:], tout[12:] = tin[:12], tout[:12]
    keys = global_keys(mx)
    batch = mx.fresh()
    out = batch.execute_split_orders(tin, tout, kind, amount, legs=True)
    p = mx.fresh()
    for r in range(len(tin)):
        pk = expected_pairs(mx, keys, int(tin[r]), int(tout[r]))
        live = [k for k in pk if k not in mx.retired]
        if live:
            ctx, order = two_token_context(cr, mx, p, live, tin[r], tout[r])  # (the state before the row)
        one = p.execute_split_orders(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], legs=True)
        assert [x[0] for x in one[:4]] == [out[0][r], out[1][r], out[2][r], out[3][r]]
        o = out[4][0]
        assert np.array_equal(one[4][1], out[4][1][o[r]:o[r + 1]]) and np.array_equal(one[4][2], out[4][2][o[r]:o[r + 1]])
        if one[3][0] != so.FILLED or amount[r] == 0.0:
            if live:
                ctx.close()
            continue
        ctx.sweep(np.array([1.0, one[2][0]]), materialize=True)
        D, L = ctx.trades()
        for k, key in enumerate(pk):
            if key in mx.retired:
                assert not one[4][1][k].any() and not one[4][2][k].any()
                continue
            g = order.index(key)
            assert np.array_equal(one[4][1][k], D[g]) and np.array_equal(one[4][2][k], L[g]), (r, key)
        ctx.apply_trades()
        for t in (P, G, U):
            ids = [i for (s, i) in order if s == t]
            if not ids:
                continue
            got = p.pool_state(t)[0][ids]
            assert np.array_equal(ctx.pool_state(t)[0], got), (r, t)
        ctx.close()
    assert same_state(mx.state(batch), mx.state(p))
    batch.close()
    p.close()


def test_optimal_against_single_pools(mx):
    rng = np.random.default_rng(13)
    tin, tout, kind, amount = rows_on(mx, rng, 80, (P, G, U))
    amount[amount == 0.0] = 1.0
    paid, got, price, st = mx.p.quote_split_orders(tin, tout, kind, amount)
    keys = global_keys(mx)
    for r in np.flatnonzero(st == so.FILLED):
        best = 0.0 if kind[r] == 0 else np.inf
        for t, i in expected_pairs(mx, keys, int(tin[r]), int(tout[r])):
            if (t, i) in mx.retired:
                continue
            tok1 = int(mx.Ai[t][i][0]) == int(tin[r])
            row = np.array([[amount[r], 0.0] if tok1 else [0.0, amount[r]]])
            if kind[r] == 0:
                best = max(best, float(mx.p.quote_swaps(t, [i], row).max()))
            else:
                want = np.array([[0.0, amount[r]] if tok1 else [amount[r], 0.0]])
                best = min(best, float(mx.p.quote_swaps_exact_out(t, [i], want).max()))
        if kind[r] == 0:
            assert got[r] >= best * (1 - 1e-11), r
        else:
            assert paid[r] <= best * (1 + 1e-11), r


def test_statuses_and_validation(cr, mx):
    p = mx.fresh()
    keys = global_keys(mx)
    pairs = all_pairs(mx.n)
    a, b = next((a, b) for a, b in pairs if len(expected_pairs(mx, keys, a, b)) >= 2)
    paid, got, price, st = p.quote_split_orders([a, a], [b, b], [0, 1], [0.0, 0.0])
    assert st.tolist() == [so.FILLED, so.FILLED] and not paid.any() and not got.any() and not price.any()
    # limits: an equal limit fills, one ulp tighter reverts, and the next row sees the state without it
    q = p.quote_split_orders([a], [b], [0], [2.0])
    before = mx.state(p)
    r = p.execute_split_orders([a, a], [b, b], [0, 0], [2.0, 2.0], [np.nextafter(q[1][0], np.inf), 0.0])
    assert r[3].tolist() == [so.LIMIT, so.FILLED] and r[1][1] == q[1][0] and r[0][0] == 0.0
    p.close()
    p = mx.fresh()
    r = p.execute_split_orders([a], [b], [0], [2.0], [q[1][0]])
    assert r[3][0] == so.FILLED and r[1][0] == q[1][0]
    # only retired pools
    gone = set(mx.retired) | set(expected_pairs(mx, keys, a, b))
    for t in (P, G, U):
        act = np.ones(mx.m[t], bool)
        act[[j for (s, j) in gone if s == t]] = False
        p.set_active(t, 0, act)
    assert p.quote_split_orders([a], [b], [1], [1.0])[3][0] == so.UNREACHABLE
    # every rejection changes nothing
    before = mx.state(p)
    for args in ([0], [b], [0], [1.0], None), ([a], [a], [0], [1.0], None), ([a], [b], [2], [1.0], None), \
                ([a], [b], [0], [np.nan], None), ([a], [b], [0], [-1.0], None), ([a], [b], [0], [np.inf], None), \
                ([a], [b], [0], [1.0], [np.nan]), ([a], [b], [0], [1.0], [-1.0]), ([a], [b], [0], [1.0], [np.inf]), \
                ([a, a], [b, mx.n + 1], [0, 0], [1.0, 1.0], None):
        with pytest.raises(cr.CFMMError) as e:
            p.execute_split_orders(*args)
        assert e.value.code == -1
    assert same_state(before, mx.state(p))
    p.close()


def test_univ3_empty_last_tick_unreachable(cr):
    # one UniV3 pool on {1, 2} whose last tick is empty, a ProductTwoCoin pool elsewhere
    p = make_pools(cr, 4, product=(np.array([[100.0, 100.0]]), np.array([0.997]), np.array([[3, 4]])),
                   univ3=(np.array([1.0]), np.array([0.997]), np.array([[1, 2]]), np.array([0, 3]),
                          np.array([1.2, 1.0, 0.8]), np.array([10.0, 20.0, 0.0])))
    u = so.Univ3(1.0, [1.2, 1.0, 0.8], [10.0, 20.0, 0.0], 0.997, [1, 2])
    for tin, tout, kind, amt in [(1, 2, 0, 0.3), (1, 2, 0, 1e6), (1, 2, 1, 1e6), (2, 1, 0, 0.1), (2, 1, 1, 1e3)]:
        dev = p.quote_split_orders([tin], [tout], [kind], [amt], legs=True)
        row = so.split_row([u], tin, tout, kind, amt)
        compare(dev, [row], np.array([0, 1]))
    assert p.quote_split_orders([1], [2], [0], [1e6])[3][0] == so.UNREACHABLE
    assert p.quote_split_orders([1, 3], [3, 1], [0, 1], [1.0, 1.0])[3].tolist() == [so.UNREACHABLE] * 2  # no pool
    assert p.pair_pools([1, 4, 1], [2, 3, 4])[0].tolist() == [0, 1, 2, 2]
    p.close()
