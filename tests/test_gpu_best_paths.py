"""cfmm_find_order_paths (include/cfmm_b200.h) on the device.

The paths are checked bit for bit against a reference composed from other entry points: best_path_oracle's
DP driven by cfmm_pair_pools and cfmm_quote_swaps / cfmm_quote_swaps_exact_out, which holds for all
three pool types, GeometricMeanTwoCoin included; for ProductTwoCoin and UniV3 also against the host
mirror on pool objects.  The sets are test_gpu_routed_orders' hub sets (appended and retired pools,
pools stored with their tokens exchanged), also after cfmm_compact, a UniV3 liquidity change and a
retire that follows the adjacency build.  cfmm_quote_paths on the returned CSR gives the same amounts;
one hop is the best direct pool; two hops are the better of that and cfmm_choose_order_hubs' best hub;
on ProductTwoCoin more hops or a larger mask never lower a row's value; the execute is the find
followed by cfmm_execute_paths; a find changes no state; and the call's launches are pinned."""
import numpy as np
import pytest

import best_path_oracle as bo
from test_gpu_call_accounting import PROF, Pools
from test_gpu_order_hubs import mirror_market, order_rows, router_market
from test_gpu_paths import same_state
from test_gpu_routed_orders import HubSet

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
INF = float("inf")


def same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y)), (x, y)


# ---- the composed reference ----------------------------------------------------------------------
def device_lists(p, Ai, n):
    """best_path_oracle.dp's lists from cfmm_pair_pools: handle (type, index), ingest token 1, active."""
    a = [x for x in range(1, n + 1) for y in range(x + 1, n + 1)]
    b = [y for x in range(1, n + 1) for y in range(x + 1, n + 1)]
    off, typ, idx, act = p.pair_pools(a, b)
    return {(a[c], b[c]): [((int(typ[e]), int(idx[e])), int(Ai[int(typ[e])][int(idx[e])][0]), bool(act[e]))
                           for e in range(off[c], off[c + 1])] for c in range(len(a)) if off[c + 1] > off[c]}


def device_quote(p):
    """dp's quote through cfmm_quote_swaps / cfmm_quote_swaps_exact_out, one call per type and kind."""
    def quote(reqs):
        vals = [0.0] * len(reqs)
        for t in (P, G, U):
            for out in (False, True):
                sel = [n for n, r in enumerate(reqs) if r[0][0] == t and r[3] == out]
                if not sel:
                    continue
                ids = np.array([reqs[n][0][1] for n in sel], dtype=np.int64)
                tok1 = np.array([reqs[n][1] for n in sel])
                arg = np.zeros((len(sel), 2))
                x = np.array([reqs[n][2] for n in sel])
                if out:  # want the other side
                    arg[tok1, 1], arg[~tok1, 0] = x[tok1], x[~tok1]
                    res = p.quote_swaps_exact_out(t, ids, arg)
                    got = np.where(tok1, res[:, 0], res[:, 1])
                else:
                    arg[tok1, 0], arg[~tok1, 1] = x[tok1], x[~tok1]
                    res = p.quote_swaps(t, ids, arg)
                    got = np.where(tok1, res[:, 1], res[:, 0])
                for n, v in zip(sel, got):
                    vals[n] = float(v)
        return vals
    return quote


def composed(p, Ai, n, tin, tout, kind, amount, H, allowed):
    """(hop_off, hop_type, hop_pool, hop_token, value, status) from the composed DP; value is the DP's
    amount on filled rows, 0 elsewhere."""
    res = bo.dp(list(zip(tin, tout, kind, amount)), device_lists(p, Ai, n), n, allowed, H, device_quote(p))
    paths = [path if st == bo.FILLED else [] for path, st, _ in res]
    off = np.concatenate([[0], np.cumsum([len(x) for x in paths])]).astype(np.int64)
    return (off, np.array([h[2][0] for x in paths for h in x], np.int32),
            np.array([h[2][1] for x in paths for h in x], np.int64), np.array([h[1] for x in paths for h in x], np.int64),
            np.array([amt if st == bo.FILLED else 0.0 for _, st, amt in res]),
            np.array([st for _, st, _ in res], np.uint8))


def mirror(hs, p, tin, tout, kind, amount, H, allowed):
    """The host mirror on hs's ProductTwoCoin / UniV3 pools at p's state, the pair lists in
    cfmm_pair_pools order; hops as (type, index)."""
    pools = mirror_market(hs, p)
    key = [(P, i) for i in range(hs.m[P])] + [(U, i) for i in range(hs.m[U])]
    at = {k: n for n, k in enumerate(key)}
    pairs = {ab: [at[h] for h, _, _ in lst] for ab, lst in device_lists(p, hs.Ai, hs.n).items()}
    off, hp, ht, x, lam, value, status, _ = bo.find(pools, hs.n, tin, tout, kind, amount, H, allowed, pairs)
    return (off, np.array([key[k][0] for k in hp], np.int32), np.array([key[k][1] for k in hp], np.int64), ht, x, lam,
            value, status)


def check_paths(hs, p, rng, q=16, mirror_too=True, hops=(1, 2, 3, 4)):
    tin, tout, kind, amount = order_rows(rng, hs.n, q)
    for allowed in (np.ones(hs.n, bool), rng.random(hs.n) < 0.6):
        for H in hops:
            got = p.find_order_paths(tin, tout, kind, amount, H, allowed)
            off, ht, hp, htok, x, lam, value, status = got
            ref = composed(p, hs.Ai, hs.n, tin, tout, kind, amount, H, allowed)
            same((off, ht, hp, htok, value, status), ref)
            if mirror_too:
                same(got, mirror(hs, p, tin, tout, kind, amount, H, allowed))
            # cfmm_quote_paths on the returned CSR: the same amounts
            rows = np.flatnonzero(np.diff(off) > 0)
            if len(rows):
                sub = np.concatenate([[0], np.cumsum(np.diff(off)[rows])]).astype(np.int64)
                keep = np.concatenate([np.arange(off[r], off[r + 1]) for r in rows])
                qx, ql, qs = p.quote_paths(sub, ht[keep], hp[keep], tin[rows], kind[rows], amount[rows])
                assert np.array_equal(qx, x[keep]) and np.array_equal(ql, lam[keep]) and np.all(qs == 0)
                last = np.where(kind[rows] == 0, ql[sub[1:] - 1], qx[sub[:-1]])
                assert np.array_equal(last, value[rows])
            assert np.all(htok[off[1:][np.diff(off) > 0] - 1] == tout[np.diff(off) > 0])
    return got


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U), (P, G, U)], ids=["product", "univ3", "mixed", "all"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=150 + len(request.param) + request.param[0])
    yield hs
    hs.p.close()


# ---- 1. bit-exact ----------------------------------------------------------------------------------
def test_bit_exact_paths(hset):
    got = check_paths(hset, hset.p, np.random.default_rng(1), mirror_too=not hset.m[G])
    assert np.sum(np.diff(got[0]) > 1) > 0  # some multi-hop paths


def test_after_compact_liquidity_and_retire(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=95)
    p = hs.p
    rng = np.random.default_rng(2)
    check_paths(hs, p, rng, hops=(2, 4))  # builds the adjacency
    t_hub = [(t, i) for t in (P, U) for i in range(hs.m[t]) if 1 in hs.Ai[t][i] and (t, i) not in hs.retired][:6]
    for t, i in t_hub:
        p.set_active(t, i, [False])
    hs.retired |= set(t_hub)
    check_paths(hs, p, rng, hops=(2, 4))
    p.compact()
    check_paths(hs, p, rng, hops=(2, 4))
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:4]
    st = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, st[ui] * 0.8, st[ui] * 1.25, np.full(len(ui), 2000.0))
    check_paths(hs, p, rng, hops=(2, 4))
    p.close()


# ---- 2. against the direct pools and the hub choice ---------------------------------------------------
def test_one_and_two_hops_against_direct_and_hubs(hset):
    p, n = hset.p, hset.n
    rng = np.random.default_rng(3)
    tin, tout, kind, amount = order_rows(rng, n, 24)
    allowed = rng.random(n) < 0.7
    lists = device_lists(p, hset.Ai, n)
    quote = device_quote(p)
    direct = []
    for j, i, k, a in zip(tin, tout, kind, amount):
        # the direct hop tenders j, for both kinds
        lst = [(h, t1 == j, a, bool(k)) for h, t1, act in lists.get((min(j, i), max(j, i)), []) if act]
        v = quote(lst) if lst and a > 0 else []
        v = [x for x in v if (x < INF if k else x > 0.0)]
        direct.append((min(v) if k else max(v)) if v else None)
    one = p.find_order_paths(tin, tout, kind, amount, 1, allowed)
    two = p.find_order_paths(tin, tout, kind, amount, 2, allowed)
    h_off, hubs, score, _ = p.choose_order_hubs(tin, tout, kind, amount, 1, allowed)
    for r in range(len(tin)):
        if amount[r] == 0.0:
            continue
        d = direct[r]
        assert (one[7][r] == 0 and one[6][r] == d) if d is not None else one[7][r] == 2, r
        hub = score[h_off[r]] if h_off[r + 1] > h_off[r] else None
        cands = [x for x in (d, hub) if x is not None]
        if not cands:
            assert two[7][r] == 2
            continue
        want = min(cands) if kind[r] else max(cands)
        assert two[7][r] == 0 and two[6][r] == want, (r, two[6][r], d, hub)
        n_hops = two[0][r + 1] - two[0][r]
        assert n_hops == (1 if d is not None and d == want else 2)  # a tie goes to the direct pool
        if n_hops == 2 and hub is not None and (d is None or d != want):
            assert two[3][two[0][r]] == hubs[h_off[r]]


def test_more_hops_and_tokens_never_lower_product_values(cr, synth):
    hs = HubSet(cr, synth, (P,), seed=99)
    p = hs.p
    rng = np.random.default_rng(4)
    tin, tout, kind, amount = order_rows(rng, hs.n, 40)
    small = rng.random(hs.n) < 0.5
    masks = [small, small | (rng.random(hs.n) < 0.5), np.ones(hs.n, bool)]
    prev_m = None
    for allowed in masks:
        prev = None
        for H in range(1, 9):
            got = p.find_order_paths(tin, tout, kind, amount, H, allowed)
            for old in [x for x in (prev, prev_m if H == 8 else None) if x is not None]:
                both = (old[7] == 0) & (got[7] == 0) & (amount > 0)
                better = np.where(kind == 0, got[6] >= old[6], got[6] <= old[6])
                assert np.all(better[both])
            prev = got
        prev_m = prev
    p.close()


# ---- 3. execute -----------------------------------------------------------------------------------------
def test_execute_is_find_then_execute_paths(cr):
    r1, r2 = router_market(cr, 12), router_market(cr, 12)
    rng = np.random.default_rng(6)
    tin, tout, kind, amount = order_rows(rng, 12, 24, lo=5)
    tin[:8], tout[:8] = 5, 6  # rows sharing pools: later rows run on the state earlier rows left
    allowed = np.ones(12, bool)
    allowed[[0, 1]] = False
    q1 = r1.quote_best_paths(tin, tout, kind, amount, allowed, 3)
    lim = np.where(kind == 1, q1[0] * 1.01, q1[1] * 0.99)
    lim[::4] = np.where(kind[::4] == 1, 0.0, 1e300)  # some rows revert
    a = r1.execute_best_paths(tin, tout, kind, amount, allowed, 3, lim)
    paths, value, status = r2.find_paths(tin, tout, kind, amount, allowed, 3)
    assert a[3] == paths
    rows = [r for r in range(len(tin)) if paths[r]]
    b = r2.execute_paths([paths[r] for r in rows], tin[rows], kind[rows], amount[rows], lim[rows])
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(np.asarray(x)[rows], y)
    assert len(set(a[2].tolist())) > 1
    assert np.array_equal(r1._pools.pool_state(P)[0], r2._pools.pool_state(P)[0])
    assert all(np.array_equal(c1.R, c2.R) for c1, c2 in zip(r1.cfmms, r2.cfmms))
    # the quote is the find's amounts, and those are quote_paths' on the found paths
    paths, value, status = r1.find_paths(tin, tout, kind, amount, allowed, 3)
    qp = r1.quote_best_paths(tin, tout, kind, amount, allowed, 3)
    rows = [r for r in range(len(tin)) if paths[r]]
    qq = r1.quote_paths([paths[r] for r in rows], tin[rows], kind[rows], amount[rows])
    for x, y in zip(qp[:3], qq[:3]):
        assert np.array_equal(np.asarray(x)[rows], y)
    r1._pools.close()
    r2._pools.close()


# ---- 4. read-only and rejections --------------------------------------------------------------------------
def test_find_changes_nothing_and_rejects(cr, hset):
    p = hset.p
    before = hset.state(p)
    rng = np.random.default_rng(7)
    tin, tout, kind, amount = order_rows(rng, hset.n, 32)
    p.find_order_paths(tin, tout, kind, amount, 8, np.ones(hset.n, bool))
    assert same_state(before, hset.state(p))
    ok = np.ones(hset.n, bool)
    bad = [dict(tin=[5]), dict(tin=[0]), dict(kind=[2]), dict(amount=[np.nan]), dict(amount=[-1.0]),
           dict(amount=[np.inf]), dict(max_hops=0), dict(max_hops=9)]
    for b in bad:
        a = {**dict(tin=[4], tout=[5], kind=[0], amount=[1.0], max_hops=4), **b}
        with pytest.raises(cr.CFMMError) as e:
            p.find_order_paths(a["tin"], a["tout"], a["kind"], a["amount"], a["max_hops"], ok)
        assert e.value.code == -1 and "find_order_paths" in e.value.message
    assert same_state(before, hset.state(p))


def test_more_intermediate_tokens_than_the_cap(cr, synth):
    from test_gpu_parity import make_pools
    n = 1030
    R, g, A = synth.product_pools(2000, n, seed=21)
    p = make_pools(cr, n, product=(R, g, A))
    allowed = np.ones(n, bool)
    allowed[:4] = False  # 1026 allowed tokens: B = 1024 when both of a row's tokens are allowed
    tin, tout = np.array([10, 1]), np.array([11, 12])
    got = p.find_order_paths(tin[:1], tout[:1], [0], [1.0], 3, allowed)
    assert got[7][0] in (0, 2)
    with pytest.raises(cr.CFMMError) as e:  # row 1: token 1 is not allowed, so B = 1025
        p.find_order_paths(tin, tout, [0, 0], [1.0, 1.0], 3, allowed)
    assert e.value.code == -1 and "more than 1024" in e.value.message
    with pytest.raises(cr.CFMMError) as e:
        p._chk(p._lib.cfmm_find_order_paths(p._ctx, 0, None, None, None, None, 3, None, None, None, None, None, None,
                                            None, None, None))
    assert "null allowed" in e.value.message
    p.close()


# ---- 5. launches ---------------------------------------------------------------------------------------
def test_launches_and_profile_entries(cr, synth):
    """One call on test_gpu_call_accounting's seeded set: with nothing built, the pair index (9
    launches, one entry), the adjacency (3, one entry) and the graph and path kernels (2, one entry);
    with the pair index but no adjacency, 3 + 2; warm, 2; with no allowed token, the path kernel
    alone."""
    ps = Pools(cr, synth)
    p = ps.p
    p.set_option("profile", 256)
    ok = np.ones(p.n_tokens, bool)
    args = ([1, 2, 3], [4, 5, 6], [0, 1, 0], [1.0, 1e-3, 0.0], 4)

    def delta(fn):
        l0, c0 = p.launch_count, p.profile_read(PROF)[1]
        fn()
        return p.launch_count - l0, p.profile_read(PROF)[1] - c0

    assert delta(lambda: p.find_order_paths(*args, ok)) == (14, 3)
    assert delta(lambda: p.find_order_paths(*args, ok)) == (2, 1)
    p.append_product(*synth.product_pools(3, 16, seed=31))  # drops the pair index and the adjacency
    p.pair_pools([1], [2])  # rebuilds the pair index only
    assert delta(lambda: p.find_order_paths(*args, ok)) == (5, 2)
    assert delta(lambda: p.find_order_paths(*args, np.zeros(p.n_tokens, bool))) == (1, 1)
    assert delta(lambda: p.find_order_paths([], [], [], [], 4, ok)) == (0, 0)
    p.close()
