"""cfmm_find_order_paths_net / cfmm_quote_token_values_net (include/cfmm_b200.h) on the device.

Both calls are checked bit for bit against their definition composed from the existing device calls:
cfmm_find_order_paths / cfmm_quote_token_values at every max_hops L = 1 … H, selected per row or per
(row, token) by path_cost_oracle.select, in every output including the requested walks.  The hop
costs are 0, about 1e-6 of the amount, large enough that one hop or nothing wins, +inf on some rows or
tokens, and mixed.  At κ = 0 every output equals the existing call's except where the selection picks
a shorter L, and each such case is one the header names.  The walks price through cfmm_quote_paths;
Router.execute_best_paths with hop_cost is the find followed by cfmm_execute_paths; the results hold
after a retire, cfmm_compact, a UniV3 liquidity change and an execute; a million Zipf-skewed pools
match the numpy form; rows do not depend on their batch; the calls change no state, reject bad costs
before anything runs, and their launches are pinned."""
import numpy as np
import pytest

import path_cost_oracle as pc
import token_value_oracle as tv
from test_gpu_best_paths import same
from test_gpu_call_accounting import PROF, Pools
from test_gpu_order_hubs import order_rows, router_market
from test_gpu_paths import same_state
from test_gpu_routed_orders import HubSet
from test_gpu_token_values import consistent_market

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
INF = float("inf")


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U), (P, G, U)], ids=["product", "univ3", "mixed", "all"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=190 + len(request.param) + request.param[0])
    yield hs
    hs.p.close()


def row_costs(rng, amount, which):
    q = len(amount)
    if which == "zero":
        return np.zeros(q)
    if which == "small":
        return amount * 1e-6
    if which == "large":
        return amount * 0.5
    if which == "inf":
        return np.where(np.arange(q) % 3 == 0, INF, amount * 1e-4)
    return amount * np.choose(np.arange(q) % 4, [0.0, 1e-6, 1e-2, 0.5])  # mixed per row


COSTS = ("zero", "small", "large", "inf", "mixed")


# ---- the composed reference -------------------------------------------------------------------------
def composed_paths(p, tin, tout, kind, amount, H, allowed, kappa):
    """find_order_paths at every L, selected per row: find_order_paths_net's tuple, and L per row."""
    per = [p.find_order_paths(tin, tout, kind, amount, L, allowed) for L in range(1, H + 1)]
    parts, value, status, net, sel = [[] for _ in range(6)], [], [], [], []
    for r in range(len(tin)):
        if not amount[r] > 0.0:
            L, x = H, per[-1][6][r]
        else:
            L, x = pc.select([(f[7][r], f[6][r], f[0][r + 1] - f[0][r]) for f in per], kappa[r], kind[r] == 1)
        f = per[L - 1]
        seg = slice(f[0][r], f[0][r + 1])
        parts[0].append(f[0][r + 1] - f[0][r])
        for c in range(1, 6):
            parts[c].append(f[c][seg])
        value.append(f[6][r])
        status.append(f[7][r])
        net.append(x)
        sel.append(L)
    off = np.concatenate([[0], np.cumsum(parts[0])]).astype(np.int64)
    return (off, *(np.concatenate(parts[c]) for c in range(1, 6)), np.array(value), np.array(status, np.uint8),
            np.array(net)), np.array(sel), per


def check_paths(hs, p, rng, hops=(1, 3, 5), costs=COSTS, q=16):
    tin, tout, kind, amount = order_rows(rng, hs.n, q)
    shorter = 0
    for allowed in (np.ones(hs.n, bool), rng.random(hs.n) < 0.6):
        for H in hops:
            for which in costs:
                kappa = row_costs(rng, amount, which)
                got = p.find_order_paths_net(tin, tout, kind, amount, H, allowed, kappa)
                ref, sel, per = composed_paths(p, tin, tout, kind, amount, H, allowed, kappa)
                same(got, ref)
                shorter += int(np.sum(sel < H))
                off, ht, hp, htok, x, lam, value = got[:7]
                rows = np.flatnonzero(np.diff(off) > 0)
                if len(rows):  # the walks price through cfmm_quote_paths to the reported value
                    sub = np.concatenate([[0], np.cumsum(np.diff(off)[rows])]).astype(np.int64)
                    qx, ql, qs = p.quote_paths(sub, ht, hp, tin[rows], kind[rows], amount[rows])
                    assert np.array_equal(qx, x) and np.array_equal(ql, lam) and np.all(qs == 0)
                    last = np.where(kind[rows] == 0, ql[sub[1:] - 1], qx[sub[:-1]])
                    assert np.array_equal(last, value[rows])
    return shorter


def composed_values(p, roots, kinds, amounts, H, allowed, kappa, req):
    """quote_token_values at every L, selected per (row, token): quote_token_values_net's tuple."""
    per = [p.quote_token_values(roots, kinds, amounts, L, allowed, req) for L in range(1, H + 1)]
    q, n = per[-1][0].shape
    value, hops, status = (per[-1][c].copy() for c in range(3))
    net, sel = per[-1][0].copy(), np.full((q, n), H)
    for r in range(q):
        for t in range(n):
            if t == roots[r] - 1:
                continue
            L, x = pc.select([(f[2][r, t], f[0][r, t], int(f[1][r, t])) for f in per], kappa[t], kinds[r] == 1)
            f = per[L - 1]
            value[r, t], hops[r, t], status[r, t], net[r, t], sel[r, t] = f[0][r, t], f[1][r, t], f[2][r, t], x, L
    parts, rst = [[] for _ in range(6)], []
    for j, (r, t) in enumerate(zip(*req)):
        f = per[sel[r, t - 1] - 1]
        seg = slice(f[4][j], f[4][j + 1])
        parts[0].append(f[4][j + 1] - f[4][j])
        for c in range(1, 6):
            parts[c].append(f[4 + c][seg])
        rst.append(f[10][j])
    off = np.concatenate([[0], np.cumsum(parts[0])]).astype(np.int64)
    cols = [np.concatenate(parts[c]) if parts[c] else per[-1][4 + c][:0] for c in range(1, 6)]
    return (value, hops, status, net, per[-1][3], off, *cols, np.array(rst, np.uint8)), sel, per


def token_costs(rng, n, amount, which):
    if which == "zero":
        return np.zeros(n)
    if which == "small":
        return np.full(n, amount * 1e-6)
    if which == "large":
        return np.full(n, amount * 0.5)
    if which == "inf":
        return np.where(np.arange(n) % 3 == 0, INF, amount * 1e-4)
    return amount * 10.0 ** rng.uniform(-7, 0, size=n)  # mixed per token


def check_values(hs, p, rng, hops=(1, 3, 6), costs=COSTS, roots=2):
    n = hs.n
    tokens = np.arange(1, n + 1, dtype=np.int64)
    shorter = 0
    for allowed in (None, rng.random(n) < 0.7):
        for kind in (0, 1):
            for root in rng.choice(tokens, size=roots, replace=False):
                amount = float(10.0 ** rng.uniform(-1, 2))
                req = (np.zeros(n, np.int64), tokens)
                for H in hops:
                    for which in costs:
                        kappa = token_costs(rng, n, amount, which)
                        got = p.quote_token_values_net([root], [kind], [amount], H, kappa, allowed, req)
                        ref, sel, _ = composed_values(p, [root], [kind], [amount], H, allowed, kappa, req)
                        same(got, ref)
                        shorter += int(np.sum(sel < H))
                        off, ht, hp, x, lam = got[5], got[6], got[7], got[9], got[10]
                        rows = np.flatnonzero(np.diff(off) > 0)
                        if len(rows):
                            sub = np.concatenate([[0], np.cumsum(np.diff(off)[rows])]).astype(np.int64)
                            tin = tokens[rows] if kind else np.full(len(rows), root, np.int64)
                            qx, ql, qs = p.quote_paths(sub, ht, hp, tin, np.full(len(rows), kind, np.uint8),
                                                       np.full(len(rows), amount))
                            assert np.array_equal(qx, x) and np.array_equal(ql, lam) and np.all(qs == 0)
                            last = qx[sub[:-1]] if kind else ql[sub[1:] - 1]
                            assert np.array_equal(last, got[0][0][rows])
    return shorter


# ---- 1. the composition, bit for bit ------------------------------------------------------------------
def test_best_paths_compose_the_existing_call(hset):
    assert check_paths(hset, hset.p, np.random.default_rng(1)) > 0  # some rows pick a shorter walk


def test_token_values_compose_the_existing_call(hset):
    assert check_values(hset, hset.p, np.random.default_rng(2)) > 0


# ---- 2. κ = 0 against the existing calls ----------------------------------------------------------------
def test_zero_cost_is_the_existing_call_or_a_named_improvement(hset):
    p, n = hset.p, hset.n
    rng = np.random.default_rng(3)
    tin, tout, kind, amount = order_rows(rng, n, 32)
    cases = {"repeats": 0, "rounding": 0}
    for H in (2, 4, 8):
        allowed = np.ones(n, bool)
        got = p.find_order_paths_net(tin, tout, kind, amount, H, allowed, np.zeros(len(tin)))
        _, sel, per = composed_paths(p, tin, tout, kind, amount, H, allowed, np.zeros(len(tin)))
        base = per[-1]
        for r in range(len(tin)):
            a, b = slice(got[0][r], got[0][r + 1]), slice(base[0][r], base[0][r + 1])
            if sel[r] == H:
                assert got[6][r] == base[6][r] and got[7][r] == base[7][r]
                assert all(np.array_equal(got[c][a], base[c][b]) for c in range(1, 6))
                continue
            if base[7][r] == 4:  # CFMM_PATH_REPEATS_POOL at H, a shorter L fills
                cases["repeats"] += 1
                assert got[7][r] == 0
            else:  # rounding: the shorter walk's quote is strictly better
                cases["rounding"] += 1
                assert base[7][r] == 0 and (got[6][r] < base[6][r] if kind[r] else got[6][r] > base[6][r])
        for root in (1, 4):
            for k in (0, 1):
                v = p.quote_token_values_net([root], [k], [3.0], H, np.zeros(n))
                ref, sel, per = composed_values(p, [root], [k], [3.0], H, None, np.zeros(n),
                                                (np.zeros(0, np.int64), np.zeros(0, np.int64)))
                base = per[-1]
                keep = sel[0] == H
                for c in range(3):
                    assert np.array_equal(v[c][0][keep], base[c][0][keep])
                for t in np.flatnonzero(~keep):
                    if base[2][0, t] == 4:
                        cases["repeats"] += 1
                        assert v[2][0, t] == 0
                    else:
                        cases["rounding"] += 1
                        assert base[2][0, t] == 0 and (v[0][0, t] < base[0][0, t] if k else v[0][0, t] > base[0][0, t])
    print("kappa = 0, shorter than H:", cases)


# ---- 3. execute ----------------------------------------------------------------------------------------
def test_execute_with_hop_cost_is_find_then_execute_paths(cr):
    r1, r2 = router_market(cr, 12), router_market(cr, 12)
    rng = np.random.default_rng(6)
    tin, tout, kind, amount = order_rows(rng, 12, 24, lo=5)
    tin[:8], tout[:8] = 5, 6
    allowed = np.ones(12, bool)
    allowed[[0, 1]] = False
    cost = r1.hop_costs(5, 0.05, 4)
    assert cost[4] == 0.05 and np.all(cost > 0)
    a = r1.execute_best_paths(tin, tout, kind, amount, allowed, 3, None, cost)
    paths, value, status, net = r2.find_paths(tin, tout, kind, amount, allowed, 3, cost)
    assert a[3] == paths and np.array_equal(a[4], net)
    rows = [r for r in range(len(tin)) if paths[r]]
    b = r2.execute_paths([paths[r] for r in rows], tin[rows], kind[rows], amount[rows])
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(np.asarray(x)[rows], y)
    assert np.array_equal(r1._pools.pool_state(P)[0], r2._pools.pool_state(P)[0])
    # the Router layers against DevicePools
    settle = np.where(kind == 1, tin, tout)
    found = r2._pools.find_order_paths_net(tin, tout, kind, amount, 3, allowed, cost[settle - 1])
    paths2, value2, status2, net2 = r2.find_paths(tin, tout, kind, amount, allowed, 3, cost)
    assert np.array_equal(found[6], value2) and np.array_equal(found[8], net2)
    qv = r2.quote_token_values([5, 6], [0, 1], [1.0, 2.0], 4, None, cost)
    dv = r2._pools.quote_token_values_net([5, 6], [0, 1], [1.0, 2.0], 4, cost)
    assert all(np.array_equal(x, y) for x, y in zip(qv, dv[:4]))
    tp = r2.token_paths(5, 0, 1.0, np.arange(1, 13), 4, None, cost)
    assert np.array_equal(tp[2], dv[0][0]) and np.array_equal(tp[4], dv[3][0])
    r1._pools.close()
    r2._pools.close()


# ---- 4. state changes ----------------------------------------------------------------------------------
def test_after_retire_compact_liquidity_and_execute(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=93)
    p = hs.p
    rng = np.random.default_rng(4)
    small = dict(hops=(3,), costs=("small", "mixed"))

    def both():
        check_paths(hs, p, rng, q=8, **small)
        check_values(hs, p, rng, roots=1, **small)
    both()
    t_hub = [(t, i) for t in (P, U) for i in range(hs.m[t]) if 1 in hs.Ai[t][i] and (t, i) not in hs.retired][:6]
    for t, i in t_hub:
        p.set_active(t, i, [False])
    hs.retired |= set(t_hub)
    both()
    p.compact()
    both()
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:4]
    s = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, s[ui] * 0.8, s[ui] * 1.25, np.full(len(ui), 2000.0))
    both()
    live = [i for i in range(hs.m[P]) if (P, i) not in hs.retired][:8]
    p.execute_swaps(P, live, np.column_stack([np.full(len(live), 30.0), np.zeros(len(live))]))
    both()
    p.close()


# ---- 5. scale ------------------------------------------------------------------------------------------
def test_million_skewed_pools_against_numpy(cr):
    n, m = 20_000, 1_000_000
    p, (R, g, A) = consistent_market(cr, n, m, seed=12)
    act = np.ones(m, bool)
    roots = np.array([1, 7], np.int64)
    amounts = np.array([10.0, 3.0])
    rng = np.random.default_rng(13)
    H = 4
    for kappa in (np.zeros(n), amounts[0] * 10.0 ** rng.uniform(-9, -3, size=n)):
        value, hops, st, net, _ = p.quote_token_values_net(roots, np.zeros(2, np.uint8), amounts, H, kappa)
        for r, root in enumerate(roots):
            v, h, x = pc.product(R, g, A, act, n, root, amounts[r], H, kappa)
            assert np.all(st[r][v > 0] == tv.FILLED)
            assert np.array_equal(value[r], v) and np.array_equal(hops[r], h) and np.array_equal(net[r], x)
        assert np.sum(value > 0) > n // 2
    p.close()


# ---- 6. call behaviour ---------------------------------------------------------------------------------
def test_rows_are_independent_of_their_batch(hset):
    p, n = hset.p, hset.n
    rng = np.random.default_rng(10)
    q = 70  # more than one token-value group of 64
    roots = rng.integers(1, n + 1, size=q)
    kinds = rng.integers(0, 2, size=q).astype(np.uint8)
    amounts = 10.0 ** rng.uniform(-1, 2, size=q)
    kappa = 10.0 ** rng.uniform(-6, -1, size=n)
    batch = p.quote_token_values_net(roots, kinds, amounts, 5, kappa)
    order = rng.permutation(q)
    perm = p.quote_token_values_net(roots[order], kinds[order], amounts[order], 5, kappa)
    assert all(np.array_equal(a[order], b) for a, b in zip(batch, perm))
    for r in range(0, q, 9):
        one = p.quote_token_values_net(roots[r:r + 1], kinds[r:r + 1], amounts[r:r + 1], 5, kappa)
        assert all(np.array_equal(a[r:r + 1], b) for a, b in zip(batch, one))
    tin, tout, kind, amount = order_rows(rng, n, 40)
    rk = amount * 10.0 ** rng.uniform(-6, -1, size=40)
    ok = np.ones(n, bool)
    full = p.find_order_paths_net(tin, tout, kind, amount, 5, ok, rk)
    for r in range(0, 40, 7):
        one = p.find_order_paths_net(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], 5, ok, rk[r:r + 1])
        seg = slice(full[0][r], full[0][r + 1])
        assert all(np.array_equal(full[c][seg], one[c]) for c in range(1, 6))
        assert all(full[c][r] == one[c][0] for c in (6, 7, 8))


def test_changes_nothing_and_rejects(cr, hset):
    p, n = hset.p, hset.n
    before = hset.state(p)
    rng = np.random.default_rng(11)
    tin, tout, kind, amount = order_rows(rng, n, 16)
    ok = np.ones(n, bool)
    p.find_order_paths_net(tin, tout, kind, amount, 8, ok, amount * 1e-3)
    p.quote_token_values_net(np.arange(1, n + 1), np.arange(n) % 2, np.full(n, 5.0), 8, np.full(n, 1e-3), None,
                             (np.arange(n), np.arange(n) + 1))
    assert same_state(before, hset.state(p))
    l0 = p.launch_count
    for bad in (np.nan, -1.0, -0.0 - 1e-300):
        with pytest.raises(cr.CFMMError) as e:
            p.find_order_paths_net([4], [5], [0], [1.0], 4, ok, [bad])
        assert e.value.code == -1 and "find_order_paths_net" in e.value.message and "hop_cost" in e.value.message
        kappa = np.zeros(n)
        kappa[n // 2] = bad
        with pytest.raises(cr.CFMMError) as e:
            p.quote_token_values_net([4], [0], [1.0], 4, kappa)
        assert e.value.code == -1 and "quote_token_values_net" in e.value.message and "hop_cost" in e.value.message
    u8, i32 = np.uint8, np.int32
    tin1, tout1, k1, a1 = (np.array(x) for x in ([4], [5], [0], [1.0]))
    off, typ, pool, tok = np.zeros(2, np.int64), np.zeros(4, i32), np.zeros(4, np.int64), np.zeros(4, np.int64)
    import ctypes as C
    P8, PI = C.POINTER(C.c_uint8), C.POINTER(C.c_int)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    mask = ok.astype(u8)
    k1 = k1.astype(u8)
    with pytest.raises(cr.CFMMError) as e:
        p._chk(p._lib.cfmm_find_order_paths_net(p._ctx, 1, ip(tin1), ip(tout1), k1.ctypes.data_as(P8), dp(a1), 4,
                                                mask.ctypes.data_as(P8), None, ip(off), typ.ctypes.data_as(PI),
                                                ip(pool), ip(tok), None, None, None, None, None))
    assert "null hop_cost" in e.value.message
    val = np.zeros(n)
    with pytest.raises(cr.CFMMError) as e:
        p._chk(p._lib.cfmm_quote_token_values_net(p._ctx, 1, ip(tin1), k1.ctypes.data_as(P8), dp(a1), 4, None, None,
                                                  dp(val), None, None, None, None, 0, None, None, None, None, None,
                                                  None, None, None, None))
    assert "null hop_cost" in e.value.message
    assert p.launch_count == l0
    assert same_state(before, hset.state(p))


def test_launches_and_profile_entries(cr, synth):
    """Best paths: the graph and path kernels, as cfmm_find_order_paths (one entry).  Token values:
    per group init, H relax, H finalize and H select passes and the rebuild: 2 + 3H launches, one
    entry; with requests also the entry map (one entry) and the path kernel."""
    ps = Pools(cr, synth)
    p = ps.p
    p.set_option("profile", 256)
    ok = np.ones(p.n_tokens, bool)

    def delta(fn):
        l0, c0 = p.launch_count, p.profile_read(PROF)[1]
        fn()
        return p.launch_count - l0, p.profile_read(PROF)[1] - c0

    args = ([1, 2, 3], [4, 5, 6], [0, 1, 0], [1.0, 1e-3, 0.0], 4, ok)
    p.find_order_paths(*args)  # builds the pair index and the adjacency
    assert delta(lambda: p.find_order_paths_net(*args, [1e-3, 1e-6, 0.0])) == (2, 1)
    assert delta(lambda: p.find_order_paths_net([], [], [], [], 4, ok, [])) == (0, 0)
    kappa = np.full(p.n_tokens, 1e-4)
    assert delta(lambda: p.quote_token_values_net([1, 2, 3], [0, 1, 0], [1.0, 1e-3, 2.0], 4, kappa)) == (14, 1)
    assert delta(lambda: p.quote_token_values_net([1, 2], [0, 1], [1.0, 1.0], 8, kappa, None,
                                                  ([0, 1], [5, 6]))) == (28, 2)
    q = 65  # two groups
    assert delta(lambda: p.quote_token_values_net(np.ones(q, np.int64), np.zeros(q, np.uint8), np.ones(q), 3,
                                                  kappa)) == (22, 2)
    assert delta(lambda: p.quote_token_values_net([], [], [], 3, kappa)) == (0, 0)
    p.close()
