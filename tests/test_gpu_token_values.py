"""cfmm_quote_token_values (include/cfmm_b200.h) on the device.

Values, hops, statuses and requested walks are checked bit for bit against a reference composed from
other entry points: token_value_oracle's DP driven by cfmm_pair_pools and cfmm_quote_swaps /
cfmm_quote_swaps_exact_out, on test_gpu_routed_orders' hub sets (all three types, appended and retired
pools, pools stored with their tokens exchanged), also after a retire that follows an earlier call,
cfmm_compact, a UniV3 liquidity change and an execute that moved pools.  cfmm_quote_paths on the
returned CSR gives the same amounts; one hop is the best active pool of the pair; on sets without
gaining cycles every value and walk is cfmm_find_order_paths'; on ProductTwoCoin more hops or tokens
never lower a value.  Beyond the 1024-token cap: a million Zipf-skewed ProductTwoCoin pools against the
numpy restatement, and a converged no-arbitrage set against a one-hop fixed-point certificate.  Rows
are independent of their batch, calls are repeatable and change no state, bad arguments are rejected
before anything runs, and the launches are pinned."""
import numpy as np
import pytest

import token_value_oracle as tv
from test_gpu_best_paths import device_lists, device_quote
from test_gpu_call_accounting import PROF, Pools
from test_gpu_parity import make_pools
from test_gpu_paths import same_state
from test_gpu_routed_orders import HubSet

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
INF = float("inf")


def composed(p, Ai, n, root, kind, amount, H, allowed):
    return tv.dp(root, kind, amount, device_lists(p, Ai, n), n, allowed, H, device_quote(p))


def check(hs, p, rng, hops=range(1, 9), roots=3):
    """Every (root, kind, H, mask): the call against the composed DP, every token's walk requested
    and priced again by cfmm_quote_paths."""
    n = hs.n
    tokens = np.arange(1, n + 1, dtype=np.int64)
    multi = 0
    for allowed in (None, rng.random(n) < 0.7):
        for kind in (0, 1):
            for root in rng.choice(np.arange(1, n + 1), size=roots, replace=False):
                amount = float(10.0 ** rng.uniform(-1, 2))
                for H in hops:
                    got = p.quote_token_values([root], [kind], [amount], H, allowed,
                                               (np.zeros(n, np.int64), tokens))
                    value, hp, st, front, off, ht, hpool, htok, x, lam, rst = got
                    ref = composed(p, hs.Ai, n, int(root), kind, amount, H, allowed)
                    assert np.array_equal(value[0], ref.value), (H, kind, value[0], ref.value)
                    assert np.array_equal(hp[0], ref.hops) and np.array_equal(st[0], ref.status)
                    assert np.array_equal(front[0], [len(x) for x in ref.pred])
                    assert np.array_equal(rst, st[0])
                    for t in tokens:
                        walk = ref.walk(int(t)) if st[0][t - 1] == tv.FILLED else []
                        seg = slice(off[t - 1], off[t])
                        assert [(int(a), int(b)) for a, b in zip(ht[seg], hpool[seg])] == [w[2] for w in walk]
                        assert list(htok[seg]) == [w[1] for w in walk]
                    rows = np.flatnonzero(np.diff(off) > 0)
                    multi += int(np.sum(np.diff(off) > 1))
                    if len(rows):
                        sub = np.concatenate([[0], np.cumsum(np.diff(off)[rows])]).astype(np.int64)
                        tin = tokens[rows] if kind else np.full(len(rows), root, np.int64)
                        qx, ql, qs = p.quote_paths(sub, ht, hpool, tin, np.full(len(rows), kind, np.uint8),
                                                   np.full(len(rows), amount))
                        assert np.array_equal(qx, x) and np.array_equal(ql, lam) and np.all(qs == 0)
                        last = qx[sub[:-1]] if kind else ql[sub[1:] - 1]
                        assert np.array_equal(last, value[0][rows])
    return multi


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U), (P, G, U)], ids=["product", "univ3", "mixed", "all"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=170 + len(request.param) + request.param[0])
    yield hs
    hs.p.close()


# ---- 1. bit-exact against the composed reference ------------------------------------------------------
def test_bit_exact_values_and_paths(hset):
    assert check(hset, hset.p, np.random.default_rng(1)) > 0  # some multi-hop walks


def test_after_retire_compact_liquidity_and_execute(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=97)
    p = hs.p
    rng = np.random.default_rng(2)
    check(hs, p, rng, hops=(2, 5), roots=2)
    t_hub = [(t, i) for t in (P, U) for i in range(hs.m[t]) if 1 in hs.Ai[t][i] and (t, i) not in hs.retired][:6]
    for t, i in t_hub:
        p.set_active(t, i, [False])
    hs.retired |= set(t_hub)
    check(hs, p, rng, hops=(2, 5), roots=2)
    p.compact()
    check(hs, p, rng, hops=(2, 5), roots=2)
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:4]
    s = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, s[ui] * 0.8, s[ui] * 1.25, np.full(len(ui), 2000.0))
    check(hs, p, rng, hops=(2, 5), roots=2)
    live = [i for i in range(hs.m[P]) if (P, i) not in hs.retired][:8]
    p.execute_swaps(P, live, np.column_stack([np.full(len(live), 30.0), np.zeros(len(live))]))
    check(hs, p, rng, hops=(2, 5), roots=2)
    p.close()


# ---- 2. against single pools, cfmm_find_order_paths and monotonicity ----------------------------------
def test_one_hop_is_the_best_active_pool(hset):
    p, n = hset.p, hset.n
    lists, quote = device_lists(p, hset.Ai, n), device_quote(p)
    for kind in (0, 1):
        for root in (1, 5, 9):
            value, _, st, _ = p.quote_token_values([root], [kind], [3.0], 1)
            for t in range(1, n + 1):
                if t == root:
                    continue
                lst = [(h, (t if kind else root) == t1, 3.0, bool(kind)) for h, t1, act in
                       lists.get((min(root, t), max(root, t)), []) if act]
                v = [x for x in (quote(lst) if lst else []) if (x < INF if kind else x > 0.0)]
                want = (min(v) if kind else max(v)) if v else (INF if kind else 0.0)
                assert value[0][t - 1] == want and st[0][t - 1] == (tv.FILLED if v else tv.UNREACHABLE)


def consistent_market(cr, n, m, seed, gamma=0.997):
    """ProductTwoCoin pools whose marginal prices all agree with one price vector: no gaining cycle."""
    rng = np.random.default_rng(seed)
    nu = np.exp(rng.uniform(-2, 2, size=n + 1))
    w = 1.0 / np.arange(1, n + 1) ** 0.8
    a = rng.choice(n, size=m, p=w / w.sum()) + 1
    b = rng.choice(n, size=m, p=w / w.sum()) + 1
    b = np.where(a == b, a % n + 1, b)
    A = np.column_stack([a, b]).astype(np.int64)
    depth = 10.0 ** rng.uniform(2, 4, size=m)
    R = depth[:, None] / nu[A]
    g = np.full(m, gamma)
    return make_pools(cr, n, product=(R, g, A)), (R, g, A)


def test_agrees_with_find_order_paths_without_gaining_cycles(cr):
    n = 60
    p, _ = consistent_market(cr, n, 400, seed=5)
    ok = np.ones(n, bool)
    checked = 0
    for kind in (0, 1):
        for root in (1, 2, 17, 40):
            amount = 1.0
            for H in (2, 4, 8):
                value, hp, st, _, off, ht, hpool, htok, x, lam, rst = p.quote_token_values(
                    [root], [kind], [amount], H, None, (np.zeros(n, np.int64), np.arange(1, n + 1)))
                others = np.array([t for t in range(1, n + 1) if t != root], np.int64)
                tin = others if kind else np.full(len(others), root, np.int64)
                tout = np.full(len(others), root, np.int64) if kind else others
                f = p.find_order_paths(tin, tout, np.full(len(others), kind, np.uint8), np.full(len(others), amount),
                                       H, ok)
                for r, t in enumerate(others):
                    assert st[0][t - 1] in (tv.FILLED, tv.UNREACHABLE)
                    assert f[7][r] == st[0][t - 1]
                    if st[0][t - 1] != tv.FILLED:
                        continue
                    assert f[6][r] == value[0][t - 1]
                    a, b = slice(f[0][r], f[0][r + 1]), slice(off[t - 1], off[t])
                    assert np.array_equal(f[1][a], ht[b]) and np.array_equal(f[2][a], hpool[b])
                    assert np.array_equal(f[4][a], x[b]) and np.array_equal(f[5][a], lam[b])
                    checked += 1
    assert checked > 300
    p.close()


def test_more_hops_and_tokens_never_lower_product_values(cr, synth):
    hs = HubSet(cr, synth, (P,), seed=99)
    p, n = hs.p, hs.n
    rng = np.random.default_rng(4)
    roots, kinds, amounts = np.array([1, 4, 7, 9]), np.array([0, 1, 0, 1], np.uint8), np.array([5.0, 2.0, 50.0, 0.5])
    small = rng.random(n) < 0.5
    prev_m = None
    for allowed in (small, small | (rng.random(n) < 0.5), np.ones(n, bool)):
        prev = None
        for H in range(1, 9):
            value = p.quote_token_values(roots, kinds, amounts, H, allowed)[0]
            for old in [x for x in (prev, prev_m if H == 8 else None) if x is not None]:
                better = np.where(kinds[:, None] == 0, value >= old, value <= old)
                assert np.all(better)
            prev = value
        prev_m = prev
    p.close()


# ---- 3. scale: beyond the 1024-token cap -----------------------------------------------------------------
def test_million_skewed_pools_against_numpy(cr, synth):
    m, n = 1_000_000, 20_000
    R, g, A = synth.product_pools_skewed(m, n, seed=77)
    p = make_pools(cr, n, product=(R, g, A))
    act = np.ones(m, bool)
    roots = np.array([1, 2, 50, 3000], np.int64)
    amounts = np.array([1e-3 * R[A[:, 0] == r][:, 0].mean() if np.any(A[:, 0] == r) else 1.0 for r in roots])
    allowed = np.random.default_rng(8).random(n) < 0.8
    for mask in (None, allowed):
        for H in (3, 8):
            value, hops, st, front = p.quote_token_values(roots, np.zeros(4, np.uint8), amounts, H, mask)
            for r, root in enumerate(roots):
                val, lvl, fr = tv.product(R, g, A, act, n, root, amounts[r], H, mask)
                assert np.array_equal(value[r], val), (H, root)
                assert np.array_equal(front[r], fr)
                reached = lvl >= 0
                assert np.all(st[r][~reached] == tv.UNREACHABLE) and np.all(hops[r][~reached] == 0)
                assert np.all(hops[r][reached & (st[r] == tv.FILLED)] == lvl[reached & (st[r] == tv.FILLED)])
            assert np.sum(value > 0) > 1000
    p.close()


def test_converged_values_are_a_fixed_point(cr):
    n, m = 20_000, 1_000_000
    p, (R, g, A) = consistent_market(cr, n, m, seed=9)
    roots, kinds = np.array([1, 1, 7, 7], np.int64), np.array([0, 1, 0, 1], np.uint8)
    amounts = np.array([10.0, 10.0, 3.0, 3.0])
    v7 = p.quote_token_values(roots, kinds, amounts, 7)
    v8 = p.quote_token_values(roots, kinds, amounts, 8)
    assert all(np.array_equal(a, b) for a, b in zip(v7[:3], v8[:3]))
    assert np.all(v8[3][:, 7] == 0)  # nothing changed at level 8: the DP has converged
    ids = np.arange(m)
    for r in range(len(roots)):
        val = v8[0][r]
        for side in (0, 1):
            u, v = A[:, side] - 1, A[:, 1 - side] - 1  # u tenders, v is delivered
            arg = np.zeros((m, 2))
            if kinds[r] == 0:
                sel = (val[u] > 0) & (v != roots[r] - 1)
                arg[:, side] = np.where(sel, val[u], 0.0)
                got = p.quote_swaps(P, ids, arg)[:, 1 - side]
                assert np.all(got[sel] <= val[v][sel])
            else:
                sel = (val[v] < INF) & (u != roots[r] - 1)
                arg[:, 1 - side] = np.where(sel, val[v], 0.0)
                got = p.quote_swaps_exact_out(P, ids, arg)[:, side]
                assert np.all(got[sel] >= val[u][sel])
        assert np.sum(val[val < INF] > 0) > n // 2
    p.close()


# ---- 4. call behaviour ---------------------------------------------------------------------------------------
def test_rows_are_independent_of_their_batch(hset):
    p, n = hset.p, hset.n
    rng = np.random.default_rng(10)
    q = 70  # more than one group of 64
    roots = rng.integers(1, n + 1, size=q)
    kinds = rng.integers(0, 2, size=q).astype(np.uint8)
    amounts = 10.0 ** rng.uniform(-1, 2, size=q)
    allowed = rng.random(n) < 0.8
    batch = p.quote_token_values(roots, kinds, amounts, 6, allowed)
    again = p.quote_token_values(roots, kinds, amounts, 6, allowed)
    assert all(np.array_equal(a, b) for a, b in zip(batch, again))
    order = rng.permutation(q)
    perm = p.quote_token_values(roots[order], kinds[order], amounts[order], 6, allowed)
    assert all(np.array_equal(a[order], b) for a, b in zip(batch, perm))
    for r in range(0, q, 7):
        one = p.quote_token_values(roots[r:r + 1], kinds[r:r + 1], amounts[r:r + 1], 6, allowed)
        assert all(np.array_equal(a[r:r + 1], b) for a, b in zip(batch, one))


def test_changes_nothing_and_rejects(cr, hset):
    p, n = hset.p, hset.n
    v = np.exp(np.random.default_rng(11).uniform(-1, 1, size=n))
    psi0, _ = p.sweep(v, materialize=True)
    t0 = [x.copy() for x in p.trades()]
    before = hset.state(p)
    p.quote_token_values(np.arange(1, n + 1), np.arange(n) % 2, np.full(n, 5.0), 8, None,
                         (np.arange(n), np.arange(n) + 1))
    assert same_state(before, hset.state(p))
    psi1, _ = p.sweep(v, materialize=True)
    assert np.array_equal(psi0, psi1) and all(np.array_equal(a, b) for a, b in zip(t0, p.trades()))
    bad = [dict(root=[0]), dict(root=[n + 1]), dict(kind=[2]), dict(amount=[np.nan]), dict(amount=[np.inf]),
           dict(amount=[0.0]), dict(amount=[-1.0]), dict(H=0), dict(H=9), dict(req=([1], [1])),
           dict(req=([-1], [1])), dict(req=([0], [0])), dict(req=([0], [n + 1]))]
    l0 = p.launch_count
    for b in bad:
        a = {**dict(root=[4], kind=[0], amount=[1.0], H=4, req=None), **b}
        with pytest.raises(cr.CFMMError) as e:
            p.quote_token_values(a["root"], a["kind"], a["amount"], a["H"], None, a["req"])
        assert e.value.code == -1 and "quote_token_values" in e.value.message
    with pytest.raises(cr.CFMMError) as e:  # a null required array
        p._chk(p._lib.cfmm_quote_token_values(p._ctx, 1, None, None, None, 4, None, None, None, None, None, 0, None,
                                              None, None, None, None, None, None, None, None))
    assert e.value.code == -1 and "null" in e.value.message
    p.quote_token_values([], [], [], 4)  # q == 0 runs nothing
    assert p.launch_count == l0
    assert same_state(before, hset.state(p))


def test_launches_and_profile_entries(cr, synth):
    """One group: init, H relax and H finalize passes, the rebuild: 2 + 2H launches, one entry; with
    requests also the entry map (one entry) and the path kernel."""
    ps = Pools(cr, synth)
    p = ps.p
    p.set_option("profile", 256)

    def delta(fn):
        l0, c0 = p.launch_count, p.profile_read(PROF)[1]
        fn()
        return p.launch_count - l0, p.profile_read(PROF)[1] - c0

    assert delta(lambda: p.quote_token_values([1, 2, 3], [0, 1, 0], [1.0, 1e-3, 2.0], 4)) == (10, 1)
    assert delta(lambda: p.quote_token_values([1, 2], [0, 1], [1.0, 1.0], 8, None, ([0, 1], [5, 6]))) == (20, 2)
    q = 65  # two groups
    assert delta(lambda: p.quote_token_values(np.ones(q, np.int64), np.zeros(q, np.uint8), np.ones(q), 3)) == (16, 2)
    assert delta(lambda: p.quote_token_values([], [], [], 3)) == (0, 0)
    p.close()
