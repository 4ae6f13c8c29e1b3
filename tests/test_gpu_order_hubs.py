"""cfmm_choose_order_hubs (include/cfmm_b200.h) on the device.

The choice is checked bit for bit against a reference composed from other entry points
(cfmm_pair_pools for each candidate's two pairs, cfmm_quote_swaps / cfmm_quote_swaps_exact_out on
their pools, max / min and the ranking on the host), which holds for all three pool types,
GeometricMeanTwoCoin included; for ProductTwoCoin and UniV3 also against hub_oracle.py.  The sets are
test_gpu_routed_orders' hub sets (appended and retired pools, pools stored with their tokens
exchanged), also after cfmm_compact, a UniV3 liquidity change and a retire that follows the
adjacency build.  Auto-routed rows are never worse than the best single route they were chosen by,
certified within order_certificate's allowance; choosing changes no state; executing with auto hubs
is choosing once and executing the routed rows; and the call's launches are pinned."""
import numpy as np
import pytest

import hub_oracle as ho
import order_certificate as oc
import swap_order_oracle as oo
from test_gpu_call_accounting import PROF, Pools
from test_gpu_order_certificates import PoolSet
from test_gpu_paths import same_state
from test_gpu_routed_orders import HubSet, keys_of
from test_gpu_split_orders import expected_pairs
from test_gpu_swap_orders import univ3_host_pools

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
INF = float("inf")


# ---- the composed reference ----------------------------------------------------------------------
def composed(p, Ai, n, tin, tout, kind, amount, max_hubs, allowed=None):
    """(hub_off, hubs, score, n_eligible) from cfmm_pair_pools and the swap quotes.  Ai: {type: the
    ingest token pairs of the type's pools in insertion order}."""
    cand = [(r, h) for r in range(len(tin)) for h in range(1, n + 1)
            if h not in (tin[r], tout[r]) and (allowed is None or allowed[h - 1]) and amount[r] > 0.0]
    a = [x for r, h in cand for x in (tin[r], h)]
    b = [x for r, h in cand for x in (h, tout[r])]
    off, typ, idx, act = p.pair_pools(a, b) if cand else (np.zeros(1, np.int64), [], [], [])
    lists = [[(int(typ[e]), int(idx[e]), bool(act[e])) for e in range(off[c], off[c + 1])] for c in range(len(a))]

    def quote(pools, t_in, x, out):
        """The quote of each active pool for tender (or want, out) x of token t_in, one call per type."""
        vals = []
        for t in (P, G, U):
            sel = [(k, i) for k, i, on in pools if k == t and on]
            if not sel:
                continue
            ids = np.array([i for _, i in sel], dtype=np.int64)
            tok1 = np.array([int(Ai[t][i][0]) == t_in for i in ids])
            arg = np.zeros((len(ids), 2))
            if out:  # want the other side: (0, y) when token 1 is tendered
                arg[tok1, 1], arg[~tok1, 0] = x, x
                res = p.quote_swaps_exact_out(t, ids, arg)
                vals += [res[k, 0] if tok1[k] else res[k, 1] for k in range(len(ids))]
            else:
                arg[tok1, 0], arg[~tok1, 1] = x, x
                res = p.quote_swaps(t, ids, arg)
                vals += [res[k, 1] if tok1[k] else res[k, 0] for k in range(len(ids))]
        return vals

    per_row = [[] for _ in tin]
    for c, (r, h) in enumerate(cand):
        jh, hi = lists[2 * c], lists[2 * c + 1]
        if not jh or not hi:
            continue  # not a common neighbour
        j, i = int(tin[r]), int(tout[r])
        if kind[r] == 0:
            x = 0.0
            for v in quote(jh, j, float(amount[r]), False):
                x = v if v > x else x
            o = 0.0
            if x > 0.0:
                for v in quote(hi, h, x, False):
                    o = v if v > o else o
            if o > 0.0:
                per_row[r].append((-o, h, o))
        else:
            cc = INF
            for v in quote(hi, h, float(amount[r]), True):
                cc = v if v < cc else cc
            x = INF
            if cc < INF:
                for v in quote(jh, j, cc, True):
                    x = v if v < x else x
            if x < INF:
                per_row[r].append((x, h, x))
    rows = []
    for el in per_row:
        el.sort()
        rows.append(([h for _, h, _ in el[:max_hubs]], [s for _, _, s in el[:max_hubs]], len(el)))
    return ho._pack(rows)


def mirror_market(hs, p):
    """hub_oracle pools (a, b, pool, active) at p's state (ProductTwoCoin and UniV3 sets)."""
    out = []
    if hs.m[P]:
        st = p.pool_state(P)[0]
        out += [(int(a), int(b), oo.ProductPool(st[i], hs.g[P][i]), (P, i) not in hs.retired)
                for i, (a, b) in enumerate(hs.Ai[P])]
    if hs.m[U]:
        out += [(int(a), int(b), pool, (U, i) not in hs.retired)
                for i, ((a, b), pool) in enumerate(zip(hs.Ai[U], univ3_host_pools(p, hs.g[U])))]
    return out


def order_rows(rng, n, q, lo=4):
    tin = rng.integers(lo, n + 1, size=q)
    tout = np.array([rng.choice([x for x in range(lo, n + 1) if x != a]) for a in tin])
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    amount = 10.0 ** rng.uniform(-2, 2.5, size=q)
    amount[::9] = 0.0
    return tin.astype(np.int64), tout.astype(np.int64), kind, amount


def same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y)), (x, y)


def check_choice(hs, p, rng, q=16, mirror=True, allowed=None):
    tin, tout, kind, amount = order_rows(rng, hs.n, q)
    for max_hubs in (0, 1, 3, 7):
        got = p.choose_order_hubs(tin, tout, kind, amount, max_hubs, allowed)
        same(got, composed(p, hs.Ai, hs.n, tin, tout, kind, amount, max_hubs, allowed))
        if mirror:
            same(got, ho.choose(mirror_market(hs, p), hs.n, tin, tout, kind, amount, max_hubs, allowed))
    assert got[3].max() > 0


@pytest.fixture(scope="module", params=[(P,), (U,), (P, U), (P, G, U)], ids=["product", "univ3", "mixed", "all"])
def hset(request, cr, synth):
    hs = HubSet(cr, synth, request.param, seed=140 + len(request.param) + request.param[0])
    yield hs
    hs.p.close()


# ---- 1. bit-exact ----------------------------------------------------------------------------------
def test_bit_exact_choice(hset):
    rng = np.random.default_rng(1)
    check_choice(hset, hset.p, rng, mirror=not hset.m[G])
    allowed = np.ones(hset.n, dtype=bool)
    allowed[[0, 5, 7]] = False  # hub 1 and two other tokens masked
    check_choice(hset, hset.p, rng, mirror=not hset.m[G], allowed=allowed)


def test_after_compact_liquidity_and_retire(cr, synth):
    hs = HubSet(cr, synth, (P, U), seed=93)
    p = hs.p
    rng = np.random.default_rng(2)
    check_choice(hs, p, rng)  # builds the adjacency
    # retire pools after the adjacency is built: their pairs stay listed, their routes go
    t_hub = [(t, i) for t in (P, U) for i in range(hs.m[t]) if 1 in hs.Ai[t][i] and (t, i) not in hs.retired][:6]
    for t, i in t_hub:
        p.set_active(t, i, [False])
    hs.retired |= set(t_hub)
    check_choice(hs, p, rng)
    p.compact()
    check_choice(hs, p, rng)
    ui = [i for i in range(hs.m[U]) if (U, i) not in hs.retired][:4]
    st = p.pool_state(U)[0]
    p.modify_univ3_liquidity(ui, st[ui] * 0.8, st[ui] * 1.25, np.full(len(ui), 2000.0))
    check_choice(hs, p, rng)
    p.close()


# ---- 2. exhaustive when small ----------------------------------------------------------------------
def test_all_eligible_hubs_when_few(cr, synth):
    """Hubs 1..7 pair with every token 8..20, and the other tokens pair only in disjoint couples, so a
    row between two non-hub tokens has exactly the hubs with an active pool on both sides."""
    from test_gpu_parity import make_pools
    rng = np.random.default_rng(5)
    n = 20
    A = [(h, x) for h in range(1, 8) for x in range(8, n + 1)] + [(8 + 2 * k, 9 + 2 * k) for k in range(6)]
    A = np.array([(a, b) if rng.random() < 0.5 else (b, a) for a, b in A], dtype=np.int64)
    R = np.exp(rng.uniform(5, 8, size=(len(A), 2)))
    p = make_pools(cr, n, product=(R, np.full(len(A), 0.997), A))
    off_ = rng.choice(len(A) - 6, size=20, replace=False)
    act = np.ones(len(A), bool)
    act[off_] = False
    p.set_active(P, 0, act)
    tin, tout = np.array([8, 9, 10, 12, 20, 15], np.int64), np.array([9, 10, 19, 11, 8, 14], np.int64)
    kind, amount = np.array([0, 1, 0, 1, 0, 1], np.uint8), np.array([1.0, 0.5, 3.0, 0.1, 2.0, 1.0])
    hub_off, hubs, score, n_elig = p.choose_order_hubs(tin, tout, kind, amount, 7)
    live = {tuple(sorted(A[k])) for k in range(len(A)) if act[k]}
    for r in range(len(tin)):
        want = {h for h in range(1, 8) if tuple(sorted((tin[r], h))) in live and tuple(sorted((h, tout[r]))) in live}
        assert set(hubs[hub_off[r]:hub_off[r + 1]].tolist()) == want and n_elig[r] == len(want), r
    assert n_elig.min() > 0
    p.close()


# ---- 3. never worse than the best single route --------------------------------------------------
def test_auto_routes_beat_single_routes(cr, synth):
    hs = HubSet(cr, synth, (P, G, U), seed=97, retire=True)
    p = hs.p
    rng = np.random.default_rng(3)
    tin, tout, kind, amount = order_rows(rng, hs.n, 10)
    amount[amount == 0.0] = 1.0
    objs = PoolSet.cert_pools(hs, p)
    ks = keys_of(hs)
    lst = lambda a, b: [objs[k] for k in expected_pairs(hs, ks, a, b)]
    split = p.quote_split_orders(tin, tout, kind, amount)
    prev, seen, filled = None, {}, 0
    for max_hubs in range(1, 8):
        hub_off, hubs, score, _ = p.choose_order_hubs(tin, tout, kind, amount, max_hubs)
        dev = p.quote_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
        paid, got, price, st, hp, hsur, (o, D, L) = dev
        for r in range(len(tin)):
            if st[r] != oc.FILLED:
                continue
            hr = tuple(int(h) for h in hubs[hub_off[r]:hub_off[r + 1]])
            if (r, hr) not in seen:  # a hub list seen at a smaller max_hubs gave the same row
                j, i = int(tin[r]), int(tout[r])
                row = oc.Row(lst(j, i), [(h, lst(j, h), lst(h, i)) for h in hr], j, i)
                g = slice(int(hub_off[r]), int(hub_off[r + 1]))
                out = dict(paid=paid[r], received=got[r], price=price[r], status=st[r], hub_price=hp[g],
                           hub_surplus=hsur[g], D=D[o[r]:o[r + 1]], L=L[o[r]:o[r + 1]])
                seen[(r, hr)] = float(oc.certify_row(row, kind[r], amount[r], out, nested=False)["allowance"] or 0.0)
                filled += 1
            allow = seen[(r, hr)]
            split_ok = split[3][r] == oc.FILLED
            if kind[r] == 0:
                single = ([score[hub_off[r]]] if hr else []) + ([split[1][r]] if split_ok else [])
                assert got[r] >= max(single, default=0.0) - allow, (r, got[r], single, allow)
                if prev is not None and prev[3][r] == oc.FILLED:
                    assert got[r] >= prev[1][r] - allow, r
            else:
                single = ([score[hub_off[r]]] if hr else []) + ([split[0][r]] if split_ok else [])
                slack = allow / price[r]  # the allowance is in units of i, paid in units of j
                assert paid[r] <= min(single, default=INF) + slack, (r, paid[r], single, allow)
                if prev is not None and prev[3][r] == oc.FILLED:
                    assert paid[r] <= prev[0][r] + slack, r
        prev = dev
    assert filled > len(tin) // 2
    p.close()


# ---- 4. read-only ------------------------------------------------------------------------------------
def test_choice_changes_nothing(cr, hset):
    p = hset.p
    before = hset.state(p)
    rng = np.random.default_rng(4)
    tin, tout, kind, amount = order_rows(rng, hset.n, 32)
    p.choose_order_hubs(tin, tout, kind, amount, 7)
    assert same_state(before, hset.state(p))
    bad = [dict(tin=[5]), dict(tin=[0]), dict(kind=[2]), dict(amount=[np.nan]), dict(amount=[-1.0]),
           dict(amount=[np.inf]), dict(max_hubs=8), dict(max_hubs=-1)]
    for b in bad:
        a = {**dict(tin=[4], tout=[5], kind=[0], amount=[1.0], max_hubs=7), **b}
        with pytest.raises(cr.CFMMError) as e:
            p.choose_order_hubs(a["tin"], a["tout"], a["kind"], a["amount"], a["max_hubs"])
        assert e.value.code == -1 and "choose_order_hubs" in e.value.message
    assert same_state(before, hset.state(p))


# ---- 5. execute ---------------------------------------------------------------------------------------
def router_market(cr, seed, n=12):
    rng = np.random.default_rng(seed)
    cs = []
    for a in range(1, n + 1):
        for b in range(a + 1, n + 1):
            if a <= 4 or rng.random() < 0.25:
                R = rng.uniform(500, 5000) * np.exp(rng.uniform(-0.1, 0.1, size=2))
                cs.append(cr.ProductTwoCoin(R, 0.997, [a, b]))
    return cr.Router(cr.LinearNonnegative(np.ones(n)), cs, n)


def test_execute_is_choose_then_routed_execute(cr):
    r1, r2 = router_market(cr, 11), router_market(cr, 11)
    rng = np.random.default_rng(6)
    tin, tout, kind, amount = order_rows(rng, 12, 24, lo=5)
    tin[:8], tout[:8] = 5, 6  # rows sharing a pair: later rows run on the state earlier rows left
    q1 = r1.quote_auto_routed_orders(tin, tout, kind, amount)
    lim = np.where(kind == 1, q1[0] * 1.01, q1[1] * 0.99)
    lim[::4] = np.where(kind[::4] == 1, 0.0, 1e300)  # some rows revert
    lim = np.maximum(lim, 0.0)  # (pools priced apart: a row can arbitrage them and net a negative paid)
    a = r1.execute_auto_routed_orders(tin, tout, kind, amount, lim, max_hubs=5)
    hubs = r2.choose_hubs(tin, tout, kind, amount, max_hubs=5)
    b = r2.execute_routed_orders(tin, tout, kind, amount, hubs, lim)
    assert a[4] == hubs
    same(a[:4], b)
    assert len(set(a[3].tolist())) > 1
    assert np.array_equal(r1._pools.pool_state(P)[0], r2._pools.pool_state(P)[0])
    assert all(np.array_equal(c1.R, c2.R) for c1, c2 in zip(r1.cfmms, r2.cfmms))
    # quoting with auto hubs is choose_hubs followed by quote_routed_orders
    hq = r1.choose_hubs(tin, tout, kind, amount)
    same(r1.quote_auto_routed_orders(tin, tout, kind, amount)[:4],
         r1.quote_routed_orders(tin, tout, kind, amount, hq))
    r1._pools.close()
    r2._pools.close()


# ---- 6. launches ---------------------------------------------------------------------------------------
def test_launches_and_profile_entries(cr, synth):
    """One call on test_gpu_call_accounting's seeded set: with nothing built, the pair index (9 launches:
    one key kernel per non-empty pool set, sort, run-length, scan; one entry), the adjacency (3, one
    entry) and the choice kernel (1, one entry); with the pair index but no adjacency, 3 + 1; warm, 1."""
    ps = Pools(cr, synth)
    p = ps.p
    p.set_option("profile", 256)
    args = ([1, 2, 3], [4, 5, 6], [0, 1, 0], [1.0, 1e-3, 0.0], 7)

    def delta(fn):
        l0, c0 = p.launch_count, p.profile_read(PROF)[1]
        fn()
        return p.launch_count - l0, p.profile_read(PROF)[1] - c0

    assert delta(lambda: p.choose_order_hubs(*args)) == (13, 3)
    assert delta(lambda: p.choose_order_hubs(*args)) == (1, 1)
    p.append_product(*synth.product_pools(3, 16, seed=31))  # drops the pair index and the adjacency
    p.pair_pools([1], [2])  # rebuilds the pair index only
    assert delta(lambda: p.choose_order_hubs(*args)) == (4, 2)
    assert delta(lambda: p.choose_order_hubs(*args)) == (1, 1)
    assert delta(lambda: p.choose_order_hubs([], [], [], [], 7)) == (0, 0)
    p.close()
