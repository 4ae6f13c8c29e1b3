"""The per-row mask calls (include/cfmm_b200.h, "per-row masks") on the device: subgraph (exact-in and
exact-out), basket (sell-only and buy) and limit rows, each over its own list of allowed tokens.

On the five markets of test_gpu_subgraph_orders: every row given the same list is the one-mask call bit
for bit (every output, and on execute the per-row results and the final pool state, UniV3 ladders
included); in a batch of rows with different lists (empty ones, ones holding the row's own tokens) each
row is the one-mask call run on that row alone with its list as the mask, and lists the oracle's token
set and pools; a batch execute equals the rows executed one at a time in batch order.  The launches of
the new calls are pinned: rows on disjoint token sets share a level.  Chosen hubs go in as lists and
filled rows pass the 50-digit certificate.  Malformed lists are rejected and change nothing."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
import row_mask_oracle as rm
import subgraph_oracle as so
import limit_order_oracle as lo
import solve_certificate as sc
from test_gpu_basket_orders import baskets
from test_gpu_limit_orders import limits_around
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, certify_row, fields, fresh, global_index, mask,
                                      pair_lists, row_slices, rows, same_state, state)

pytestmark = pytest.mark.gpu

INVALID = -1  # CFMM_ERR_INVALID


def full_state(p):
    return state(p) + [p.univ3_ticks()]


def same_full(a, b):
    same_state(a[:3], b[:3])
    assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))


def same_out(a, b):
    for x, y in zip(fields(a), fields(b)):
        assert np.array_equal(x, y)
    assert np.array_equal(a.tok_off, b.tok_off) and np.array_equal(a.leg_off, b.leg_off)
    if hasattr(a, "surplus"):
        assert np.array_equal(a.surplus, b.surplus)


def same_row(a, r, b, paid=None):
    """Row r of out a against row 0 of out b, every field (paid: row r's slice of a.paid)."""
    pa = a.paid[paid] if paid is not None else a.paid[r:r + 1]
    assert np.array_equal(pa, b.paid)
    for f in ("received", "status", "solver_status", "iterations", "fun_evals", "merit"):
        assert getattr(a, f)[r] == getattr(b, f)[0], (f, r)
    ts, sl = row_slices(a, r)
    for f in ("token", "nu", "psi"):
        assert np.array_equal(getattr(a, f)[ts], getattr(b, f)), (f, r)
    for f in ("leg_type", "leg_pool", "leg_delta", "leg_lambda"):
        assert np.array_equal(getattr(a, f)[sl], getattr(b, f)), (f, r)
    if hasattr(a, "surplus"):
        assert a.surplus[r] == b.surplus[0]


def lists_of(allowed, q):
    return [np.flatnonzero(allowed).astype(np.int64) + 1 for _ in range(q)] if q else []


def mixed_lists(rng, own):
    """One list per row: empty, with the row's own tokens, or random, of up to 9 tokens."""
    out = []
    for r, o in enumerate(own):
        k = r % 4
        if k == 0:
            out.append([])
        else:
            lst = rng.choice(np.arange(1, N + 1), size=int(rng.integers(1, 9)), replace=False).tolist()
            if k == 1:
                lst = list(dict.fromkeys(lst + list(o)))
            out.append(lst)
    return out


def swap_kinds(rng, off):
    """Entry kinds with some buy rows (one bought entry) and some sell-only rows."""
    kind = np.zeros(off[-1], np.uint8)
    for r in range(len(off) - 1):
        if r % 3 == 1:
            kind[off[r + 1] - 1] = 1
    return kind


def batch(rng, q=9):
    tin, tout, amt = rows(rng, q)
    kind = np.array([r % 3 == 2 for r in range(q)], np.uint8)
    amt[kind == 1] *= 0.1                          # exact-out: buy a smaller amount
    amt[4] = 0.0
    tb, ob, kb, ab = baskets(rng, q, 4)
    ek = swap_kinds(rng, ob)
    ab[ek == 1] *= 0.1
    return (tin, tout, amt, kind), (tb, ob, kb, ab, ek)


# ---- 1. the same list on every row is the one-mask call ---------------------------------------------
@pytest.mark.parametrize("state_name", STATES)
def test_same_list_everywhere_is_the_one_mask_call(state_name):
    rng = np.random.default_rng(21)
    ma, mb = Market(state_name), Market(state_name)
    try:
        pa, pb = ma.p, mb.p
        allowed = mask(rng, 6)
        (tin, tout, amt, kind), (tb, ob, kb, ab, ek) = batch(rng)
        lst = lists_of(allowed, len(tin))
        c = limits_around(pa, tb, ob, kb, ab, allowed, rng)
        same_out(pa.quote_subgraph_orders(tin, tout, amt, allowed, kind=kind),
                 pb.quote_subgraph_orders(tin, tout, amt, lst, kind=kind))
        same_out(pa.quote_basket_orders(tb, ob, kb, ab, allowed), pb.quote_basket_orders(tb, ob, kb, ab, lst))
        same_out(pa.quote_basket_orders(tb, ob, kb, ab, allowed, kind=ek),
                 pb.quote_basket_orders(tb, ob, kb, ab, lst, kind=ek))
        same_out(pa.quote_limit_orders(tb, ob, kb, ab, c, allowed), pb.quote_limit_orders(tb, ob, kb, ab, c, lst))
        same_full(full_state(pa), full_state(pb))
        # executes: outputs and the final state after each family
        same_out(pa.execute_subgraph_orders(tin, tout, amt, allowed, kind=kind),
                 pb.execute_subgraph_orders(tin, tout, amt, lst, kind=kind))
        same_full(full_state(pa), full_state(pb))
        same_out(pa.execute_basket_orders(tb, ob, kb, ab, allowed, kind=ek),
                 pb.execute_basket_orders(tb, ob, kb, ab, lst, kind=ek))
        same_full(full_state(pa), full_state(pb))
        same_out(pa.execute_limit_orders(tb, ob, kb, ab, c, allowed), pb.execute_limit_orders(tb, ob, kb, ab, c, lst))
        same_full(full_state(pa), full_state(pb))
    finally:
        ma.close()
        mb.close()


# ---- 2. a row depends only on its own list ------------------------------------------------------------
@pytest.mark.parametrize("state_name", STATES)
def test_each_row_is_the_one_mask_call_on_its_own_list(state_name):
    rng = np.random.default_rng(22)
    m = Market(state_name)
    try:
        p = m.p
        pl = pair_lists(p)
        (tin, tout, amt, kind), (tb, ob, kb, ab, ek) = batch(rng, 12)
        ls = mixed_lists(rng, [(int(a), int(b)) for a, b in zip(tin, tout)])
        out = p.quote_subgraph_orders(tin, tout, amt, ls, kind=kind)
        for r in range(len(tin)):
            one = p.quote_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], rm.row_mask(ls[r], N),
                                          kind=kind[r:r + 1])
            same_row(out, r, one)
            T, pools = so.row_subgraph(pl, int(tin[r]), int(tout[r]), rm.row_mask(ls[r], N))
            ts, sl = row_slices(out, r)
            assert out.token[ts].tolist() == T
            assert set(T) <= rm.own_subgraph(tin[r], tout[r], ls[r])
            want = sorted(pools, key=lambda h: global_index(*h))
            assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == want
        bl = mixed_lists(rng, [[int(tb[r])] + kb[ob[r]:ob[r + 1]].tolist() for r in range(len(tb))])
        c = limits_around(p, tb, ob, kb, ab, bl, rng)
        outs = [(p.quote_basket_orders(tb, ob, kb, ab, bl, kind=ek), "basket"),
                (p.quote_limit_orders(tb, ob, kb, ab, c, bl), "limit")]
        for out, fam in outs:
            for r in range(len(tb)):
                e = slice(ob[r], ob[r + 1])
                args = (tb[r:r + 1], np.array([0, ob[r + 1] - ob[r]], np.int64), kb[e], ab[e])
                if fam == "basket":
                    one = p.quote_basket_orders(*args, rm.row_mask(bl[r], N), kind=ek[e])
                else:
                    one = p.quote_limit_orders(*args, c[e], rm.row_mask(bl[r], N))
                    T = lo.row_limit(pl, kb[e].tolist(), ab[e].tolist(), c[e].tolist(), int(tb[r]),
                                     rm.row_mask(bl[r], N))[0]
                    assert out.token[row_slices(out, r)[0]].tolist() == T
                same_row(out, r, one, paid=e)
    finally:
        m.close()


# ---- 3. execute: batch order, levels over each row's own tokens ---------------------------------------
@pytest.mark.parametrize("state_name", STATES)
def test_batch_execute_is_rows_one_at_a_time(state_name):
    rng = np.random.default_rng(23)
    ma, mb = Market(state_name), Market(state_name)
    try:
        pa, pb = ma.p, mb.p
        (tin, tout, amt, kind), (tb, ob, kb, ab, ek) = batch(rng, 10)
        ls = mixed_lists(rng, [(int(a), int(b)) for a, b in zip(tin, tout)])
        out = pa.execute_subgraph_orders(tin, tout, amt, ls, kind=kind)
        for r in range(len(tin)):
            one = pb.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], [ls[r]], kind=kind[r:r + 1])
            same_row(out, r, one)
        assert np.any(out.status == 0)
        same_full(full_state(pa), full_state(pb))
        bl = mixed_lists(rng, [[int(tb[r])] + kb[ob[r]:ob[r + 1]].tolist() for r in range(len(tb))])
        c = limits_around(pa, tb, ob, kb, ab, bl, rng)
        for fam in ("basket", "limit"):
            if fam == "basket":
                out = pa.execute_basket_orders(tb, ob, kb, ab, bl, kind=ek)
            else:
                out = pa.execute_limit_orders(tb, ob, kb, ab, c, bl)
            for r in range(len(tb)):
                e = slice(ob[r], ob[r + 1])
                args = (tb[r:r + 1], np.array([0, ob[r + 1] - ob[r]], np.int64), kb[e], ab[e])
                if fam == "basket":
                    one = pb.execute_basket_orders(*args, [bl[r]], kind=ek[e])
                else:
                    one = pb.execute_limit_orders(*args, c[e], [bl[r]])
                same_row(out, r, one, paid=e)
            same_full(full_state(pa), full_state(pb))
    finally:
        ma.close()
        mb.close()


def test_launches_rows_on_disjoint_tokens_share_a_level():
    """Launches per call (the plan, then one per kind of row in each level; the size query first runs
    the plan alone).  The rows revert on their limits, so no bookkeeping runs."""
    m = Market()
    try:
        p = m.p
        p.quote_subgraph_orders([1], [2], [1.0], [[3]])               # (the adjacency is built once)
        tin, tout = np.arange(1, 9, 2, dtype=np.int64), np.arange(2, 10, 2, dtype=np.int64)
        amt, big = np.full(4, 2.0), np.full(4, 1e300)
        disjoint = [[11], [12], [13], [14]]
        shared = [[11, 15], [12, 15], [13, 15], [14, 15]]

        def delta(f):
            n0 = p.launch_count
            out = f()
            return p.launch_count - n0, out

        n, _ = delta(lambda: p.quote_subgraph_orders(tin, tout, amt, disjoint))
        assert n == 3
        n, _ = delta(lambda: p.quote_subgraph_orders(tin, tout, amt, disjoint, kind=[0, 1, 0, 1]))
        assert n == 4
        before = full_state(p)
        n, out = delta(lambda: p.execute_subgraph_orders(tin, tout, amt, disjoint, limit=big))
        assert n == 3 and np.all(out.status == cr._lib.ORDER_LIMIT)
        assert rm.launches(rm.levels([rm.own_subgraph(a, b, l) for a, b, l in zip(tin, tout, disjoint)]),
                           [False] * 4) == 1
        n, out = delta(lambda: p.execute_subgraph_orders(tin, tout, amt, shared, limit=big))
        assert n == 6 and np.all(out.status == cr._lib.ORDER_LIMIT)
        # (an exact-out row can pay nothing when its pools hold a cycle, so it cannot be made to revert on
        # its limit: these ask for more than their pools hold and are unreachable)
        n, out = delta(lambda: p.execute_subgraph_orders(tin, tout, np.array([2.0, 1e15, 2.0, 1e15]), disjoint,
                                                         limit=big, kind=[0, 1, 0, 1]))
        assert n == 4 and out.status.tolist() == [cr._lib.ORDER_LIMIT, cr._lib.ORDER_UNREACHABLE] * 2
        # basket and limit rows: one launch per level; buy rows a second one
        tb = np.array([1, 3, 5, 7], np.int64)
        ob = np.arange(0, 5, dtype=np.int64)
        kb = np.array([2, 4, 6, 8], np.int64)
        ab = np.full(4, 2.0)
        n, _ = delta(lambda: p.quote_basket_orders(tb, ob, kb, ab, disjoint))
        assert n == 3
        n, _ = delta(lambda: p.quote_basket_orders(tb, ob, kb, ab * 0.1, disjoint, kind=[0, 1, 0, 0]))
        assert n == 4
        n, out = delta(lambda: p.execute_basket_orders(tb, ob, kb, ab, disjoint, limit=big))
        assert n == 3 and np.all(out.status == cr._lib.ORDER_LIMIT)
        n, out = delta(lambda: p.execute_basket_orders(tb, ob, kb, ab, shared, limit=big))
        assert n == 6
        n, _ = delta(lambda: p.quote_limit_orders(tb, ob, kb, ab, np.zeros(4), disjoint))
        assert n == 3
        n, out = delta(lambda: p.execute_limit_orders(tb, ob, kb, ab, np.zeros(4), disjoint, min_received=big))
        assert n == 3 and np.all(out.status == cr._lib.ORDER_LIMIT)
        n, out = delta(lambda: p.execute_limit_orders(tb, ob, kb, ab, np.zeros(4), shared, min_received=big))
        assert n == 6
        same_full(before, full_state(p))
    finally:
        m.close()


# ---- 4. chosen hubs as lists ---------------------------------------------------------------------------
def test_chosen_hubs_as_lists_certify():
    m = Market()
    try:
        p = m.p
        rng = np.random.default_rng(24)
        tin, tout, amt = rows(rng, 12)
        kind = np.zeros(len(tin), np.uint8)
        off, flat, _, _ = p.choose_order_hubs(tin, tout, kind, amt, 7)
        hubs = [flat[off[r]:off[r + 1]].tolist() for r in range(len(tin))]
        out = p.quote_subgraph_orders(tin, tout, amt, hubs)
        done = 0
        for r in np.flatnonzero(out.status == 0)[:4]:
            ts, sl = row_slices(out, r)
            pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
            q, order, cert = fresh(m, pools)
            try:
                certify_row(cert, order, out, r, amt[r], int(tin[r]), int(tout[r]))
                done += 1
            finally:
                q.close()
        assert done >= 3
        # limit rows selling token_in for token_out over the same hubs, with their limits
        ob = np.arange(len(tin) + 1, dtype=np.int64)
        c = limits_around(p, tout, ob, tin, amt, hubs, rng)
        out = p.quote_limit_orders(tout, ob, tin, amt, c, hubs)
        done = 0
        for r in np.flatnonzero((out.status == 0) & (out.solver_status == 0))[:3]:
            ts, sl = row_slices(out, r)
            toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
            pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
            q, order, cert = fresh(m, pools)
            try:
                nu = np.ones(N)
                nu[toks - 1] = nu_r
                D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
                D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
                lin, cc = np.zeros(N), np.zeros(N)
                if int(tin[r]) in set(toks.tolist()):
                    lin[tin[r] - 1], cc[tin[r] - 1] = amt[r], c[r]
                obj = cr.LimitBasket(int(tout[r]), lin, cc)
                ref = cc.copy()
                ref[int(tout[r]) - 1] = 1.0
                box = sc.Box(obj.linear_term(), obj.lower_limit(), ref=ref)
                V = float(np.sum(lin[toks - 1] * nu_r))
                pgtol = float(np.max(out.merit[r] * V / nu_r)) * (1 + 1e-9)
                res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
                floor, _ = lo.surplus_floor(toks.tolist(), tin[r:r + 1], amt[r:r + 1], c[r:r + 1], nu_r, psi, RTOL)
                assert res["gap"] <= -floor + res["allowance"], (res, floor)
                done += 1
            finally:
                q.close()
        assert done >= 2
    finally:
        m.close()


def test_router_takes_choose_hubs_output():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 25)
    try:
        rng = np.random.default_rng(25)
        tin = rng.integers(5, 13, size=6)
        tout = (tin - 5 + rng.integers(1, 8, size=6)) % 8 + 5
        amt = rng.uniform(1.0, 20.0, size=6)
        kinds = np.zeros(6, np.uint8)
        hubs = r.choose_hubs(tin, tout, kinds, amt)
        paid, recv, st, det = r.quote_subgraph_orders(tin, tout, amt, hubs)
        for k in range(6):
            one = r.quote_subgraph_orders(tin[k:k + 1], tout[k:k + 1], amt[k:k + 1], rm.row_mask(hubs[k], 12))[3]
            same_row(det, k, one)
        assert np.any(st == 0)
    finally:
        r.close() if hasattr(r, "close") else None


# ---- 5. rejections -------------------------------------------------------------------------------------
def test_rejections_change_nothing():
    m = Market()
    try:
        p = m.p
        lib = p._lib
        ip, dp, u8 = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_uint8)
        before = full_state(p)
        a64 = lambda x: np.asarray(x, np.int64)  # noqa: E731

        def calls(aoff, atok, amount=1.0):
            """Every _rows call on row (1 -> 2) or the basket {1} -> 2, with the given CSR (None: null)."""
            P = lambda x: None if x is None else x.ctypes.data_as(ip)  # noqa: E731
            q = 1 if aoff is None else len(aoff) - 1
            ti, to = a64([1] * q), a64([2] * q)
            am = np.full(q, amount)
            bo, bt, ba, lp = a64(range(q + 1)), a64([1] * q), np.full(q, amount), np.zeros(q)
            so_, bo_, lo_ = cr._lib.SubgraphOut(), cr._lib.BasketOut(), cr._lib.LimitOut()
            o, t = P(aoff), P(atok)
            return [
                lib.cfmm_quote_subgraph_swap_orders_rows(p._ctx, q, P(ti), P(to), None, am.ctypes.data_as(dp), o, t,
                                                         None, C.byref(so_)),
                lib.cfmm_execute_subgraph_swap_orders_rows(p._ctx, q, P(ti), P(to), None, am.ctypes.data_as(dp), None,
                                                           o, t, None, C.byref(so_)),
                lib.cfmm_quote_basket_swap_orders_rows(p._ctx, q, P(to), P(bo), P(bt), None, ba.ctypes.data_as(dp), o,
                                                       t, None, C.byref(bo_)),
                lib.cfmm_execute_basket_swap_orders_rows(p._ctx, q, P(to), P(bo), P(bt), None, ba.ctypes.data_as(dp),
                                                         None, o, t, None, C.byref(bo_)),
                lib.cfmm_quote_limit_orders_rows(p._ctx, q, P(to), P(bo), P(bt), ba.ctypes.data_as(dp),
                                                 lp.ctypes.data_as(dp), o, t, None, C.byref(lo_)),
                lib.cfmm_execute_limit_orders_rows(p._ctx, q, P(to), P(bo), P(bt), ba.ctypes.data_as(dp),
                                                   lp.ctypes.data_as(dp), None, o, t, None, C.byref(lo_)),
            ]

        assert calls(a64([0, 1]), a64([3]), amount=0.0) == [0] * 6     # (amount 0: no trade)
        bad = [
            (None, a64([3])),                    # a null allow_off
            (a64([0, 1]), None),                 # a null allow_token with a listed token
            (a64([1, 1]), a64([3])),             # allow_off[0] != 0
            (a64([0, 2, 1]), a64([3, 4])),       # decreasing
            (a64([0, 2, 0]), None),              # decreasing back to 0, with a null allow_token
            (a64([0, 1]), a64([0])),             # outside 1..n_tokens
            (a64([0, 1]), a64([N + 1])),
            (a64([0, 2]), a64([3, 3])),          # listed twice in one row
        ]
        for aoff, atok in bad:
            assert calls(aoff, atok) == [INVALID] * 6, (aoff, atok)
        assert calls(a64([0, 1]), a64([3]), amount=float("nan")) == [INVALID] * 6   # the one-mask call's errors
        same_full(before, full_state(p))
    finally:
        m.close()


def test_size_limit_and_the_largest_rows():
    """At most CFMM_SUBGRAPH_MAX_TOKENS tokens in B_r (basket rows: that plus one besides i, entries
    included); the largest rows run, over a row graph of CFMM_SUBGRAPH_MAX_TOKENS + 2 slots."""
    from cfmmrouter_b200 import synth
    n = 300
    p = cr.DevicePools(n, device=0)
    try:
        R, g, A = synth.product_pools(2000, n, seed=31)
        p.add_product(R, g, A)
        p.finalize()
        before = state(p)
        B = [t for t in range(1, n + 1) if t not in (1, 2)]
        ip, dp = C.POINTER(C.c_int64), C.POINTER(C.c_double)
        keep = []

        def P(x, t=np.int64, ptr=ip):
            keep.append(np.asarray(x, t))
            return keep[-1].ctypes.data_as(ptr)

        def c_quote(lst, basket):
            off = P([0, len(lst)])
            if basket:
                return p._lib.cfmm_quote_basket_swap_orders_rows(p._ctx, 1, P([2]), P([0, 1]), P([1]), None,
                                                                 P([1.0], np.float64, dp), off, P(lst), None,
                                                                 C.byref(cr._lib.BasketOut()))
            return p._lib.cfmm_quote_subgraph_swap_orders_rows(p._ctx, 1, P([1]), P([2]), None, P([1.0], np.float64, dp),
                                                               off, P(lst), None, C.byref(cr._lib.SubgraphOut()))

        assert c_quote([1, 2] + B[:257], False) == INVALID and c_quote([1, 2] + B[:256], False) == 0
        assert c_quote(B[:257], True) == INVALID and c_quote([1, 2] + B[:256], True) == 0
        with pytest.raises(ValueError, match="more than 256"):
            p.quote_subgraph_orders([1], [2], [1.0], [[1, 2] + B[:257]])
        out = p.quote_subgraph_orders([1], [2], [1.0], [[2, 1] + B[:256]])
        one = p.quote_subgraph_orders([1], [2], [1.0], rm.row_mask([1, 2] + B[:256], n))
        same_out(out, one)
        with pytest.raises(ValueError, match="more than 256"):
            p.quote_basket_orders([2], [0, 1], [1], [1.0], [B[:257]])
        out = p.quote_basket_orders([2], [0, 1], [1], [1.0], [[1, 2] + B[:256]])
        same_out(out, p.quote_basket_orders([2], [0, 1], [1], [1.0], rm.row_mask([1, 2] + B[:256], n)))
        same_state(before, state(p))
    finally:
        p.close()
