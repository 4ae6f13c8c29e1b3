"""Exact-out rows of cfmm_quote_subgraph_swap_orders / cfmm_execute_subgraph_swap_orders
(include/cfmm_b200.h) on the device.

On the five states of test_gpu_subgraph_orders (plain, pools stored exchanged, after cfmm_compact,
after a UniV3 liquidity change, retires after the adjacency build): each filled exact-out row keeps the
fill promise, its legs are a materialising cfmm_sweep at its ν bit for bit, its Ψ the stated warp-tree
sums, and a row asking for what the exact-in quote of the same row received pays that row's tender
within both stops.  On the plain market: the 50-digit certificate on the row's raw box and
cfmm_solve's dual value on a fresh context holding only the row's pools; exact-in rows unchanged
(kind None, 0 and the old entry points); mixed batches independent of their rows' company; paid no
more than split, auto-routed and best-path exact-out; a mixed batch execute equal to its rows one at a
time; max-paid limits; the execute's transition equal to cfmm_apply_trades on a fresh context; the
capacity rule, an unservable row, amount 0; argument errors that change nothing; and the Router."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
import solve_certificate as sc
import subgraph_exact_out_oracle as xo
import subgraph_oracle as so
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, fields, fresh, global_index, mask, pair_lists,
                                      row_slices, rows, same_state, state)

pytestmark = pytest.mark.gpu

OUT = cr._lib.SWAP_EXACT_OUT
NC = cr._lib.ORDER_NOT_CONVERGED
DBL_MAX = float(np.finfo(np.float64).max)


@pytest.fixture(scope="module")
def mk():
    m = Market()
    yield m.p, m.Ai, m
    m.close()


def out_rows(p, rng, allowed, q):
    """Rows whose exact-out amounts are what the exact-in quote of the same row received (the rest of
    the exact-in quote is returned too)."""
    tin, tout, delta = rows(rng, q)
    qi = p.quote_subgraph_orders(tin, tout, delta, allowed)
    y = np.where(qi.status == 0, qi.received, delta)
    return tin, tout, delta, y, qi


def check_out_row(p, Ai, out, r, y):
    """The fill promise of filled exact-out row r; legs against a materialising sweep, Ψ the stated sums."""
    ts, sl = row_slices(out, r)
    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
    v = np.ones(N)
    v[toks - 1] = nu
    p.sweep(v, materialize=True)
    D, L = p.trades()
    g = np.array([global_index(int(t), int(i)) for t, i in zip(out.leg_type[sl], out.leg_pool[sl])], np.int64)
    assert np.array_equal(D[g], out.leg_delta[sl]) and np.array_equal(L[g], out.leg_lambda[sl])
    A = so.ingest_tokens(Ai, out.leg_type[sl], out.leg_pool[sl])
    assert np.array_equal(so.warp_psi(A, out.leg_delta[sl], out.leg_lambda[sl], toks), psi)
    assert out.received[r] == psi[0] and out.paid[r] == 0.0 - psi[1]
    assert out.merit[r] <= RTOL and out.solver_status[r] == 0
    assert nu[1] == 1.0 and np.all(nu >= xo.SQRT_EPS)
    assert out.received[r] >= y
    if nu[0] > xo.SQRT_EPS:
        assert out.received[r] <= y * (1 + 2 * RTOL) * (1 + 1e-12), (out.received[r], y)
    assert np.all(psi[2:] >= -1.01 * RTOL * y * nu[0] / nu[2:])


def check_not_filled(out, r):
    _, sl = row_slices(out, r)
    assert out.paid[r] == 0.0 and out.received[r] == 0.0 and not np.any(out.leg_delta[sl])
    assert not np.any(out.leg_lambda[sl])


@pytest.mark.parametrize("state_name", STATES)
def test_fill_promise_and_round_trip_on_every_state(state_name):
    m = Market(state_name)
    try:
        p = m.p
        rng = np.random.default_rng(21)
        lists = pair_lists(p)
        n_fill = n_short = 0
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            tin, tout, delta, y, qi = out_rows(p, rng, allowed, 10)
            y[4] = 0.0
            out = p.quote_subgraph_orders(tin, tout, y, allowed, kind=OUT)
            for r in range(len(tin)):
                T, pools = so.row_subgraph(lists, int(tin[r]), int(tout[r]), allowed)
                ts, sl = row_slices(out, r)
                assert out.token[ts].tolist() == T
                want = sorted([(t, i) for t, i in pools], key=lambda h: global_index(*h))
                assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == want
                if y[r] == 0.0:
                    assert out.status[r] == 0 and out.solver_status[r] == -1
                    check_not_filled(out, r)
                elif int(tin[r]) not in T:
                    assert out.status[r] == cr._lib.ORDER_UNREACHABLE
                    check_not_filled(out, r)
                elif out.status[r] == 0:
                    n_fill += 1
                    check_out_row(p, m.Ai, out, r, y[r])
                    if qi.status[r] == 0:
                        # the round trip: buying what δ bought pays δ, within both stops and both gaps
                        nt = len(T)
                        bound = (nt + 1) * RTOL * delta[r] + (nt + 2) * RTOL * y[r] * out.nu[ts][0]
                        assert abs(out.paid[r] - delta[r]) <= bound, (state_name, k, r, out.paid[r], delta[r])
                else:
                    assert out.status[r] == NC, out.status[r]
                    n_short += out.solver_status[r] == 0
                    check_not_filled(out, r)
        assert n_fill >= 15, (state_name, n_fill)
        print(f"{state_name}: {n_fill} filled, {n_short} converged below y")
    finally:
        m.close()


def certify_out_row(cert, order, out, r, y, j, i):
    """solve_certificate.certify of exact-out row r over its pools on its raw box, with the per-token
    tolerance its stop gives, and the header's gap bound."""
    ts, sl = row_slices(out, r)
    toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
    nu = np.ones(N)
    nu[toks - 1] = nu_r
    D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
    D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
    box = xo.box(N, i, j, y, RTOL)
    scale = y * nu_r[0]
    pgtol = float(np.max(out.merit[r] * scale / nu_r)) * (1 + 1e-9)
    res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
    z = box.lin[toks - 1] + psi
    on = (nu_r <= box.lower[toks - 1]) & (toks != j)
    box_terms = float(np.sum(np.maximum(z[on], 0.0) * (nu_r[on] - box.ref[toks - 1][on])))
    assert res["gap"] <= len(toks) * RTOL * scale + box_terms + res["allowance"], (res, box_terms)
    return res, box


def test_certificate_fresh_context_and_cfmm_solve(mk):
    p, Ai, m = mk
    rng = np.random.default_rng(27)
    allowed = mask(rng, 5)
    tin, tout, _, y, _ = out_rows(p, rng, allowed, 8)
    out = p.quote_subgraph_orders(tin, tout, y, allowed, kind=OUT)
    done = 0
    for r in np.flatnonzero(out.status == 0)[:4]:
        ts, sl = row_slices(out, r)
        pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
        q, order, cert = fresh(m, pools)
        try:
            nu = np.ones(N)
            nu[out.token[ts] - 1] = out.nu[ts]
            q.sweep(nu, materialize=True)
            D, L = q.trades()
            assert np.array_equal(D[order], out.leg_delta[sl]) and np.array_equal(L[order], out.leg_lambda[sl])
            res, box = certify_out_row(cert, order, out, r, y[r], int(tin[r]), int(tout[r]))
            # cfmm_solve on the fresh context with the same box (tokens outside the row sit at their
            # lower bound and hold no pool): the two dual values agree within the two gaps
            xs, _ = q.solve(**box.solve_args())
            Ds, Ls = q.trades()
            rs = sc.certify(cert, box, xs, Ds, Ls, check_stop=False)
            slack = (abs(res["gap"]) + res["allowance"] + abs(rs["gap"]) + rs["allowance"]
                     + rs["infeasibility"] * float(np.sum(xs)))
            assert abs(res["g50"] - rs["g50"]) <= slack, (res, rs)
            done += 1
        finally:
            q.close()
    assert done >= 3


def old_quote(p, tin, tout, amt, allowed):
    """cfmm_quote_subgraph_orders itself, through ctypes."""
    from cfmmrouter_b200.router import _dp, _ip
    tin, tout = np.ascontiguousarray(tin, np.int64), np.ascontiguousarray(tout, np.int64)
    amt, m8 = np.ascontiguousarray(amt, np.float64), np.ascontiguousarray(allowed, np.uint8)
    u8 = m8.ctypes.data_as(C.POINTER(C.c_uint8))
    return p._order_solve(len(tin), len(tin), cr._lib.SubgraphOut,
                          lambda size, out: p._lib.cfmm_quote_subgraph_orders(p._ctx, len(tin), _ip(tin), _ip(tout),
                                                                              _dp(amt), u8, None, C.byref(out)))


def test_exact_in_rows_unchanged(mk):
    p = mk[0]
    rng = np.random.default_rng(22)
    allowed = mask(rng, 5)
    tin, tout, amt = rows(rng, 9)
    ref = old_quote(p, tin, tout, amt, allowed)
    for kind in (None, 0, np.zeros(len(tin), np.uint8)):
        got = p.quote_subgraph_orders(tin, tout, amt, allowed, kind=kind)
        for x, z in zip(fields(ref), fields(got)):
            assert np.array_equal(x, z)
    # exact-in rows inside a mixed batch: the same bits
    kind = np.array([0, 1] * 4 + [0], np.uint8)
    mixed = p.quote_subgraph_orders(tin, tout, amt, allowed, kind=kind)
    for r in np.flatnonzero(kind == 0):
        assert mixed.received[r] == ref.received[r] and mixed.status[r] == ref.status[r]
        ts, sl = row_slices(ref, r)
        assert np.array_equal(mixed.nu[ts], ref.nu[ts]) and np.array_equal(mixed.leg_delta[sl], ref.leg_delta[sl])
    # executes: the old entry point and kind = 0 leave the same outputs and state
    m1, m2 = Market(), Market()
    try:
        a = m1.p.execute_subgraph_orders(tin, tout, amt, allowed)
        b = m2.p.execute_subgraph_orders(tin, tout, amt, allowed, kind=0)
        for x, z in zip(fields(a), fields(b)):
            assert np.array_equal(x, z)
        same_state(state(m1.p), state(m2.p))
    finally:
        m1.close()
        m2.close()


def test_mixed_batch_independent_and_no_state_change(mk):
    p = mk[0]
    rng = np.random.default_rng(23)
    allowed = mask(rng, 5)
    tin, tout, _, y, _ = out_rows(p, rng, allowed, 9)
    kind = np.array([1, 0, 1, 1, 0, 1, 0, 1, 1], np.uint8)
    before = state(p)
    a = p.quote_subgraph_orders(tin, tout, y, allowed, kind=kind)
    b = p.quote_subgraph_orders(tin, tout, y, allowed, kind=kind)
    for x, z in zip(fields(a), fields(b)):
        assert np.array_equal(x, z)
    same_state(before, state(p))
    for r in range(len(tin)):
        one = p.quote_subgraph_orders(tin[r:r + 1], tout[r:r + 1], y[r:r + 1], allowed, kind=int(kind[r]))
        ts, sl = row_slices(a, r)
        for x, z in zip(fields(one), [a.paid[r:r + 1], a.received[r:r + 1], a.status[r:r + 1],
                                      a.solver_status[r:r + 1], a.iterations[r:r + 1], a.fun_evals[r:r + 1],
                                      a.merit[r:r + 1], a.token[ts], a.nu[ts], a.psi[ts], a.leg_type[sl],
                                      a.leg_pool[sl], a.leg_delta[sl], a.leg_lambda[sl]]):
            assert np.array_equal(x, z), r
    assert np.any(a.status[kind == 1] == 0) and np.any(a.status[kind == 0] == 0)


def overbuy(out, r, y):
    """What the stop lets an exact-out row pay beyond the least payment for y: it receives up to
    y·(1 + 2·rtol), and its gap is at most |T|·rtol·y·ν_i, both at the marginal price ν_i (ν_j = 1).
    Near a pool's capacity that price is steep, so this can exceed rtol·paid."""
    ts, _ = row_slices(out, r)
    return (2 + len(out.token[ts])) * RTOL * y * out.nu[ts][0]


def test_paid_against_split_auto_routed_and_best_paths(mk):
    p = mk[0]
    rng = np.random.default_rng(24)
    ones = np.ones(12, np.uint8)
    # an empty mask: the pair's pools, as split orders' exact-out
    none = np.zeros(N, bool)
    tin, tout, _, y, _ = out_rows(p, rng, none, 12)
    out = p.quote_subgraph_orders(tin, tout, y, none, kind=OUT)
    paid, recv, _, st = p.quote_split_orders(tin, tout, ones, y)
    n_cmp = 0
    for r in range(len(tin)):
        if out.status[r] == 0 and st[r] == 0:
            n_cmp += 1
            tol = 3 * RTOL * max(abs(paid[r]), 1.0) + overbuy(out, r, y[r])
            assert abs(out.paid[r] - paid[r]) <= tol, (r, out.paid[r], paid[r], tol)
    assert n_cmp >= 6
    # a mask: auto-routed orders whose hubs lie in B, and best paths of 1..4 hops, pay at least as much
    # (a fifth of what the exact-in row received, so that one path can deliver it)
    allowed = mask(rng, 8)
    tin, tout, _, y, _ = out_rows(p, rng, allowed, 12)
    y = 0.2 * y
    out = p.quote_subgraph_orders(tin, tout, y, allowed, kind=OUT)
    off, flat, _, _ = p.choose_order_hubs(tin, tout, ones, y, 7, allowed)
    paid, _, _, st = p.quote_routed_orders(tin, tout, ones, y, off, flat)[:4]
    for r in range(len(tin)):
        if out.status[r] == 0 and st[r] == 0:
            tol = 3 * RTOL * max(abs(paid[r]), 1.0) + overbuy(out, r, y[r])
            assert out.paid[r] <= paid[r] + tol, (r, out.paid[r], paid[r], tol)
    n_cmp = 0
    for H in (1, 2, 3, 4):
        value, pst = p.find_order_paths(tin, tout, ones, y, H, allowed)[6:]
        for r in range(len(tin)):
            if out.status[r] == 0 and pst[r] == 0:
                n_cmp += 1
                tol = 3 * RTOL * max(value[r], 1.0) + overbuy(out, r, y[r])
                assert out.paid[r] <= value[r] + tol, (r, H, out.paid[r], value[r], tol)
    assert n_cmp >= 6


def test_execute_mixed_batch_equals_sequence_and_limits():
    rng = np.random.default_rng(25)
    allowed = mask(rng, 5)
    m1, m2, m3 = Market(), Market(), Market()
    p1, p2 = m1.p, m2.p
    try:
        tin, tout, delta, y, _ = out_rows(p1, rng, allowed, 6)
        kind = np.array([1, 0, 1, 1, 0, 1], np.uint8)
        amt = np.where(kind == 1, y, delta)
        batch = p1.execute_subgraph_orders(tin, tout, amt, allowed, kind=kind)
        seq = [p2.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], allowed, kind=int(kind[r]))
               for r in range(len(tin))]
        for r in range(len(tin)):
            ts, sl = row_slices(batch, r)
            assert batch.paid[r] == seq[r].paid[0] and batch.received[r] == seq[r].received[0]
            assert batch.status[r] == seq[r].status[0]
            assert np.array_equal(batch.leg_delta[sl], seq[r].leg_delta) and np.array_equal(batch.nu[ts], seq[r].nu)
        same_state(state(p1), state(p2))
        assert np.any(batch.status[kind == 1] == 0)
        # max-paid limits, on a fresh copy of the market: one ulp below the quote reverts and changes
        # nothing, an equal one fills
        p3 = m3.p
        qa = p3.quote_subgraph_orders(tin, tout, y, allowed, kind=OUT)
        r = int(np.flatnonzero(qa.status == 0)[0])
        a, b, yy = tin[r:r + 1], tout[r:r + 1], y[r:r + 1]
        before = state(p3)
        rev = p3.execute_subgraph_orders(a, b, yy, allowed, limit=np.nextafter(qa.paid[r:r + 1], -np.inf), kind=OUT)
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.paid[0] == 0.0 and not np.any(rev.leg_delta)
        same_state(before, state(p3))
        ok = p3.execute_subgraph_orders(a, b, yy, allowed, limit=qa.paid[r:r + 1], kind=OUT)
        assert ok.status[0] == 0 and ok.paid[0] == qa.paid[r] and ok.received[0] == qa.received[r]
        # +inf: no cap
        qq = p3.quote_subgraph_orders(a, b, yy, allowed, kind=OUT)
        inf = p3.execute_subgraph_orders(a, b, yy, allowed, limit=[np.inf], kind=OUT)
        assert inf.status[0] == qq.status[0] and inf.paid[0] == qq.paid[0]
    finally:
        m1.close()
        m2.close()
        m3.close()


def test_execute_transition_is_apply_trades_on_a_fresh_context():
    rng = np.random.default_rng(26)
    allowed = mask(rng, 5)
    m = Market()
    try:
        tin, tout, _, y, _ = out_rows(m.p, rng, allowed, 6)
        out = m.p.quote_subgraph_orders(tin, tout, y, allowed, kind=OUT)
        r = int(np.flatnonzero(out.status == 0)[0])
        ex = m.p.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], y[r:r + 1], allowed, kind=OUT)
        assert ex.status[0] == 0 and ex.paid[0] == out.paid[r]
        pools = list(zip(ex.leg_type.tolist(), ex.leg_pool.tolist()))
        q, order, _ = fresh(m, pools)
        try:
            nu = np.ones(N)
            nu[ex.token - 1] = ex.nu
            q.sweep(nu, materialize=True)
            q.apply_trades()
            sel = {t: sorted(i for tt, i in pools if tt == t) for t in (0, 1, 2)}
            for t in (0, 1, 2):
                if sel[t]:
                    got, _ = m.p.pool_state(t)
                    want, _ = q.pool_state(t)
                    assert np.array_equal(got[sel[t]], want), t
        finally:
            q.close()
    finally:
        m.close()


def row_capacity(p, Ai, out, r, i):
    """C_i of row r by the stated rule: per pool in the row's order, 0 unless active and holding i; a
    two-coin reserve of i; a UniV3 quote of a DBL_MAX tender of the other token; summed as the kernel."""
    _, sl = row_slices(out, r)
    terms = []
    for t, k in zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()):
        a = Ai[t][k]
        st, act = p.pool_state(t, k, 1)
        if not act[0] or i not in (a[0], a[1]):
            terms.append(0.0)
            continue
        side = 0 if a[0] == i else 1
        if t < 2:
            terms.append(float(st[0][side]))
        else:
            tender = np.zeros((1, 2))
            tender[0, 1 - side] = DBL_MAX
            terms.append(float(p.quote_swaps(t, [k], tender)[0, side]))
    return xo.capacity(terms), terms


def test_edge_rows(mk):
    p, Ai, m = mk
    lists = pair_lists(p)
    none = np.zeros(N, bool)
    # a pair with a UniV3 and a two-coin pool, both active: the capacity rule at its edge
    pair = next(ab for ab, l in lists.items()
                if any(t == 2 and a for t, _, a in l) and any(t < 2 and a for t, _, a in l))
    j, i = pair
    one = p.quote_subgraph_orders([j], [i], [1.0], none, kind=OUT)
    C_i, terms = row_capacity(p, m.Ai, one, 0, i)
    assert C_i > 0.0 and sum(x > 0 for x in terms) >= 2
    at = p.quote_subgraph_orders([j, j, j], [i, i, i], [C_i, 2 * C_i, np.nextafter(C_i, 0.0)], none, kind=OUT)
    assert at.status[0] == cr._lib.ORDER_UNREACHABLE and at.status[1] == cr._lib.ORDER_UNREACHABLE
    assert at.status[2] != cr._lib.ORDER_UNREACHABLE and at.status[2] in (0, NC)
    for r in range(3):
        if at.status[r] != 0:
            check_not_filled(at, r)
    # j ∉ T: a pair no pool holds, with an empty mask
    pair = next(ab for ab, l in lists.items() if not l)
    no = p.quote_subgraph_orders([pair[0]], [pair[1]], [1.0], none, kind=OUT)
    assert no.status[0] == cr._lib.ORDER_UNREACHABLE and no.solver_status[0] == -1
    # amount 0 fills with zeros and runs no solve
    z = p.quote_subgraph_orders([j], [i], [0.0], none, kind=OUT)
    assert z.status[0] == 0 and z.solver_status[0] == -1 and z.paid[0] == 0.0 and z.received[0] == 0.0


def test_unservable_row_is_not_converged():
    # i = 1 is deep in its pool with token 3, but 3 reaches j = 2 only through a thin pool: y < C_i,
    # and no payment in j buys y
    p = cr.DevicePools(4, device=0)
    try:
        R = np.array([[1000.0, 1000.0], [1e-6, 1e-6], [50.0, 60.0]])
        p.add_product(R, np.full(3, 0.997), np.array([[1, 3], [3, 2], [3, 4]], np.int64))
        p.finalize()
        allowed = np.array([0, 0, 1, 0], bool)
        before = p.pool_state(0)[0]
        out = p.quote_subgraph_orders([2], [1], [10.0], allowed, kind=OUT)
        assert out.token.tolist() == [1, 2, 3]
        assert out.status[0] == NC, (out.status[0], out.solver_status[0], out.merit[0])
        check_not_filled(out, 0)
        ex = p.execute_subgraph_orders([2], [1], [10.0], allowed, kind=OUT)
        assert ex.status[0] == NC
        assert np.array_equal(before, p.pool_state(0)[0])
    finally:
        p.close()


def test_rejections_change_nothing(mk):
    p = mk[0]
    from cfmmrouter_b200.router import _dp, _ip
    tin, tout, amt = np.array([1, 2], np.int64), np.array([3, 4], np.int64), np.array([1.0, 2.0])
    allowed = np.ones(N, np.uint8)
    u8 = C.POINTER(C.c_uint8)
    before = state(p)

    def call(kind, limit, a=amt):
        k = np.array(kind, np.uint8)
        lim = np.array(limit, np.float64)
        out = cr._lib.SubgraphOut()
        return p._lib.cfmm_execute_subgraph_swap_orders(p._ctx, 2, _ip(tin), _ip(tout), k.ctypes.data_as(u8),
                                                        _dp(a), _dp(lim), allowed.ctypes.data_as(u8), None,
                                                        C.byref(out))

    for kind, limit in (([0, 2], [1.0, 1.0]), ([1, 7], [1.0, 1.0]), ([0, 1], [np.inf, 1.0]),
                        ([1, 1], [1.0, np.nan]), ([1, 0], [-1.0, 1.0]), ([0, 0], [1.0, np.nan])):
        assert call(kind, limit) == cr._lib.CFMM_ERR_INVALID, (kind, limit)
        same_state(before, state(p))
    k = np.array([1, 2], np.uint8)
    out = cr._lib.SubgraphOut()
    assert p._lib.cfmm_quote_subgraph_swap_orders(p._ctx, 2, _ip(tin), _ip(tout), k.ctypes.data_as(u8), _dp(amt),
                                                  allowed.ctypes.data_as(u8), None,
                                                  C.byref(out)) == cr._lib.CFMM_ERR_INVALID
    # exact-out rows take +inf as the maximum paid (amount 0 rows: nothing trades)
    assert call([1, 1], [np.inf, np.inf], np.zeros(2)) == cr._lib.CFMM_OK
    same_state(before, state(p))
    with pytest.raises(ValueError):
        p.execute_subgraph_orders(tin, tout, amt, allowed, limit=[np.inf, 1.0], kind=0)


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 21)
    try:
        n = 12
        allowed = np.zeros(n, bool)
        allowed[:6] = True
        tin, tout, amt = np.array([7, 8, 9, 10]), np.array([11, 12, 7, 8]), np.array([5.0, 20.0, 50.0, 1.0])
        paid, recv, st, det = r.quote_subgraph_orders(tin, tout, amt, allowed, kind=1)
        reach = st != cr._lib.ORDER_UNREACHABLE
        assert np.any(reach) and np.all(np.isin(st[reach], (0, NC))) and np.any(st == 0)
        assert np.all(recv[st == 0] >= amt[st == 0])
        with pytest.raises(ValueError):
            r.quote_subgraph_orders(tin, tout, amt, allowed, kind=[1, 0])
        paid2, recv2, st2, det2 = r.execute_subgraph_orders(tin, tout, amt, allowed, limits=np.full(len(tin), np.inf),
                                                            kind=1)
        assert np.any(st2 == 0) and not np.any(recv2[st2 != 0])
        for k in np.flatnonzero(st2 == 0):
            sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
            for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
                dev, _ = r._pools.pool_state(int(t), int(i), 1)
                c = r.cfmms[r._type_lists[int(t)][int(i)]]
                assert np.array_equal(np.asarray(c.R), dev[0])
    finally:
        r.close() if hasattr(r, "close") else None
