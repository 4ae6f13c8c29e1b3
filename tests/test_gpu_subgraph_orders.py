"""cfmm_quote_subgraph_orders / cfmm_execute_subgraph_orders (include/cfmm_b200.h) on the device.

A market of all three pool types with appended and retired pools, also with ProductTwoCoin pools
stored exchanged (orient_by_degree = 1), after cfmm_compact, after a UniV3 liquidity change and
after a retire that follows the adjacency build.  On every state: each row's token set and pool list
against an enumeration over cfmm_pair_pools, its legs bit for bit against a materialising cfmm_sweep
at the reported ν, its Ψ, paid and received against the stated warp-tree sums, and every reachable
row with an amount filling under the default options with the header's bounds.  On the plain market:
every filled row passes the 50-digit certificate (solve_certificate) at its m_r; a fresh context
holding only the row's pools gives the legs (cfmm_sweep) and the execute's new state
(cfmm_apply_trades) bit for bit, and cfmm_solve's dual value within the two gaps; B = ∅ agrees with
split orders, hubs without pools between them with routed orders, and the received is at least the
best path's and the auto-routed orders'.  Quotes are deterministic, batch-independent and change no
state; a batch execute equals one-row executes in sequence (one row per launch with a mask, several
with B = ∅); limits revert (an equal one fills); rows that do not converge change nothing; bad
arguments are rejected; and the Router refreshes the pool objects it traded with."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import order_certificate as oc
import solve_certificate as sc
import subgraph_oracle as so

pytestmark = pytest.mark.gpu

N = 20
M = {0: 150, 1: 60, 2: 40}
APPENDED = 15
RTOL = 1e-4  # the default
RETIRED = {(0, 3), (0, 4), (2, 5)}
STATES = ("plain", "orient", "compact", "liquidity", "retire_after_adjacency")


class Market:
    """The device context and its pools' construction arrays (ProductTwoCoin: main then appended)."""

    def __init__(self, state="plain"):
        self.p = p = cr.DevicePools(N, device=0)
        if state == "orient":
            p.set_option("orient_by_degree", 1)
        Rp, gp, Ap = synth.product_pools(M[0], N, seed=11)
        Rg, gg, Ag, wg = synth.geomean_pools(M[1], N, seed=12)
        self.u3 = synth.univ3_pools(M[2], N, seed=13)
        p.add_product(Rp, gp, Ap)
        p.add_geomean(Rg, gg, Ag, wg)
        p.add_univ3(*self.u3)
        p.finalize()
        Ra, ga, Aa = synth.product_pools(APPENDED, N, seed=14)
        p.append_product(Ra, ga, Aa)
        self.prod = (np.concatenate([Rp, Ra]), np.concatenate([gp, ga]), np.concatenate([Ap, Aa]))
        self.geo = (Rg, gg, Ag, wg)
        self.Ai = {0: self.prod[2], 1: Ag, 2: self.u3[2]}
        retired = set(RETIRED)
        if state == "retire_after_adjacency":
            p.quote_subgraph_orders([1], [2], [1.0], np.ones(N, bool))   # builds the adjacency
            retired.add((1, 7))
        for t, i in sorted(retired):
            p.set_active(t, i, [0])
        self.retired = retired
        if state == "compact":
            p.compact()
        if state == "liquidity":
            cp = self.u3[0]
            p.modify_univ3_liquidity([0, 1, 9], cp[[0, 1, 9]] * 0.8, cp[[0, 1, 9]] * 1.3, [50.0, 80.0, 120.0])

    def close(self):
        self.p.close()


def global_index(t, i):
    """cfmm_num_pools numbering: the main sets in type order, then the appended ProductTwoCoin pools."""
    if t == 0:
        return i if i < M[0] else M[0] + M[1] + M[2] + (i - M[0])
    return (M[0] if t >= 1 else 0) + (M[1] if t == 2 else 0) + i


def rows(rng, q):
    tin = rng.integers(1, N + 1, size=q)
    tout = (tin + rng.integers(1, N, size=q) - 1) % N + 1
    return tin.astype(np.int64), tout.astype(np.int64), rng.uniform(1.0, 20.0, size=q)


def mask(rng, k):
    m = np.zeros(N, bool)
    m[rng.choice(N, size=k, replace=False)] = True
    return m


@pytest.fixture(scope="module")
def mk():
    m = Market()
    yield m.p, m.Ai, m
    m.close()


def pair_lists(p):
    a = [x for x in range(1, N + 1) for y in range(x + 1, N + 1)]
    b = [y for x in range(1, N + 1) for y in range(x + 1, N + 1)]
    off, typ, idx, act = p.pair_pools(a, b)
    return {(a[c], b[c]): [(int(typ[e]), int(idx[e]), bool(act[e])) for e in range(off[c], off[c + 1])]
            for c in range(len(a))}


def row_slices(out, r):
    return slice(out.tok_off[r], out.tok_off[r + 1]), slice(out.leg_off[r], out.leg_off[r + 1])


def check_row(p, Ai, out, r, amt):
    """Legs against a materialising sweep, the stated sums, and the stop's bounds, for filled row r."""
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
    d, vj = amt, nu[1]
    if vj > so.SQRT_EPS:
        assert abs(out.paid[r] - d) <= 1.01 * RTOL * d
    assert np.all(psi[2:] >= -1.01 * RTOL * d * vj / nu[2:])


@pytest.mark.parametrize("state", STATES)
def test_lists_legs_sums_and_default_fill_on_every_state(state):
    m = Market(state)
    try:
        p = m.p
        rng = np.random.default_rng(1)
        lists = pair_lists(p)
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            tin, tout, amt = rows(rng, 10)
            amt[4] = 0.0
            out = p.quote_subgraph_orders(tin, tout, amt, allowed)
            for r in range(len(tin)):
                T, pools = so.row_subgraph(lists, int(tin[r]), int(tout[r]), allowed)
                ts, sl = row_slices(out, r)
                assert out.token[ts].tolist() == T, (r, out.token[ts], T)
                want = sorted([(t, i) for t, i in pools], key=lambda h: global_index(*h))
                assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == want
                if amt[r] == 0.0:
                    assert out.status[r] == 0 and out.received[r] == 0.0 and out.solver_status[r] == -1
                elif int(tin[r]) not in T:
                    assert out.status[r] == cr._lib.ORDER_UNREACHABLE
                    assert out.received[r] == 0.0 and not np.any(out.leg_delta[sl])
                else:
                    # the default rtol is met on every reachable row
                    assert out.status[r] == 0, (state, k, r, out.solver_status[r], out.merit[r])
                    check_row(p, m.Ai, out, r, amt[r])
    finally:
        m.close()


def test_empty_mask_is_split_orders_and_paths_are_a_floor(mk):
    p = mk[0]
    rng = np.random.default_rng(3)
    tin, tout, amt = rows(rng, 12)
    none = np.zeros(N, bool)
    out = p.quote_subgraph_orders(tin, tout, amt, none)
    paid, recv, _, st = p.quote_split_orders(tin, tout, np.zeros(len(tin), np.uint8), amt)
    for r in range(len(tin)):
        assert out.status[r] == st[r]
        if out.status[r] == 0:
            assert abs(out.received[r] - recv[r]) <= 3 * RTOL * max(recv[r], 1.0), (r, out.received[r], recv[r])
    allowed = mask(rng, 7)
    out = p.quote_subgraph_orders(tin, tout, amt, allowed)
    for H in (1, 2, 3, 4):
        value, pst = p.find_order_paths(tin, tout, np.zeros(len(tin), np.uint8), amt, H, allowed)[6:]
        for r in range(len(tin)):
            assert out.status[r] in (0, 2)
            if out.status[r] == 0 and pst[r] == 0:
                assert out.received[r] >= value[r] * (1 - 3 * RTOL), (r, H, out.received[r], value[r])  # within the gap


def state(p):
    return [p.pool_state(t) for t in (0, 1, 2)]


def same_state(a, b):
    for (x, xa), (y, ya) in zip(a, b):
        assert np.array_equal(x, y) and np.array_equal(xa, ya)


def fields(o):
    return [o.paid, o.received, o.status, o.solver_status, o.iterations, o.fun_evals, o.merit, o.token, o.nu, o.psi,
            o.leg_type, o.leg_pool, o.leg_delta, o.leg_lambda]


def test_deterministic_batch_independent_no_state_change(mk):
    p = mk[0]
    rng = np.random.default_rng(4)
    allowed = mask(rng, 5)
    tin, tout, amt = rows(rng, 9)
    before = state(p)
    a = p.quote_subgraph_orders(tin, tout, amt, allowed)
    b = p.quote_subgraph_orders(tin, tout, amt, allowed)
    for x, y in zip(fields(a), fields(b)):
        assert np.array_equal(x, y)
    same_state(before, state(p))
    for r in (0, 4, 8):
        one = p.quote_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], allowed)
        sl = slice(a.leg_off[r], a.leg_off[r + 1])
        assert one.received[0] == a.received[r] and one.paid[0] == a.paid[r] and one.status[0] == a.status[r]
        assert np.array_equal(one.leg_delta, a.leg_delta[sl]) and np.array_equal(one.nu,
                                                                                 a.nu[a.tok_off[r]:a.tok_off[r + 1]])


def test_execute_batch_equals_sequence_and_limits():
    rng = np.random.default_rng(5)
    allowed = mask(rng, 5)
    tin, tout, amt = rows(rng, 6)
    m1, m2 = Market(), Market()
    p1, p2 = m1.p, m2.p
    try:
        batch = p1.execute_subgraph_orders(tin, tout, amt, allowed)
        seq = [p2.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], allowed) for r in range(len(tin))]
        for r in range(len(tin)):
            assert batch.received[r] == seq[r].received[0] and batch.status[r] == seq[r].status[0]
            sl = slice(batch.leg_off[r], batch.leg_off[r + 1])
            assert np.array_equal(batch.leg_delta[sl], seq[r].leg_delta)
        same_state(state(p1), state(p2))
        assert np.all(batch.status[batch.status != cr._lib.ORDER_UNREACHABLE] == 0) and np.any(batch.status == 0)
        # limits: an equal limit fills, a larger one reverts and changes nothing
        q = p1.quote_subgraph_orders(tin[:1], tout[:1], amt[:1], allowed)
        if q.status[0] == 0:
            before = state(p1)
            lim = np.nextafter(q.received, np.inf)
            rev = p1.execute_subgraph_orders(tin[:1], tout[:1], amt[:1], allowed, limit=lim)
            assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.received[0] == 0.0
            same_state(before, state(p1))
            ok = p1.execute_subgraph_orders(tin[:1], tout[:1], amt[:1], allowed, limit=q.received)
            assert ok.status[0] == 0 and ok.received[0] == q.received[0]
        # max_iter = 1: not converged, nothing changes
        before = state(p1)
        nc = p1.execute_subgraph_orders(tin, tout, amt, allowed, opts={"max_iter": 1, "rtol": 1e-12})
        reach = nc.status != cr._lib.ORDER_UNREACHABLE
        assert np.all(nc.status[reach] == cr._lib.ORDER_NOT_CONVERGED)
        assert not np.any(nc.leg_delta) and not np.any(nc.received)
        same_state(before, state(p1))
    finally:
        m1.close()
        m2.close()


def test_rejections(mk):
    p = mk[0]
    tin, tout, amt = np.array([1, 2], np.int64), np.array([3, 4], np.int64), np.array([1.0, 2.0])
    allowed = np.ones(N, bool)
    lib, u8 = p._lib, C.POINTER(C.c_uint8)
    ip, dp = C.POINTER(C.c_int64), C.POINTER(C.c_double)
    out = cr._lib.SubgraphOut()
    rc = lib.cfmm_quote_subgraph_orders(p._ctx, 2, tin.ctypes.data_as(ip), tout.ctypes.data_as(ip),
                                        amt.ctypes.data_as(dp), None, None, C.byref(out))
    assert rc == cr._lib.CFMM_ERR_INVALID
    for bad in ({"rtol": 0.0}, {"rtol": float("nan")}, {"max_iter": 0}, {"max_fun": 0}, {"factr": -1.0}):
        with pytest.raises(cr.CFMMError):
            p.quote_subgraph_orders(tin, tout, amt, allowed, opts=bad)
    for lim in (float("nan"), -1.0, float("inf")):
        with pytest.raises(cr.CFMMError):
            p.execute_subgraph_orders(tin, tout, amt, allowed, limit=[1.0, lim])
    with pytest.raises(cr.CFMMError):
        p.quote_subgraph_orders(tin, tin, amt, allowed)
    with pytest.raises(cr.CFMMError):
        p.quote_subgraph_orders(tin, tout, [1.0, float("nan")], allowed)
    big = cr.DevicePools(300, device=0)
    try:
        R, g, A = synth.product_pools(50, 300, seed=3)
        big.add_product(R, g, A)
        big.finalize()
        with pytest.raises(cr.CFMMError, match="row 0"):
            big.quote_subgraph_orders([1], [2], [1.0], np.ones(300, bool))
        n0 = big.launch_count
        r = big.quote_subgraph_orders([1], [2], [1.0], np.r_[np.ones(200, bool), np.zeros(100, bool)])
        assert r.status[0] in (0, 2)
        assert big.launch_count > n0
    finally:
        big.close()


# ---- a fresh context holding only a row's pools, and the 50-digit certificate --------------------
def fresh(m, pools):
    """A context of N tokens holding only `pools` ((type, index) of m) at m's construction state, retired
    ones retired.  Returns (context, the fresh global index of each pool, certificate pools in the
    fresh global order)."""
    sel = {t: sorted(i for tt, i in pools if tt == t) for t in (0, 1, 2)}
    q = cr.DevicePools(N, device=0)
    cert = []
    if sel[0]:
        R, g, A = (x[sel[0]] for x in m.prod)
        q.add_product(R, g, A)
        cert += [oc.product(R[k], g[k], A[k], active=(0, i) not in m.retired) for k, i in enumerate(sel[0])]
    if sel[1]:
        R, g, A, w = (x[sel[1]] for x in m.geo)
        q.add_geomean(R, g, A, w)
        cert += [oc.geomean(R[k], g[k], w[k], A[k], active=(1, i) not in m.retired) for k, i in enumerate(sel[1])]
    if sel[2]:
        cp, gu, Au, off, lt, lq = m.u3
        idx = sel[2]
        lens = np.array([off[i + 1] - off[i] for i in idx], np.int64)
        off2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        lt2 = np.concatenate([lt[off[i]:off[i + 1]] for i in idx])
        lq2 = np.concatenate([lq[off[i]:off[i + 1]] for i in idx])
        q.add_univ3(cp[idx], gu[idx], Au[idx], off2, lt2, lq2)
        cert += [oc.univ3(cp[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], gu[i], Au[i], active=(2, i) not in m.retired)
                 for i in idx]
    q.finalize()
    base = {0: 0, 1: len(sel[0]), 2: len(sel[0]) + len(sel[1])}
    for t in (0, 1, 2):
        for k, i in enumerate(sel[t]):
            if (t, i) in m.retired:
                q.set_active(t, k, [0])
    where = {(t, i): base[t] + k for t in (0, 1, 2) for k, i in enumerate(sel[t])}
    return q, [where[h] for h in pools], cert


def certify_row(cert, order, out, r, amt, j, i):
    """solve_certificate.certify of row r over its pools (cert in fresh order, order: each listed pool's
    fresh index) under Swap's box, with the per-token tolerance the stop m_r <= rtol gives."""
    ts, sl = row_slices(out, r)
    toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
    nu = np.ones(N)
    nu[toks - 1] = nu_r
    D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
    D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
    lin = np.zeros(N)
    lin[j - 1] = amt
    box = sc.basket(i, lin)
    scale = amt * nu_r[1]
    pgtol = float(np.max(out.merit[r] * scale / nu_r)) * (1 + 1e-9)
    res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
    # the header's gap bound: |T|·rtol·δ·ν_j plus the box terms of the tokens on their bounds
    z = lin[toks - 1] + psi
    on = nu_r <= box.lower[toks - 1]
    box_terms = float(np.sum(np.maximum(z[on], 0.0) * (nu_r[on] - box.ref[toks - 1][on])))
    assert res["gap"] <= len(toks) * RTOL * scale + box_terms + res["allowance"], (res, box_terms)
    return res


def test_certificate_fresh_context_and_cfmm_solve(mk):
    p, Ai, m = mk
    rng = np.random.default_rng(7)
    allowed = mask(rng, 5)
    tin, tout, amt = rows(rng, 8)
    out = p.quote_subgraph_orders(tin, tout, amt, allowed)
    done = 0
    for r in np.flatnonzero(out.status == 0)[:4]:
        ts, sl = row_slices(out, r)
        pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
        q, order, cert = fresh(m, pools)
        try:
            # legs: a materialising sweep of the fresh context at the reported ν
            nu = np.ones(N)
            nu[out.token[ts] - 1] = out.nu[ts]
            q.sweep(nu, materialize=True)
            D, L = q.trades()
            assert np.array_equal(D[order], out.leg_delta[sl]) and np.array_equal(L[order], out.leg_lambda[sl])
            res = certify_row(cert, order, out, r, amt[r], int(tin[r]), int(tout[r]))
            # cfmm_solve on the fresh context with the same box: the two dual values within the gaps
            lin = np.zeros(N)
            lin[tin[r] - 1] = amt[r]
            box = sc.basket(int(tout[r]), lin)
            xs, info = q.solve(lower=box.lower, lin=box.lin)
            Ds, Ls = q.trades()
            rs = sc.certify(cert, box, xs, Ds, Ls, check_stop=False)
            # both are dual values: each exceeds the optimum by at most its gap (taken in magnitude, as
            # cfmm_solve's trades may be slightly infeasible), plus the rounding allowances
            slack = (abs(res["gap"]) + res["allowance"] + abs(rs["gap"]) + rs["allowance"]
                     + rs["infeasibility"] * float(np.sum(xs)))
            assert abs(res["g50"] - rs["g50"]) <= slack, (res, rs)
            done += 1
        finally:
            q.close()
    assert done >= 3


def test_execute_transition_is_apply_trades_on_a_fresh_context():
    rng = np.random.default_rng(8)
    allowed = mask(rng, 5)
    tin, tout, amt = rows(rng, 6)
    m = Market()
    try:
        out = m.p.quote_subgraph_orders(tin, tout, amt, allowed)
        r = int(np.flatnonzero(out.status == 0)[0])
        ex = m.p.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], allowed)
        assert ex.status[0] == 0 and ex.received[0] == out.received[r]
        pools = list(zip(ex.leg_type.tolist(), ex.leg_pool.tolist()))
        q, order, _ = fresh(m, pools)
        try:
            nu = np.ones(N)
            nu[ex.token - 1] = ex.nu
            q.sweep(nu, materialize=True)
            q.apply_trades()
            sel = {t: sorted(i for tt, i in pools if tt == t) for t in (0, 1, 2)}
            for t in (0, 1, 2):
                if not sel[t]:
                    continue
                got, _ = m.p.pool_state(t)
                want, _ = q.pool_state(t)
                assert np.array_equal(got[sel[t]], want), t
        finally:
            q.close()
    finally:
        m.close()


def test_routed_orders_without_hub_pools_and_auto_routed_floor(mk):
    p, _, _ = mk
    lists = pair_lists(p)
    tin, tout, hubs = [], [], []
    for j in range(1, N + 1):
        for i in range(1, N + 1):
            if i == j or not lists[(min(i, j), max(i, j))]:
                continue
            for h1 in range(1, N + 1):
                for h2 in range(h1 + 1, N + 1):
                    if {h1, h2} & {i, j} or lists[(h1, h2)]:
                        continue
                    tin.append(j)
                    tout.append(i)
                    hubs.append((h1, h2))
                    break
                if len(tin) and tin[-1] == j and tout[-1] == i:
                    break
    rows_ = np.random.default_rng(9).choice(len(tin), size=8, replace=False)
    n_cmp = 0
    for r in rows_:
        allowed = np.zeros(N, bool)
        allowed[np.array(hubs[r]) - 1] = True
        a = np.array([tin[r]], np.int64)
        b = np.array([tout[r]], np.int64)
        out = p.quote_subgraph_orders(a, b, [5.0], allowed)
        _, recv, _, st = p.quote_routed_orders(a, b, np.zeros(1, np.uint8), [5.0], np.array([0, 2], np.int64),
                                               np.array(hubs[r], np.int64))[:4]
        assert st[0] == 0 and out.status[0] in (0, cr._lib.ORDER_NOT_CONVERGED)
        if out.status[0] == 0:
            n_cmp += 1
            assert abs(out.received[0] - recv[0]) <= 3 * RTOL * max(recv[0], 1.0), (out.received[0], recv[0])
        else:
            assert out.received[0] == 0.0
    assert n_cmp >= 4
    # auto-routed orders whose hubs lie in B are a floor
    rng = np.random.default_rng(10)
    allowed = mask(rng, 8)
    a, b, amt = rows(rng, 10)
    kind = np.zeros(len(a), np.uint8)
    off, flat, _, _ = p.choose_order_hubs(a, b, kind, amt, 7, allowed)
    _, recv, _, st = p.quote_routed_orders(a, b, kind, amt, off, flat)[:4]
    out = p.quote_subgraph_orders(a, b, amt, allowed)
    for r in range(len(a)):
        if out.status[r] == 0 and st[r] == 0:
            assert out.received[r] >= recv[r] * (1 - 3 * RTOL), (r, out.received[r], recv[r])


def test_empty_mask_execute_runs_disjoint_rows_together():
    tin = np.array([1, 3, 1, 5, 3, 7], np.int64)
    tout = np.array([2, 4, 2, 6, 4, 8], np.int64)
    amt = np.array([3.0, 4.0, 5.0, 2.0, 1.0, 6.0])
    none = np.zeros(N, bool)
    m1, m2 = Market(), Market()
    try:
        n0 = m1.p.launch_count
        batch = m1.p.execute_subgraph_orders(tin, tout, amt, none)
        n_batch = m1.p.launch_count - n0
        n0 = m2.p.launch_count
        seq = [m2.p.execute_subgraph_orders(tin[r:r + 1], tout[r:r + 1], amt[r:r + 1], none) for r in range(len(tin))]
        n_seq = m2.p.launch_count - n0
        for r in range(len(tin)):
            assert batch.received[r] == seq[r].received[0] and batch.status[r] == seq[r].status[0]
            ts, sl = row_slices(batch, r)
            assert np.array_equal(batch.leg_delta[sl], seq[r].leg_delta)
            assert np.array_equal(batch.nu[ts], seq[r].nu)
        same_state(state(m1.p), state(m2.p))
        assert n_batch < n_seq   # three levels: {1, 2} twice, {3, 4} twice; 5-6 and 7-8 share level 1
    finally:
        m1.close()
        m2.close()


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 21)
    try:
        n = r.n_tokens if hasattr(r, "n_tokens") else 12
        allowed = np.zeros(n, bool)
        allowed[:6] = True
        tin, tout, amt = np.array([7, 8, 9, 10]), np.array([11, 12, 7, 8]), np.array([5.0, 20.0, 50.0, 1.0])
        paid, recv, st, det = r.quote_subgraph_orders(tin, tout, amt, allowed)
        reach = st != cr._lib.ORDER_UNREACHABLE
        assert np.all(st[reach] == 0) and np.any(reach)
        with pytest.raises(ValueError):
            r.quote_subgraph_orders(tin, tout, amt, None)
        paid2, recv2, st2, det2 = r.execute_subgraph_orders(tin, tout, amt, allowed, limits=np.zeros(len(tin)))
        # each row is re-solved on the state the earlier rows left: a row may end NOT_CONVERGED there
        # (the default rtol is not a guarantee, DESIGN §4.5), and then trades nothing
        assert np.all(np.isin(st2[reach], (0, cr._lib.ORDER_NOT_CONVERGED))) and np.any(st2 == 0)
        assert not np.any(recv2[st2 != 0]) and not np.any(det2.leg_delta[np.concatenate(
            [np.arange(det2.leg_off[k], det2.leg_off[k + 1]) for k in np.flatnonzero(st2 != 0)] + [[]]).astype(int)])
        for k in np.flatnonzero(st2 == 0):
            sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
            for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
                dev, _ = r._pools.pool_state(int(t), int(i), 1)
                c = r.cfmms[r._type_lists[int(t)][int(i)]]
                assert np.array_equal(np.asarray(c.R), dev[0])
    finally:
        r.close() if hasattr(r, "close") else None
