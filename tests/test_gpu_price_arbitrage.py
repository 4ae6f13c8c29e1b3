"""cfmm_quote_price_arbitrage / cfmm_execute_price_arbitrage (include/cfmm_b200.h) on the device.

test/arb.jl restated as rows (the simple market and the 100-pool, 10-token random market): rows fill
with Ψ >= −1e-4 (on the random market valued at c, see ARB_JL_OPTS), ν >= c + 1e-8 − 1e-4 and every
traded pool keeping φ.  On the five markets of
test_gpu_subgraph_orders: each row lists every pool among T in insertion order, its legs equal a
materialising cfmm_sweep at its ν bit for bit, its Ψ the warp-tree sums and its profit the local-order
sum, and filled rows meet the stop's promise; on the plain market they pass the 50-digit certificate.
With every token priced, a row agrees with cfmm_solve and the host route() within their certified gaps.
An executed row leaves no arbitrage; a market without arbitrage fills with zeros after one evaluation;
a batch execute equals single-row executes in sequence and rows on disjoint price subsets share a launch;
a price of 0 is the row without that token, bit for bit; min_profit reverts (an equal one fills);
quotes and rejections change nothing; and the Router refreshes the pool objects it traded with."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import order_certificate as oc
import price_arb_oracle as pa
import solve_certificate as sc
import subgraph_oracle as so
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, fresh, global_index, mask, pair_lists, row_slices,
                                      same_state, state)

pytestmark = pytest.mark.gpu

NC = cr._lib.ORDER_NOT_CONVERGED
SQRT_EPS = float(np.sqrt(np.finfo(float).eps))


def product_context(n, spec):
    """A context holding ProductTwoCoin pools spec = [(R, γ, Ai)]."""
    p = cr.DevicePools(n, device=0)
    p.add_product(np.array([s[0] for s in spec], float), np.array([s[1] for s in spec], float),
                  np.array([s[2] for s in spec], np.int64))
    p.finalize()
    return p


def fields(o):
    return [o.profit, o.status, o.solver_status, o.iterations, o.fun_evals, o.merit, o.token, o.nu, o.psi,
            o.leg_type, o.leg_pool, o.leg_delta, o.leg_lambda]


def same(a, b):
    for x, y in zip(fields(a), fields(b)):
        assert np.array_equal(x, y)


def row_prices(out, r, allowed, price_row):
    """The row's prices in local order (T ascending)."""
    A = (np.flatnonzero(allowed) + 1).tolist()
    ts, _ = row_slices(out, r)
    return np.array([price_row[A.index(int(t))] for t in out.token[ts]])


def check_filled(out, r, c):
    """The fill promise of filled row r (c: its prices in local order).  Returns g ≈ νᵀΨ."""
    ts, _ = row_slices(out, r)
    nu, psi = out.nu[ts], out.psi[ts]
    assert out.status[r] == 0 and out.solver_status[r] == 0 and out.merit[r] <= RTOL
    assert np.all(nu >= pa.box(c))
    assert out.profit[r] == pa.profit(c, psi)
    g = float(nu @ psi)
    if out.merit[r] > 0.0:
        assert pa.merit(nu, psi, pa.box(c), g) <= RTOL * 1.01
        assert np.all(psi >= -RTOL * g / nu * 1.01 - 1e-12)
    return g


def check_lists_legs_sums(p, Ai, lists, out, r, allowed, price_row):
    T, pools = pa.row_order(lists, allowed, price_row)
    ts, sl = row_slices(out, r)
    assert out.token[ts].tolist() == T, (r, out.token[ts], T)
    assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == sorted(
        pools, key=lambda h: global_index(*h))
    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
    v = np.ones(N)
    v[toks - 1] = nu
    p.sweep(v, materialize=True)
    D, L = p.trades()
    g = np.array([global_index(int(t), int(i)) for t, i in zip(out.leg_type[sl], out.leg_pool[sl])], np.int64)
    if out.status[r] == 0:
        assert np.array_equal(D[g], out.leg_delta[sl]) and np.array_equal(L[g], out.leg_lambda[sl])
        A = so.ingest_tokens(Ai, out.leg_type[sl], out.leg_pool[sl])
        assert np.array_equal(so.warp_psi(A, out.leg_delta[sl], out.leg_lambda[sl], toks), psi)
    else:
        assert out.status[r] == NC and out.solver_status[r] != 0 and out.profit[r] == 0.0
        assert not np.any(out.leg_delta[sl]) and not np.any(out.leg_lambda[sl])


def prices(rng, q, nA, zero=0.2):
    c = rng.uniform(0.5, 2.0, size=(q, nA))
    c[rng.random((q, nA)) < zero] = 0.0
    c[np.arange(q), rng.integers(0, nA, q)] = rng.uniform(0.5, 2.0, q)  # every row has a price
    return c


# ---- test/arb.jl as rows ----------------------------------------------------------------------
# The random market's rows make profits near 1e4 at prices down to 1e-2, and the per-row solver's m_r
# floor there is near 1e-10 (its factr stop fires first below that).  At rtol = 1e-8 the promise
# Ψ_t >= −rtol·g/ν_t leaves up to a few 1e-4 tokens short, so test/arb.jl's 1e-4 is applied to the net
# valued at c (c_t·Ψ_t) there, and to Ψ itself on the simple market.
ARB_JL_OPTS = {"rtol": 1e-8}


def check_arb_jl(out, r, c, spec, valued=False):
    ts, sl = row_slices(out, r)
    assert out.status[r] == 0, (out.solver_status[r], out.merit[r])
    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
    assert np.all((c[toks - 1] * psi if valued else psi) >= -1e-4) and np.all(nu >= c[toks - 1] + 1e-8 - 1e-4)
    for t, i, D, L in zip(out.leg_type[sl], out.leg_pool[sl], out.leg_delta[sl], out.leg_lambda[sl]):
        R, gam, Ai = spec[int(i)]
        assert t == 0 and np.all(D >= -1e-4) and np.all(L >= -1e-4)
        pool = cr.ProductTwoCoin(R, gam, Ai)
        assert pool.phi(np.asarray(R) + gam * D - L) >= pool.phi() - SQRT_EPS
    assert out.profit[r] == pa.profit(c[toks - 1], psi)


def test_arb_jl_markets():
    spec = [([100.0, 100.0], 1.0, [1, 2]), ([1.0, 2.0], 1.0, [1, 2])]
    p = product_context(2, spec)
    try:
        out = p.quote_price_arbitrage([[1.0, 1.0]], np.ones(2, bool))
        check_arb_jl(out, 0, np.ones(2), spec)
        assert out.profit[0] > 0.0
    finally:
        p.close()
    rng = np.random.default_rng(1234)
    n = 10
    spec = [(1000 * rng.random(2), fee, rng.choice(np.arange(1, n + 1), size=2, replace=False))
            for fee in [1.0] * 50 + [0.997] * 50]
    p = product_context(n, spec)
    try:
        c = rng.random((4, n)) + 1e-3
        out = p.quote_price_arbitrage(c, np.ones(n, bool), opts=ARB_JL_OPTS)
        for r in range(4):
            check_arb_jl(out, r, c[r], spec, valued=True)
    finally:
        p.close()


# ---- the five market states ---------------------------------------------------------------------
@pytest.mark.parametrize("state_", STATES)
def test_lists_legs_sums_and_fill_on_every_state(state_):
    m = Market(state_)
    try:
        p = m.p
        rng = np.random.default_rng(41)
        lists = pair_lists(p)
        n_filled = n_rows = 0
        for k in (2, 5, 8, 12, 20):
            allowed = mask(rng, k)
            c = prices(rng, 6, k)
            out = p.quote_price_arbitrage(c, allowed)
            for r in range(len(c)):
                check_lists_legs_sums(p, m.Ai, lists, out, r, allowed, c[r])
                n_rows += 1
                if out.status[r] == 0:
                    n_filled += 1
                    check_filled(out, r, row_prices(out, r, allowed, c[r]))
        assert n_filled >= n_rows // 2, (n_filled, n_rows)
    finally:
        m.close()


def test_certificate_on_the_plain_market():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(42)
        done = 0
        for k in (4, 8):
            allowed = mask(rng, k)
            c = prices(rng, 4, k)
            out = p.quote_price_arbitrage(c, allowed)
            for r in np.flatnonzero(out.status == 0)[:3]:
                ts, sl = row_slices(out, r)
                if sl.stop == sl.start:
                    continue
                pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
                q, order, cert = fresh(m, pools)
                q.close()
                cl = row_prices(out, r, allowed, c[r])
                D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
                D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
                g = max(float(out.nu[ts] @ out.psi[ts]), out.profit[r]) * 1.01
                res = pa.certify(cert, N, out.token[ts], cl, out.nu[ts], D, L, out.merit[r], g)
                assert res["gap"] <= pa.gap_bound(out.nu[ts], out.psi[ts], cl, RTOL, g) + res["allowance"], res
                done += 1
        assert done >= 2
    finally:
        m.close()


# ---- every token priced: the row, cfmm_solve and the host route() ---------------------------------
def test_all_tokens_agree_with_cfmm_solve_and_route():
    n = 8
    rng = np.random.default_rng(43)
    R, g, A = synth.product_pools(40, n, seed=44)
    spec = list(zip(R, g, A))
    cert = [oc.product(Rk, gk, Ak) for Rk, gk, Ak in spec]
    p = product_context(n, spec)
    try:
        c = rng.uniform(0.5, 2.0, n)
        out = p.quote_price_arbitrage(c[None, :], np.ones(n, bool))
        assert out.status[0] == 0 and out.token.tolist() == sorted(set(A.ravel().tolist()))
        assert out.leg_type.tolist() == [0] * len(spec) and out.leg_pool.tolist() == list(range(len(spec)))
        gd = max(float(out.nu @ out.psi), out.profit[0]) * 1.01
        rd = pa.certify(cert, n, out.token, c, out.nu, out.leg_delta, out.leg_lambda, out.merit[0], gd)
        box = sc.linear_nonnegative(c)
        xs, info = p.solve(lower=box.lower)
        Ds, Ls = p.trades()
        rs = sc.certify(cert, box, xs, Ds, Ls, check_stop=False)
        ps = float(c @ sum(np.bincount(A[:, s] - 1, weights=Ls[:, s] - Ds[:, s], minlength=n) for s in (0, 1)))
        # each profit exceeds the optimum by at most its infeasibility valued at c; each falls short
        # of it by at most its gap
        inf_d = rd["infeasibility"] * float(np.sum(c))
        slack = (abs(rd["gap"]) + rd["allowance"] + inf_d + abs(rs["gap"]) + rs["allowance"]
                 + rs["infeasibility"] * float(np.sum(xs)))
        assert abs(out.profit[0] - ps) <= slack + 1e-9 * abs(ps), (out.profit[0], ps, rd, rs)
        r = cr.Router(cr.LinearNonnegative(c), [cr.ProductTwoCoin(*s) for s in spec], n)
        cr.route(r)
        rh = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
        ph = float(c @ cr.netflows(r))
        slack = (abs(rd["gap"]) + rd["allowance"] + inf_d + abs(rh["gap"]) + rh["allowance"]
                 + rh["infeasibility"] * float(np.sum(r.v)))
        assert abs(out.profit[0] - ph) <= slack + 1e-9 * abs(ph), (out.profit[0], ph, rd, rh)
    finally:
        p.close()


# ---- execute ------------------------------------------------------------------------------------
def test_execute_leaves_no_arbitrage_and_no_arbitrage_fills_with_zeros():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(45)
        allowed = mask(rng, 8)
        c = prices(rng, 1, 8, zero=0.0)
        q0 = p.quote_price_arbitrage(c, allowed)
        assert q0.status[0] == 0 and q0.profit[0] > 0.0
        e = p.execute_price_arbitrage(c, allowed)
        same(q0, e)
        ts, sl = row_slices(e, 0)
        cl = row_prices(e, 0, allowed, c[0])
        g = max(float(e.nu[ts] @ e.psi[ts]), e.profit[0])
        # no pool of the row trades (beyond rounding) at the executed ν: g there is ~0
        v = np.ones(N)
        v[e.token[ts] - 1] = e.nu[ts]
        p.sweep(v, materialize=True)
        D, L = p.trades()
        gi = np.array([global_index(int(t), int(i)) for t, i in zip(e.leg_type[sl], e.leg_pool[sl])], np.int64)
        A = np.asarray(so.ingest_tokens(m.Ai, e.leg_type[sl], e.leg_pool[sl]), np.int64)
        after = float(np.sum(v[A - 1] * (L[gi] - D[gi])))
        assert abs(after) <= 1e-6 * g, (after, g)
        # quoting the row again finds a profit within the first row's gap bound
        q1 = p.quote_price_arbitrage(c, allowed)
        assert q1.profit[0] <= pa.gap_bound(e.nu[ts], e.psi[ts], cl, RTOL, g) + 1e-6 * g, (q1.profit[0], g)
    finally:
        m.close()
    # pools priced exactly at c (within their fee): nothing trades at ν⁰
    spec = [([100.0, 200.0], 0.997, [1, 2]), ([50.0, 150.0], 0.997, [1, 3]), ([300.0, 450.0], 0.997, [2, 3])]
    p = product_context(4, spec)
    try:
        allowed = np.array([1, 1, 1, 1], bool)
        before = state(p)
        out = p.execute_price_arbitrage([[1.0, 0.5, 1.0 / 3.0, 0.0], [0.0, 0.0, 1.0, 2.0]], allowed)
        assert out.status.tolist() == [0, 0] and out.solver_status.tolist() == [0, 0]
        assert out.iterations.tolist() == [0, 0] and out.fun_evals.tolist() == [1, 1]
        assert out.merit.tolist() == [0.0, 0.0] and out.profit.tolist() == [0.0, 0.0]
        assert out.token.tolist() == [1, 2, 3] and out.tok_off.tolist() == [0, 3, 3]  # row 1: T empty
        assert not np.any(out.psi) and not np.any(out.leg_delta) and not np.any(out.leg_lambda)
        same_state(before, state(p))
    finally:
        p.close()


def test_batch_equals_sequence_and_disjoint_rows_share_a_launch():
    rng = np.random.default_rng(46)
    allowed = mask(rng, 10)
    c = prices(rng, 6, 10)
    m1, m2 = Market(), Market()
    try:
        batch = m1.p.execute_price_arbitrage(c, allowed)
        seq = [m2.p.execute_price_arbitrage(c[r:r + 1], allowed) for r in range(len(c))]
        for r in range(len(c)):
            ts, sl = row_slices(batch, r)
            for f in ("profit", "status", "solver_status", "iterations", "fun_evals", "merit"):
                assert getattr(batch, f)[r] == getattr(seq[r], f)[0], (f, r)
            for f in ("token", "nu", "psi"):
                assert np.array_equal(getattr(batch, f)[ts], getattr(seq[r], f)), (f, r)
            for f in ("leg_type", "leg_pool", "leg_delta", "leg_lambda"):
                assert np.array_equal(getattr(batch, f)[sl], getattr(seq[r], f)), (f, r)
        same_state(state(m1.p), state(m2.p))
        assert np.any(batch.status == 0)
    finally:
        m1.close()
        m2.close()
    # two rows on disjoint halves of the tokens: one level; two rows sharing a token: two levels (one
    # ProductTwoCoin set, so every execute that fills a row has the same bookkeeping launches)
    n = 10
    spec = list(zip(*synth.product_pools(200, n, seed=46)))
    allowed = np.ones(n, bool)
    a = np.r_[rng.uniform(0.5, 2.0, 5), np.zeros(5)]
    b = np.r_[np.zeros(5), rng.uniform(0.5, 2.0, 5)]
    launches, outs, states = [], [], []
    for rows in ([a], [a, b], [a, a * 1.1]):
        p = product_context(n, spec)
        try:
            n0 = p.launch_count
            outs.append(p.execute_price_arbitrage(np.array(rows), allowed))
            launches.append(p.launch_count - n0)
            states.append(state(p))
        finally:
            p.close()
    assert np.all(outs[1].status == 0) and outs[2].status[0] == 0
    assert launches[1] == launches[0] and launches[2] == launches[0] + 1, launches
    p = product_context(n, spec)
    try:
        ea = p.execute_price_arbitrage(a[None, :], allowed)
        eb = p.execute_price_arbitrage(b[None, :], allowed)
        for f in ("profit", "status", "solver_status", "iterations", "fun_evals", "merit"):
            assert np.array_equal(getattr(outs[1], f), np.r_[getattr(ea, f), getattr(eb, f)]), f
        for f in ("token", "nu", "psi", "leg_type", "leg_pool", "leg_delta", "leg_lambda"):
            assert np.array_equal(getattr(outs[1], f), np.concatenate([getattr(ea, f), getattr(eb, f)])), f
        same_state(states[1], state(p))
    finally:
        p.close()


def test_zero_price_is_the_row_without_the_token():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(47)
        for k in (6, 10):
            allowed = mask(rng, k)
            A = np.flatnonzero(allowed)
            c = prices(rng, 4, k, zero=0.0)
            drop = rng.integers(0, k, 4)
            c[np.arange(4), drop] = 0.0
            full = p.quote_price_arbitrage(c, allowed)
            for r in range(4):
                sub = allowed.copy()
                sub[A[drop[r]]] = False
                one = p.quote_price_arbitrage(np.delete(c[r], drop[r])[None, :], sub)
                ts, sl = row_slices(full, r)
                for f in ("profit", "status", "solver_status", "iterations", "fun_evals", "merit"):
                    assert getattr(full, f)[r] == getattr(one, f)[0], (f, r)
                for f in ("token", "nu", "psi"):
                    assert np.array_equal(getattr(full, f)[ts], getattr(one, f)), (f, r)
                for f in ("leg_type", "leg_pool", "leg_delta", "leg_lambda"):
                    assert np.array_equal(getattr(full, f)[sl], getattr(one, f)), (f, r)
    finally:
        m.close()


def test_limits_quotes_and_rejections_change_nothing():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(48)
        allowed = mask(rng, 8)
        c = prices(rng, 3, 8)
        before = state(p)
        a = p.quote_price_arbitrage(c, allowed)
        b = p.quote_price_arbitrage(c, allowed)
        same(a, b)
        same_state(before, state(p))
        r = int(np.flatnonzero((a.status == 0) & (a.profit > 0))[0])
        row = c[r:r + 1]
        rev = p.execute_price_arbitrage(row, allowed, min_profit=np.nextafter(a.profit[r], np.inf))
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.profit[0] == 0.0 and not np.any(rev.leg_delta)
        same_state(before, state(p))
        ok = p.execute_price_arbitrage(row, allowed, min_profit=a.profit[r])
        assert ok.status[0] == 0 and ok.profit[0] == a.profit[r]
        after = state(p)
        # rejections, before anything runs
        lib, ctx = p._lib, p._ctx
        dp, u8 = C.POINTER(C.c_double), C.POINTER(C.c_uint8)
        mk = allowed.astype(np.uint8)
        ok_price = np.ascontiguousarray(row)
        for price, mp, msk in ((None, None, mk), (np.array([[-1.0] + [1.0] * 7]), None, mk),
                               (np.array([[np.nan] + [1.0] * 7]), None, mk), (np.array([[np.inf] + [1.0] * 7]), None, mk),
                               (np.zeros((1, 8)), None, mk), (ok_price, np.array([-1.0]), mk),
                               (ok_price, np.array([np.nan]), mk), (ok_price, np.array([np.inf]), mk),
                               (ok_price, None, None)):
            out = cr._lib.PriceArbOut()
            rc = lib.cfmm_execute_price_arbitrage(ctx, 1, None if price is None else price.ctypes.data_as(dp),
                                                  None if mp is None else mp.ctypes.data_as(dp),
                                                  None if msk is None else msk.ctypes.data_as(u8), None, C.byref(out))
            assert rc == cr._lib.CFMM_ERR_INVALID
        for bad in ({"rtol": 0.0}, {"max_iter": 0}, {"factr": -1.0}):
            with pytest.raises(cr.CFMMError):
                p.execute_price_arbitrage(row, allowed, opts=bad)
        assert lib.cfmm_execute_price_arbitrage(ctx, 0, None, None, mk.ctypes.data_as(u8), None, None) == 0
        same_state(after, state(p))
    finally:
        m.close()
    big = cr.DevicePools(300, device=0)
    try:
        R, g, A = synth.product_pools(50, 300, seed=3)
        big.add_product(R, g, A)
        big.finalize()
        with pytest.raises(cr.CFMMError, match="allowed tokens"):
            big._chk(big._lib.cfmm_quote_price_arbitrage(big._ctx, 1, np.ones(300).ctypes.data_as(C.POINTER(C.c_double)),
                                                         np.ones(300, np.uint8).ctypes.data_as(C.POINTER(C.c_uint8)),
                                                         None, None))
        sub = np.r_[np.ones(258, bool), np.zeros(42, bool)]
        out = big.quote_price_arbitrage(np.ones((1, 258)), sub)
        assert out.status[0] in (0, NC)
    finally:
        big.close()


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 22)
    n = 12
    allowed = np.zeros(n, bool)
    allowed[:8] = True
    rng = np.random.default_rng(49)
    c = prices(rng, 3, 8)
    profit, st, det = r.quote_price_arbitrage(c, allowed)
    assert np.array_equal(profit, det.profit) and np.any(st == 0)
    with pytest.raises(ValueError):
        r.quote_price_arbitrage(c, None)
    profit2, st2, det2 = r.execute_price_arbitrage(c, allowed)
    assert np.any(st2 == 0)
    for k in np.flatnonzero(st2 == 0):
        sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
        for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
            dev, _ = r._pools.pool_state(int(t), int(i), 1)
            pool = r.cfmms[r._type_lists[int(t)][int(i)]]
            assert np.array_equal(np.asarray(pool.R), dev[0])
