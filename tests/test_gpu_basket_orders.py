"""cfmm_quote_basket_orders / cfmm_execute_basket_orders (include/cfmm_b200.h) on the device.

On the five markets of test_gpu_subgraph_orders (plain, pools stored exchanged, after cfmm_compact,
after a UniV3 liquidity change, after a retire that follows the adjacency build): one-entry baskets
give cfmm_quote/execute_subgraph_orders' outputs bit for bit; each basket row's tokens and pool list
match basket_oracle over cfmm_pair_pools, its legs a materialising cfmm_sweep at the reported ν, and
its Ψ, paid and received the stated warp-tree sums.  On the plain market: filled rows with 2 to 16
entries pass the 50-digit certificate with the header's gap bound; on ProductTwoCoin markets a basket
receives at least its entries sold one by one, within the certified gaps; the execute is the quote
followed by the transition, equals row-by-row executes, reverts on limits and levels its launches;
quotes change no state and do not depend on the batch; bad arguments are rejected; the Router calls
refresh the pool objects; and the examples/liquidate.jl market agrees with route()."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import basket_oracle as bo
import solve_certificate as sc
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, fields, fresh, global_index, mask, pair_lists,
                                      row_slices, same_state, state)

pytestmark = pytest.mark.gpu


def baskets(rng, q, kmax):
    """q rows of 1..kmax distinct entries (amounts in [1, 20), one in five 0) and an output token."""
    tout, off, toks, amts = [], [0], [], []
    for _ in range(q):
        K = int(rng.integers(1, kmax + 1))
        pick = rng.choice(np.arange(1, N + 1), size=K + 1, replace=False)
        tout.append(int(pick[0]))
        toks += pick[1:].tolist()
        a = rng.uniform(1.0, 20.0, size=K)
        a[rng.random(K) < 0.2] = 0.0
        amts += a.tolist()
        off.append(len(toks))
    return np.array(tout, np.int64), np.array(off, np.int64), np.array(toks, np.int64), np.array(amts)


def entries(off, toks, amts, r):
    return toks[off[r]:off[r + 1]], amts[off[r]:off[r + 1]]


def check_basket_row(p, Ai, out, r, bt, ba):
    """Legs against a materialising sweep, the stated sums, paid per entry, and the stop's bounds."""
    ts, sl = row_slices(out, r)
    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
    v = np.ones(N)
    v[toks - 1] = nu
    p.sweep(v, materialize=True)
    D, L = p.trades()
    g = np.array([global_index(int(t), int(i)) for t, i in zip(out.leg_type[sl], out.leg_pool[sl])], np.int64)
    assert np.array_equal(D[g], out.leg_delta[sl]) and np.array_equal(L[g], out.leg_lambda[sl])
    A = bo.ingest_tokens(Ai, out.leg_type[sl], out.leg_pool[sl])
    assert np.array_equal(bo.warp_psi(A, out.leg_delta[sl], out.leg_lambda[sl], toks), psi)
    assert out.received[r] == psi[0]
    loc = {int(t): k for k, t in enumerate(toks)}
    paid = out.paid[out.basket_off[r]:out.basket_off[r + 1]]
    inT = [k for k, t in enumerate(bt) if int(t) in loc]
    for k, t in enumerate(bt):
        assert paid[k] == (0.0 - psi[loc[int(t)]] if int(t) in loc else 0.0)
    assert out.merit[r] <= RTOL and out.solver_status[r] == 0
    V = bo.basket_value(ba[inT], nu[[loc[int(bt[k])] for k in inT]])
    lin = np.zeros(len(toks))
    for k in inT:
        lin[loc[int(bt[k])]] = ba[k]
    lower = np.full(len(toks), bo.SQRT_EPS)
    lower[0] = 1 + bo.SQRT_EPS
    m, ok = bo.stop_bounds(nu, lin + psi, lower, V, RTOL * 1.01)
    assert ok, (m, out.merit[r])
    return V


@pytest.mark.parametrize("state_", STATES)
def test_one_entry_baskets_are_subgraph_orders(state_):
    m1, m2 = Market(state_), Market(state_)
    try:
        rng = np.random.default_rng(1)
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            tin = rng.integers(1, N + 1, size=10).astype(np.int64)
            tout = ((tin + rng.integers(1, N, size=10) - 1) % N + 1).astype(np.int64)
            amt = rng.uniform(1.0, 20.0, size=10)
            amt[4] = 0.0
            off = np.arange(11, dtype=np.int64)
            a = m1.p.quote_subgraph_orders(tin, tout, amt, allowed)
            b = m1.p.quote_basket_orders(tout, off, tin, amt, allowed)
            for x, y in zip(fields(a), fields(b)):
                assert np.array_equal(x, y)
            a = m1.p.execute_subgraph_orders(tin, tout, amt, allowed)
            b = m2.p.execute_basket_orders(tout, off, tin, amt, allowed)
            for x, y in zip(fields(a), fields(b)):
                assert np.array_equal(x, y)
            same_state(state(m1.p), state(m2.p))
    finally:
        m1.close()
        m2.close()


@pytest.mark.parametrize("state_", STATES)
def test_lists_legs_sums_and_fill_on_every_state(state_):
    m = Market(state_)
    try:
        p = m.p
        rng = np.random.default_rng(2)
        lists = pair_lists(p)
        n_filled = 0
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            tout, off, bt, ba = baskets(rng, 10, 5)
            out = p.quote_basket_orders(tout, off, bt, ba, allowed)
            for r in range(len(tout)):
                t, a = entries(off, bt, ba, r)
                T, pools, unreach = bo.row_basket(lists, t, a, int(tout[r]), allowed)
                ts, sl = row_slices(out, r)
                assert out.token[ts].tolist() == T, (r, out.token[ts], T)
                want = sorted(pools, key=lambda h: global_index(*h))
                assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == want
                if not np.any(a > 0):
                    assert out.status[r] == 0 and out.received[r] == 0.0 and out.solver_status[r] == -1
                elif unreach:
                    assert out.status[r] == cr._lib.ORDER_UNREACHABLE
                    assert out.received[r] == 0.0 and not np.any(out.leg_delta[sl])
                elif out.status[r] == 0:
                    check_basket_row(p, m.Ai, out, r, t, a)
                    n_filled += 1
                else:
                    assert out.status[r] == cr._lib.ORDER_NOT_CONVERGED and out.received[r] == 0.0
        assert n_filled >= 15
    finally:
        m.close()


def basket_certificate(cert, order, out, r, bt, ba, i):
    """solve_certificate.certify of basket row r under BasketLiquidation(i, Δin)'s box, with the
    per-token tolerance m_r <= rtol gives, and the header's gap bound |T|·rtol·V plus the box terms."""
    ts, sl = row_slices(out, r)
    toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
    nu = np.ones(N)
    nu[toks - 1] = nu_r
    D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
    D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
    lin = np.zeros(N)
    lin[np.asarray(bt) - 1] = ba
    box = sc.basket(i, lin)
    V = float(np.sum(lin[toks - 1] * nu_r))
    pgtol = float(np.max(out.merit[r] * V / nu_r)) * (1 + 1e-9)
    res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
    z = lin[toks - 1] + psi
    on = nu_r <= box.lower[toks - 1]
    box_terms = float(np.sum(np.maximum(z[on], 0.0) * (nu_r[on] - box.ref[toks - 1][on])))
    assert res["gap"] <= len(toks) * RTOL * V + box_terms + res["allowance"], (res, box_terms)
    return res, V


def test_certificate_k_2_to_16(mk_plain):
    p, m = mk_plain
    rng = np.random.default_rng(7)
    done = {}
    for K in (2, 4, 8, 16):
        allowed = mask(rng, 3)
        tout, bt = [], []
        for _ in range(4):
            pick = rng.choice(np.arange(1, N + 1), size=K + 1, replace=False)
            tout.append(int(pick[0]))
            bt += pick[1:].tolist()
        tout, bt = np.array(tout, np.int64), np.array(bt, np.int64)
        ba = rng.uniform(1.0, 20.0, size=len(bt))
        off = np.arange(0, len(bt) + 1, K, dtype=np.int64)
        out = p.quote_basket_orders(tout, off, bt, ba, allowed)
        for r in np.flatnonzero(out.status == 0)[:2]:
            ts, sl = row_slices(out, r)
            pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
            q, order, cert = fresh(m, pools)
            try:
                basket_certificate(cert, order, out, r, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], int(tout[r]))
                done[K] = done.get(K, 0) + 1
            finally:
                q.close()
    assert all(done.get(K, 0) >= 1 for K in (2, 4, 8, 16)), done


@pytest.fixture(scope="module")
def mk_plain():
    m = Market()
    yield m.p, m
    m.close()


def product_market(seed):
    p = cr.DevicePools(N, device=0)
    R, g, A = synth.product_pools(200, N, seed=seed)
    p.add_product(R, g, A)
    p.finalize()
    return p


def test_basket_beats_selling_one_by_one_on_product_pools():
    """A fee makes a ProductTwoCoin pool's net trade over a sequence no better than one trade, so the
    entries sold one after another are a feasible basket trade: the basket receives at least as much,
    less the certified gaps of the basket row and of the sequential rows."""
    rng = np.random.default_rng(11)
    allowed = mask(rng, 6)
    n_cmp = 0
    for K in (2, 3, 5):
        for _ in range(3):
            pick = rng.choice(np.arange(1, N + 1), size=K + 1, replace=False)
            i, bt = int(pick[0]), pick[1:].astype(np.int64)
            ba = rng.uniform(1.0, 20.0, size=K)
            a, b = product_market(21), product_market(21)
            try:
                out = a.execute_basket_orders([i], [0, K], bt, ba, allowed)
                seq = b.execute_subgraph_orders(bt, np.full(K, i, np.int64), ba, allowed)
                if out.status[0] != 0 or np.any(seq.status != 0):
                    continue
                nu_b = out.nu[out.tok_off[0]:out.tok_off[1]]
                V = bo.basket_value(ba, nu_b[1:K + 1])
                slack = len(nu_b) * RTOL * V / nu_b[0]
                for r in range(K):
                    nu_r = seq.nu[seq.tok_off[r]:seq.tok_off[r + 1]]
                    slack += len(nu_r) * RTOL * ba[r] * nu_r[1] / nu_r[0]
                assert out.received[0] >= np.sum(seq.received) - slack, (out.received[0], seq.received, slack)
                n_cmp += 1
            finally:
                a.close()
                b.close()
    assert n_cmp >= 5


def test_execute_is_quote_then_transition_and_row_by_row():
    rng = np.random.default_rng(5)
    allowed = mask(rng, 5)
    tout, off, bt, ba = baskets(rng, 6, 4)
    m1, m2 = Market(), Market()
    try:
        p1, p2 = m1.p, m2.p
        # one solved row: the execute's outputs are the quote's, and its two-coin pools move by its legs
        q = p1.quote_basket_orders(tout, off, bt, ba, allowed)
        r = int(np.flatnonzero((q.status == 0) & (q.solver_status == 0))[0])
        o1 = np.array([0, off[r + 1] - off[r]], np.int64)
        ex = p1.execute_basket_orders(tout[r:r + 1], o1, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], allowed)
        one = p2.quote_basket_orders(tout[r:r + 1], o1, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], allowed)
        for x, y in zip(fields(ex), fields(one)):
            assert np.array_equal(x, y)
        # the transition of the two-coin pools: R <- (R + γΔ) − Λ at the row's legs
        assert ex.status[0] == 0
        t0 = ex.leg_type == 0
        idx = ex.leg_pool[t0]
        R0, g0 = p2.pool_state(0)[0][idx], m1.prod[1][idx]
        want = (R0 + g0[:, None] * ex.leg_delta[t0]) - ex.leg_lambda[t0]
        assert np.any(ex.leg_delta[t0]) and np.allclose(p1.pool_state(0)[0][idx], want, rtol=1e-12, atol=0.0)
    finally:
        m1.close()
        m2.close()
    m1, m2 = Market(), Market()
    try:
        batch = m1.p.execute_basket_orders(tout, off, bt, ba, allowed)
        for r in range(len(tout)):
            o1 = np.array([0, off[r + 1] - off[r]], np.int64)
            one = m2.p.execute_basket_orders(tout[r:r + 1], o1, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], allowed)
            ts, sl = row_slices(batch, r)
            assert batch.received[r] == one.received[0] and batch.status[r] == one.status[0]
            assert np.array_equal(batch.paid[off[r]:off[r + 1]], one.paid)
            assert np.array_equal(batch.leg_delta[sl], one.leg_delta) and np.array_equal(batch.nu[ts], one.nu)
        same_state(state(m1.p), state(m2.p))
        assert np.any(batch.status == 0)
    finally:
        m1.close()
        m2.close()


def test_limits_launches_and_no_state_change(mk_plain):
    p, _ = mk_plain
    rng = np.random.default_rng(6)
    allowed = mask(rng, 5)
    tout, off, bt, ba = baskets(rng, 9, 6)
    before = state(p)
    a = p.quote_basket_orders(tout, off, bt, ba, allowed)
    b = p.quote_basket_orders(tout, off, bt, ba, allowed)
    for x, y in zip(fields(a), fields(b)):
        assert np.array_equal(x, y)
    same_state(before, state(p))
    for r in (0, 4, 8):   # a row's result does not depend on the batch
        o1 = np.array([0, off[r + 1] - off[r]], np.int64)
        one = p.quote_basket_orders(tout[r:r + 1], o1, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], allowed)
        ts, sl = row_slices(a, r)
        assert one.received[0] == a.received[r] and one.status[0] == a.status[r]
        assert np.array_equal(one.paid, a.paid[off[r]:off[r + 1]]) and np.array_equal(one.nu, a.nu[ts])
        assert np.array_equal(one.leg_delta, a.leg_delta[sl])
    m = Market()
    try:
        r = int(np.flatnonzero((a.status == 0) & (a.solver_status == 0))[0])
        o1 = np.array([0, off[r + 1] - off[r]], np.int64)
        args = (tout[r:r + 1], o1, bt[off[r]:off[r + 1]], ba[off[r]:off[r + 1]], allowed)
        before = state(m.p)
        rev = m.p.execute_basket_orders(*args, limit=np.nextafter(a.received[r:r + 1], np.inf))
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.received[0] == 0.0 and not np.any(rev.paid)
        same_state(before, state(m.p))
        ok = m.p.execute_basket_orders(*args, limit=a.received[r:r + 1])
        assert ok.status[0] == 0 and ok.received[0] == a.received[r]
        # rows on disjoint tokens with an empty mask run in one launch; rows sharing a token do not
        none = np.zeros(N, bool)
        dis = (np.array([1, 4, 7], np.int64), np.array([0, 2, 4, 6], np.int64),
               np.array([2, 3, 5, 6, 8, 9], np.int64), np.full(6, 3.0))
        n0 = m.p.launch_count
        m.p.execute_basket_orders(*dis, none)
        n_dis = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_basket_orders(dis[0][:1], dis[1][:2], dis[2][:2], dis[3][:2], none)
        n_one = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_basket_orders(np.array([1, 4], np.int64), np.array([0, 2, 4], np.int64),
                                  np.array([2, 3, 5, 3], np.int64), np.full(4, 3.0), none)
        n_two = m.p.launch_count - n0
        assert n_dis == n_one and n_two == n_one + 1
    finally:
        m.close()


def test_rejections(mk_plain):
    p, _ = mk_plain
    lib = p._lib
    ip, dp, u8 = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    allowed = np.ones(N, bool)

    def call(tout, off, bt, ba, amask=allowed, execute=False, limit=None, opts=None, out=None):
        tout, off, bt = (np.asarray(x, np.int64) for x in (tout, off, bt))
        ba = np.asarray(ba, np.float64)
        mk = np.asarray(amask, np.uint8)
        o = out or cr._lib.BasketOut()
        if execute:
            lim = None if limit is None else np.asarray(limit, np.float64).ctypes.data_as(dp)
            return lib.cfmm_execute_basket_orders(p._ctx, len(tout), tout.ctypes.data_as(ip), off.ctypes.data_as(ip),
                                                  bt.ctypes.data_as(ip), ba.ctypes.data_as(dp), lim,
                                                  mk.ctypes.data_as(u8), opts, C.byref(o))
        return lib.cfmm_quote_basket_orders(p._ctx, len(tout), tout.ctypes.data_as(ip), off.ctypes.data_as(ip),
                                            bt.ctypes.data_as(ip), ba.ctypes.data_as(dp), mk.ctypes.data_as(u8),
                                            opts, C.byref(o))

    assert call([1], [0, 2], [2, 3], [1.0, 1.0]) == 0
    bad = [
        ([1], [1, 2], [2, 3], [1.0, 1.0]),            # basket_off[0] != 0
        ([1, 2], [0, 2, 1], [2, 3], [1.0, 1.0]),      # decreasing
        ([1, 2], [0, 2, 2], [2, 3], [1.0, 1.0]),      # an empty basket
        ([1], [0, 17], list(range(2, 19)), [1.0] * 17),   # 17 entries
        ([1], [0, 2], [2, 2], [1.0, 1.0]),            # a duplicate
        ([1], [0, 2], [2, 1], [1.0, 1.0]),            # token_out in the basket
        ([0], [0, 1], [2], [1.0]),                    # token_out outside 1..n
        ([1], [0, 1], [N + 1], [1.0]),                # a basket token outside 1..n
        ([1], [0, 1], [2], [-1.0]),                   # a negative amount
        ([1], [0, 1], [2], [float("nan")]),
    ]
    for args in bad:
        assert call(*args) == cr._lib.CFMM_ERR_INVALID, args
    assert call([1], [0, 1], [2], [1.0], execute=True, limit=[float("inf")]) == cr._lib.CFMM_ERR_INVALID
    assert call([1], [0, 1], [2], [1.0], execute=True, limit=[-1.0]) == cr._lib.CFMM_ERR_INVALID
    o = cr._lib.SubgraphOpts(1000, 4000, 0.0, 0.0)
    assert call([1], [0, 1], [2], [1.0], opts=C.byref(o)) == cr._lib.CFMM_ERR_INVALID
    assert lib.cfmm_quote_basket_orders(p._ctx, 1, np.array([1], np.int64).ctypes.data_as(ip),
                                        np.array([0, 1], np.int64).ctypes.data_as(ip),
                                        np.array([2], np.int64).ctypes.data_as(ip),
                                        np.array([1.0]).ctypes.data_as(dp), None, None, None) == cr._lib.CFMM_ERR_INVALID
    # an execute whose outputs do not fit changes nothing
    before = state(p)
    small = cr._lib.BasketOut()
    tokbuf = np.zeros(1, np.int64)
    small.token, small.tok_cap = tokbuf.ctypes.data_as(ip), 1
    assert call([1], [0, 2], [2, 3], [1.0, 1.0], execute=True, out=small) == cr._lib.CFMM_ERR_INVALID
    same_state(before, state(p))
    # tokens other than token_out: basket ∪ B at most 257
    big = cr.DevicePools(300, device=0)
    try:
        R, g, A = synth.product_pools(50, 300, seed=3)
        big.add_product(R, g, A)
        big.finalize()
        am = np.r_[np.ones(257, bool), np.zeros(43, bool)]
        big.quote_basket_orders([1], [0, 2], [2, 290], [1.0, 1.0], am)          # 256 allowed + 290 = 257
        with pytest.raises(cr.CFMMError, match="row 0"):
            big.quote_basket_orders([1], [0, 2], [290, 291], [1.0, 1.0], am)    # 256 allowed + 2 = 258
    finally:
        big.close()


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 21)
    try:
        n = 12
        allowed = np.zeros(n, bool)
        allowed[:6] = True
        tout = np.array([11, 12, 7])
        bsk = [{7: 5.0, 8: 2.0}, ([9, 10], [20.0, 1.0]), {8: 3.0}]
        paid, recv, st, det = r.quote_basket_orders(tout, bsk, allowed)
        assert [len(x) for x in paid] == [2, 2, 1]
        reach = st != cr._lib.ORDER_UNREACHABLE
        assert np.all(st[reach] == 0) and np.any(reach)
        with pytest.raises(ValueError):
            r.quote_basket_orders(tout, bsk, None)
        paid2, recv2, st2, det2 = r.execute_basket_orders(tout, bsk, allowed, limits=np.zeros(len(tout)))
        assert np.all(np.isin(st2[reach], (0, cr._lib.ORDER_NOT_CONVERGED))) and np.any(st2 == 0)
        for k in np.flatnonzero(st2 == 0):
            sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
            for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
                dev, _ = r._pools.pool_state(int(t), int(i), 1)
                c = r.cfmms[r._type_lists[int(t)][int(i)]]
                assert np.array_equal(np.asarray(c.R), dev[0])
    finally:
        r.close() if hasattr(r, "close") else None


@pytest.mark.parametrize("i, delta_in", [(1, [0.0, 10.0, 100.0]), (2, [10.0, 0.0, 0.0])])
def test_liquidate_example_against_route(i, delta_in):
    spec = [([1e3, 1e4], [1, 2]), ([1e3, 1e2], [2, 3]), ([1e3, 2e4], [1, 3])]
    p = cr.DevicePools(3, device=0)
    try:
        p.add_product(np.array([s[0] for s in spec]), np.full(3, 0.997), np.array([s[1] for s in spec], np.int64))
        p.finalize()
        bt = [t + 1 for t in range(3) if delta_in[t] > 0]
        out = p.quote_basket_orders([i], [0, len(bt)], bt, [delta_in[t - 1] for t in bt], np.ones(3, bool))
        assert out.status[0] == 0
    finally:
        p.close()
    r = cr.Router(cr.BasketLiquidation(i, delta_in), [cr.ProductTwoCoin(R, 0.997, A) for R, A in spec], 3)
    try:
        cr.route(r, pgtol=1e-10, factr=1e1)
        net = cr.netflows(r)
        nu = out.nu
        V = bo.basket_value([delta_in[t - 1] for t in bt], nu[1:1 + len(bt)])
        assert abs(out.received[0] - net[i - 1]) <= 3 * RTOL * V / nu[0] + 1e-6 * net[i - 1]
    finally:
        r.close() if hasattr(r, "close") else None
