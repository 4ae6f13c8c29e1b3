"""cfmm_quote_basket_swap_orders / cfmm_execute_basket_swap_orders (include/cfmm_b200.h) on the device.

On the five markets of test_gpu_subgraph_orders: a buy row with one bought entry and nothing sold gives
the exact-out subgraph row's outputs bit for bit (quote and execute, limits translated, same final
state); mixed rows list basket_swap_oracle's tokens in the buy row's local order and their pools, their
legs match a materialising cfmm_sweep at the reported ν, their Ψ the warp-tree sums, and every filled row
meets the stop's bounds with every bought entry receiving at least y.  Sell-only rows through the new
calls are basket rows bit for bit with the same launches.  On the plain market: filled mixed rows with 2
to 16 entries pass the 50-digit certificate on their raw box; on ProductTwoCoin markets a mixed row nets
at least the same order run in turn (basket sale, then one exact-out row per bought token), within the
certified gaps; with every token allowed a row agrees with the host route() and cfmm_solve under
BasketSwap; the execute is the quote followed by the transition, equals row-by-row executes, takes
signed limits and levels its launches; quotes change no state and do not depend on the batch; edge rows
and rejections change nothing; and the Router calls refresh the pool objects."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import basket_oracle as bo
import basket_swap_oracle as bs
import solve_certificate as sc
from subgraph_exact_out_oracle import capacity, y_prime
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, fields, fresh, global_index, mask, pair_lists,
                                      row_slices, same_state, state)

pytestmark = pytest.mark.gpu

OUT = cr._lib.SWAP_EXACT_OUT
NC = cr._lib.ORDER_NOT_CONVERGED
UNREACH = cr._lib.ORDER_UNREACHABLE


def mixed(rng, q, kmax, y_hi=5.0):
    """q rows of 2..kmax distinct entries, at least one sold (δ in [1, 20)) and one bought (y in
    [0.2, y_hi)), and a settlement token.  Returns (token_out, off, tokens, amounts, kind)."""
    tout, off, toks, amts, kind = [], [0], [], [], []
    for _ in range(q):
        K = int(rng.integers(2, kmax + 1))
        pick = rng.choice(np.arange(1, N + 1), size=K + 1, replace=False)
        k = rng.permutation(np.r_[[0, OUT], rng.integers(0, 2, size=K - 2)]).astype(np.uint8)
        tout.append(int(pick[0]))
        toks += pick[1:].tolist()
        amts += np.where(k == OUT, rng.uniform(0.2, y_hi, K), rng.uniform(1.0, 20.0, K)).tolist()
        kind += k.tolist()
        off.append(len(toks))
    return (np.array(tout, np.int64), np.array(off, np.int64), np.array(toks, np.int64), np.array(amts),
            np.array(kind, np.uint8))


def one_row(args, r):
    """Row r of (token_out, off, tokens, amounts, kind) as a batch of one."""
    tout, off, toks, amts, kind = args
    sl = slice(off[r], off[r + 1])
    return tout[r:r + 1], np.array([0, off[r + 1] - off[r]], np.int64), toks[sl], amts[sl], kind[sl]


def terms(out, r, toks_r, amts_r, kind_r):
    ts, _ = row_slices(out, r)
    toks = out.token[ts]
    lin, amt, slots = bs.entry_terms(toks, toks_r, amts_r, kind_r == OUT, RTOL)
    n_buy = int(sum(1 for t, k in zip(toks_r, kind_r) if k == OUT and int(t) in set(toks.tolist())))
    return toks, lin, amt, slots, n_buy


def check_buy_row(p, Ai, out, r, toks_r, amts_r, kind_r):
    """Legs against a materialising sweep, the stated sums, paid per entry, and the stop's bounds of
    filled buy row r.  Returns (V, n_buy)."""
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
    toks, lin, amt, slots, n_buy = terms(out, r, toks_r, amts_r, kind_r)
    assert out.received[r] == psi[n_buy] and nu[n_buy] == 1.0 and np.all(nu >= sc.SQRT_EPS)
    loc = {int(t): k for k, t in enumerate(toks)}
    paid = out.paid[out.basket_off[r]:out.basket_off[r + 1]]
    for k, t in enumerate(toks_r):
        assert paid[k] == (0.0 - psi[loc[int(t)]] if int(t) in loc else 0.0)
        if kind_r[k] == OUT and amts_r[k] > 0.0:
            assert psi[loc[int(t)]] >= amts_r[k]
            if nu[loc[int(t)]] > sc.SQRT_EPS:
                assert psi[loc[int(t)]] <= amts_r[k] * (1 + 2 * RTOL) * (1 + 1e-12)
    assert out.merit[r] <= RTOL and out.solver_status[r] == 0
    m, ok = bs.stop_bounds(nu, lin + psi, n_buy, amt, slots, n_buy, RTOL * 1.01)
    assert ok, (m, out.merit[r])
    return bs.local_sum(amt, nu, slots), n_buy


def same_as_exact_out(a, b):
    """Subgraph exact-out outputs a and one-entry buy-row outputs b agree bit for bit on every row that
    is not unreachable (an unreachable row lists the component of a different token in each call), with
    received ↔ −paid and paid ↔ −received.  Returns the number of rows compared."""
    n = 0
    for r in range(len(a.status)):
        assert a.status[r] == b.status[r], r
        if b.status[r] == UNREACH:
            continue
        n += 1
        ta, la = row_slices(a, r)
        tb, lb = row_slices(b, r)
        for f in ("solver_status", "iterations", "fun_evals", "merit"):
            assert getattr(a, f)[r] == getattr(b, f)[r], (f, r)
        for f in ("token", "nu", "psi"):
            assert np.array_equal(getattr(a, f)[ta], getattr(b, f)[tb]), (f, r)
        for f in ("leg_type", "leg_pool", "leg_delta", "leg_lambda"):
            assert np.array_equal(getattr(a, f)[la], getattr(b, f)[lb]), (f, r)
        assert a.received[r] == 0.0 - b.paid[r] and a.paid[r] == 0.0 - b.received[r], r
    return n


def check_not_filled(out, r):
    _, sl = row_slices(out, r)
    assert out.received[r] == 0.0 and not np.any(out.paid[out.basket_off[r]:out.basket_off[r + 1]])
    assert not np.any(out.leg_delta[sl]) and not np.any(out.leg_lambda[sl])


@pytest.mark.parametrize("state_", STATES)
def test_one_buy_rows_are_exact_out_rows(state_):
    m1, m2 = Market(state_), Market(state_)
    try:
        rng = np.random.default_rng(31)
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            settle = rng.integers(1, N + 1, size=10).astype(np.int64)
            bought = ((settle + rng.integers(1, N, size=10) - 1) % N + 1).astype(np.int64)
            y = rng.uniform(0.2, 8.0, size=10)
            off = np.arange(11, dtype=np.int64)
            a = m1.p.quote_subgraph_orders(settle, bought, y, allowed, kind=OUT)
            b = m1.p.quote_basket_orders(settle, off, bought, y, allowed, kind=OUT)
            assert same_as_exact_out(a, b) >= 5
            # executes with the limits translated: a maximum paid p is a minimum net of −p
            # (a row over pools that disagree on prices can be paid to buy: its paid is negative, and an
            # exact-out limit is at least 0)
            paid = np.maximum(np.where(a.status == 0, a.paid, 1.0) * rng.uniform(0.99, 1.01, 10), 0.0)
            lim = np.where(rng.random(10) < 0.5, np.inf, paid)
            ea = m1.p.execute_subgraph_orders(settle, bought, y, allowed, limit=lim, kind=OUT)
            eb = m2.p.execute_basket_orders(settle, off, bought, y, allowed, limit=0.0 - lim, kind=OUT)
            same_as_exact_out(ea, eb)
            same_state(state(m1.p), state(m2.p))
    finally:
        m1.close()
        m2.close()


@pytest.mark.parametrize("state_", ("plain", "compact"))
def test_sell_only_rows_are_basket_rows(state_):
    from test_gpu_basket_orders import baskets
    m1, m2 = Market(state_), Market(state_)
    try:
        rng = np.random.default_rng(32)
        for k in (0, 5):
            allowed = mask(rng, k)
            tout, off, bt, ba = baskets(rng, 8, 5)
            for execute in (False, True):
                run = "execute_basket_orders" if execute else "quote_basket_orders"
                n0 = m1.p.launch_count
                a = getattr(m1.p, run)(tout, off, bt, ba, allowed)
                na = m1.p.launch_count - n0
                n0 = m2.p.launch_count
                b = getattr(m2.p, run)(tout, off, bt, ba, allowed, kind=np.zeros(len(bt), np.uint8))
                nb = m2.p.launch_count - n0
                assert na == nb
                for x, y in zip(fields(a), fields(b)):
                    assert np.array_equal(x, y)
                same_state(state(m1.p), state(m2.p))
    finally:
        m1.close()
        m2.close()


@pytest.mark.parametrize("state_", STATES)
def test_mixed_rows_lists_legs_sums_and_fill(state_):
    m = Market(state_)
    try:
        p = m.p
        rng = np.random.default_rng(33)
        lists = pair_lists(p)
        n_filled = n_nc = 0
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            args = mixed(rng, 10, 5)
            tout, off, bt, ba, kd = args
            out = p.quote_basket_orders(tout, off, bt, ba, allowed, kind=kd)
            for r in range(len(tout)):
                sl_e = slice(off[r], off[r + 1])
                T, pools, unreach = bs.row_order(lists, bt[sl_e], ba[sl_e], kd[sl_e] == OUT, int(tout[r]), allowed)
                ts, sl = row_slices(out, r)
                assert out.token[ts].tolist() == T, (r, out.token[ts], T)
                assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == sorted(
                    pools, key=lambda h: global_index(*h))
                if unreach:
                    assert out.status[r] == UNREACH and out.solver_status[r] == -1
                    check_not_filled(out, r)
                elif out.status[r] == 0:
                    check_buy_row(p, m.Ai, out, r, bt[sl_e], ba[sl_e], kd[sl_e])
                    n_filled += 1
                else:
                    assert out.status[r] in (NC, UNREACH)
                    n_nc += out.status[r] == NC
                    check_not_filled(out, r)
        print(f"{state_}: {n_filled} filled, {n_nc} not converged")
        assert n_filled >= 15
    finally:
        m.close()


def buy_certificate(cert, order, out, r, toks_r, amts_r, kind_r, i):
    """solve_certificate.certify of buy row r on its raw box (lin = Δin − y′, ν_i = 1), with the
    per-token tolerance m_r <= rtol gives and the header's gap bound |T|·rtol·V plus the box terms."""
    ts, sl = row_slices(out, r)
    toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
    nu = np.ones(N)
    nu[toks - 1] = nu_r
    D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
    D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
    d_in, y = np.zeros(N), np.zeros(N)
    for t, a, k in zip(toks_r, amts_r, kind_r):
        (y if k == OUT else d_in)[int(t) - 1] = a
    box = bs.box(N, i, d_in, y, RTOL)
    _, _, amt, slots, _ = terms(out, r, toks_r, amts_r, kind_r)
    V = bs.local_sum(amt, nu_r, slots)
    pgtol = float(np.max(out.merit[r] * V / nu_r)) * (1 + 1e-9)
    res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
    z = box.lin[toks - 1] + psi
    on = (nu_r <= box.lower[toks - 1]) & (toks != i)
    box_terms = float(np.sum(np.maximum(z[on], 0.0) * (nu_r[on] - box.ref[toks - 1][on])))
    assert res["gap"] <= len(toks) * RTOL * V + box_terms + res["allowance"], (res, box_terms)
    return res, box, V


@pytest.fixture(scope="module")
def mk_plain():
    m = Market()
    yield m.p, m
    m.close()


def test_certificate_k_2_to_16(mk_plain):
    p, m = mk_plain
    rng = np.random.default_rng(37)
    done = {}
    for K in (2, 4, 8, 16):
        allowed = mask(rng, 3)
        for _ in range(3):
            args = mixed(rng, 4, K, y_hi=2.0)
            tout, off, bt, ba, kd = args
            keep = [r for r in range(4) if off[r + 1] - off[r] == K] or [int(np.argmax(np.diff(off)))]
            out = p.quote_basket_orders(tout, off, bt, ba, allowed, kind=kd)
            for r in [r for r in keep if out.status[r] == 0][:1]:
                ts, sl = row_slices(out, r)
                pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
                q, order, cert = fresh(m, pools)
                try:
                    e = slice(off[r], off[r + 1])
                    buy_certificate(cert, order, out, r, bt[e], ba[e], kd[e], int(tout[r]))
                    n = int(off[r + 1] - off[r])
                    done[n] = done.get(n, 0) + 1
                finally:
                    q.close()
    assert len(done) >= 3 and max(done) >= 8, done


def product_market(seed):
    p = cr.DevicePools(N, device=0)
    R, g, A = synth.product_pools(200, N, seed=seed)
    p.add_product(R, g, A)
    p.finalize()
    return p


def test_joint_row_beats_the_sequence_on_product_pools():
    """A fee makes a ProductTwoCoin pool's net trade over a sequence no better than one trade, so the
    basket sale into i followed by one exact-out row per bought token (paid in i) is a feasible joint
    trade: the joint row nets at least as much of i, less both sides' certified gaps and the cost of the
    overbuy y′ − y at the bought tokens' prices."""
    rng = np.random.default_rng(41)
    allowed = mask(rng, 6)
    n_cmp = 0
    for _ in range(12):
        args = mixed(rng, 1, 5)
        tout, off, bt, ba, kd = args
        i = int(tout[0])
        a, b = product_market(21), product_market(21)
        try:
            out = a.execute_basket_orders(*args[:4], allowed, kind=kd)
            s_t, s_a = bt[kd != OUT], ba[kd != OUT]
            b_t, b_a = bt[kd == OUT], ba[kd == OUT]
            sale = b.execute_basket_orders([i], [0, len(s_t)], s_t, s_a, allowed)
            buys = b.execute_subgraph_orders(np.full(len(b_t), i, np.int64), b_t, b_a, allowed, kind=OUT)
            if out.status[0] != 0 or sale.status[0] != 0 or np.any(buys.status != 0):
                continue
            toks, _, amt, slots, n_buy = terms(out, 0, bt, ba, kd)
            nu = out.nu[out.tok_off[0]:out.tok_off[1]]
            V = bs.local_sum(amt, nu, slots)
            slack = len(nu) * RTOL * V + sum(2 * RTOL * amt[l] * nu[l] for l in range(n_buy))
            nu_s = sale.nu[sale.tok_off[0]:sale.tok_off[1]]
            slack += len(nu_s) * RTOL * bo.basket_value(s_a, nu_s[1:1 + len(s_t)]) / nu_s[0]
            for r in range(len(b_t)):
                nu_r = buys.nu[buys.tok_off[r]:buys.tok_off[r + 1]]
                slack += (len(nu_r) + 2) * RTOL * b_a[r] * nu_r[0]
            seq = sale.received[0] - np.sum(buys.paid)
            assert out.received[0] >= seq - slack, (out.received[0], seq, slack)
            n_cmp += 1
        finally:
            a.close()
            b.close()
    assert n_cmp >= 5, n_cmp


def test_whole_set_agrees_with_route_and_cfmm_solve():
    """Every token allowed on a small ProductTwoCoin market: the buy row, the host route() and cfmm_solve
    under BasketSwap(i, Δin, y′) over the same pools reach dual values within their certified gaps."""
    import order_certificate as oc
    from test_host_logic import OraclePools

    n = 6
    R, g, A = synth.product_pools(12, n, seed=5)
    cert = [oc.product(R[k], g[k], A[k]) for k in range(len(R))]
    i, d_in, y = 1, np.zeros(n), np.zeros(n)
    d_in[[2, 4]] = [8.0, 3.0]
    y[[1, 5]] = [2.0, 1.5]
    yp = np.array([y_prime(v, RTOL) if v > 0 else 0.0 for v in y])
    box = bs.box(n, i, d_in, y, RTOL)
    p = cr.DevicePools(n, device=0)
    try:
        p.add_product(R, g, A)
        p.finalize()
        tk = np.array([3, 2, 5, 6], np.int64)
        ta = d_in[tk - 1] + y[tk - 1]
        kd = np.array([0, OUT, 0, OUT], np.uint8)
        out = p.quote_basket_orders([i], [0, 4], tk, ta, np.ones(n, bool), kind=kd)
        assert out.status[0] == 0 and sorted(out.leg_pool.tolist()) == list(range(len(R)))
        nu = np.ones(n)
        nu[out.token - 1] = out.nu
        D, L = np.zeros((len(R), 2)), np.zeros((len(R), 2))
        D[out.leg_pool], L[out.leg_pool] = out.leg_delta, out.leg_lambda
        _, _, amt, slots, _ = terms(out, 0, tk, ta, kd)
        V = bs.local_sum(amt, out.nu, slots)
        a = sc.certify(cert, box, nu, D, L, pgtol=float(np.max(out.merit[0] * V / out.nu)) * (1 + 1e-9))
        xs, _ = p.solve(**box.solve_args())
        Ds, Ls = p.trades()
        b = sc.certify(cert, box, xs, Ds, Ls, check_stop=False)
    finally:
        p.close()
    r = cr.Router(cr.BasketSwap(i, d_in, yp), [cr.ProductTwoCoin(R[k], g[k], A[k]) for k in range(len(R))], n,
                  _pools_factory=OraclePools)
    cr.route(r, pgtol=1e-11, factr=1e1)
    c = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
    for x, z in ((a, b), (a, c), (b, c)):
        slack = (abs(x["gap"]) + x["allowance"] + abs(z["gap"]) + z["allowance"]
                 + (x.get("infeasibility", 0.0) + z.get("infeasibility", 0.0)) * float(np.sum(xs) + np.sum(r.v)))
        assert abs(x["g50"] - z["g50"]) <= slack, (x, z)
    assert out.psi[list(out.token).index(2)] >= y[1] and out.psi[list(out.token).index(6)] >= y[5]


def test_execute_is_quote_then_transition_and_row_by_row():
    rng = np.random.default_rng(43)
    allowed = mask(rng, 5)
    args = mixed(rng, 6, 4)
    tout, off, bt, ba, kd = args
    m = Market()
    try:
        q = m.p.quote_basket_orders(tout, off, bt, ba, allowed, kind=kd)
        r = int(np.flatnonzero(q.status == 0)[0])
        one = one_row(args, r)
        ex = m.p.execute_basket_orders(*one[:4], allowed, kind=one[4])
        assert ex.status[0] == 0 and ex.received[0] == q.received[r]
        pools = list(zip(ex.leg_type.tolist(), ex.leg_pool.tolist()))
        f, _, _ = fresh(m, pools)
        try:
            nu = np.ones(N)
            nu[ex.token - 1] = ex.nu
            f.sweep(nu, materialize=True)
            f.apply_trades()
            sel = {t: sorted(i for tt, i in pools if tt == t) for t in (0, 1, 2)}
            for t in (0, 1, 2):
                if sel[t]:
                    assert np.array_equal(m.p.pool_state(t)[0][sel[t]], f.pool_state(t)[0]), t
        finally:
            f.close()
    finally:
        m.close()
    m1, m2 = Market(), Market()
    try:
        batch = m1.p.execute_basket_orders(tout, off, bt, ba, allowed, kind=kd)
        for r in range(len(tout)):
            one = m2.p.execute_basket_orders(*one_row(args, r)[:4], allowed, kind=one_row(args, r)[4])
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
    rng = np.random.default_rng(44)
    allowed = mask(rng, 5)
    args = mixed(rng, 9, 5)
    tout, off, bt, ba, kd = args
    before = state(p)
    a = p.quote_basket_orders(tout, off, bt, ba, allowed, kind=kd)
    b = p.quote_basket_orders(tout, off, bt, ba, allowed, kind=kd)
    for x, y in zip(fields(a), fields(b)):
        assert np.array_equal(x, y)
    same_state(before, state(p))
    for r in (0, 4, 8):   # a row's result does not depend on the batch
        one = p.quote_basket_orders(*one_row(args, r)[:4], allowed, kind=one_row(args, r)[4])
        ts, sl = row_slices(a, r)
        assert one.received[0] == a.received[r] and one.status[0] == a.status[r]
        assert np.array_equal(one.paid, a.paid[off[r]:off[r + 1]]) and np.array_equal(one.nu, a.nu[ts])
        assert np.array_equal(one.leg_delta, a.leg_delta[sl])
    m = Market()
    try:
        r = int(np.flatnonzero(a.status == 0)[0])
        one = one_row(args, r)
        before = state(m.p)
        lim = np.nextafter(a.received[r:r + 1], np.inf)
        rev = m.p.execute_basket_orders(*one[:4], allowed, limit=lim, kind=one[4])
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.received[0] == 0.0 and not np.any(rev.paid)
        same_state(before, state(m.p))
        ok = m.p.execute_basket_orders(*one[:4], allowed, limit=a.received[r:r + 1], kind=one[4])
        assert ok.status[0] == 0 and ok.received[0] == a.received[r]
        # signed limits on a row that pays on net (it only buys, on two pools that agree on prices):
        # −inf and a limit at or below the net fill, a limit above it reverts and changes nothing
        tiny = cr.DevicePools(3, device=0)
        try:
            tiny.add_product(np.array([[1000.0, 1000.0], [1000.0, 1000.0]]), np.full(2, 0.997),
                             np.array([[1, 2], [2, 3]], np.int64))
            tiny.finalize()
            pay = ([1], [0, 1], [3], [2.0])
            via2 = np.array([0, 1, 0], bool)
            for lim in (-np.inf, None, "equal"):
                qp = tiny.quote_basket_orders(*pay, via2, kind=OUT)
                assert qp.status[0] == 0 and qp.received[0] < -2.0
                if lim is None:
                    before = tiny.pool_state(0)[0]
                    rev = tiny.execute_basket_orders(*pay, via2, limit=np.nextafter(qp.received, np.inf), kind=OUT)
                    assert rev.status[0] == cr._lib.ORDER_LIMIT and not np.any(rev.leg_delta)
                    assert np.array_equal(before, tiny.pool_state(0)[0])
                    continue
                ex = tiny.execute_basket_orders(*pay, via2, limit=qp.received if lim == "equal" else [lim], kind=OUT)
                assert ex.status[0] == 0 and ex.received[0] == qp.received[0] and ex.paid[0] <= -2.0
        finally:
            tiny.close()
        # launches: with an empty mask, sell-only and buy rows on disjoint tokens are one level of two
        # launches; rows sharing a token take one level each (rows that cannot converge trade nothing,
        # so the bookkeeping after the levels is the same in every call)
        none = np.zeros(N, bool)
        stop = {"max_iter": 1, "rtol": 1e-12}
        dis = (np.array([1, 4, 7], np.int64), np.array([0, 2, 4, 6], np.int64),
               np.array([2, 3, 5, 6, 8, 9], np.int64), np.full(6, 3.0), np.array([0, 0, 0, 1, 1, 0], np.uint8))
        n0 = m.p.launch_count
        m.p.execute_basket_orders(*dis[:4], none, kind=dis[4], opts=stop)
        n_dis = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_basket_orders(dis[0][1:2], [0, 2], dis[2][2:4], dis[3][2:4], none, kind=dis[4][2:4], opts=stop)
        n_one = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_basket_orders(np.array([1, 4], np.int64), np.array([0, 2, 4], np.int64),
                                  np.array([2, 3, 5, 3], np.int64), np.full(4, 3.0), none,
                                  kind=np.array([0, 1, 0, 1], np.uint8), opts=stop)
        n_two = m.p.launch_count - n0
        assert n_dis == n_one + 1 and n_two == n_one + 1, (n_dis, n_one, n_two)
        n0 = m.p.launch_count
        m.p.quote_basket_orders(*dis[:4], none, kind=dis[4])
        n_q = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.quote_basket_orders(*dis[:4], none)
        assert n_q == m.p.launch_count - n0 + 1
    finally:
        m.close()


def test_edge_rows(mk_plain):
    p, m = mk_plain
    lists = pair_lists(p)
    none = np.zeros(N, bool)
    before = state(p)
    # a bought token outside T (an empty mask: T is the settlement token and the entries joined to it)
    live = {ab for ab, l in lists.items() if any(x for _, _, x in l)}
    link = lambda u, v: (min(u, v), max(u, v)) in live  # noqa: E731
    i, s, t = next((i, s, t) for i in range(1, N + 1) for s in range(1, N + 1) for t in range(1, N + 1)
                   if len({i, s, t}) == 3 and link(i, s) and not link(i, t) and not link(s, t))
    no = p.quote_basket_orders([i], [0, 2], [s, t], [1.0, 1.0], none, kind=[0, OUT])
    assert no.status[0] == UNREACH and no.solver_status[0] == -1
    # ... with y = 0 it is dropped from the row's tokens
    z = p.quote_basket_orders([i], [0, 2], [s, t], [1.0, 0.0], none, kind=[0, OUT])
    assert z.token.tolist() == [i, s] and z.status[0] in (0, NC)
    # y at or above what the row's pools holding the bought token can pay out (C by the stated rule:
    # the reserves of the bought token, summed in the row's pool order as the kernel adds them)
    a, b = next(ab for ab, l in lists.items() if len(l) >= 2 and all(x for _, _, x in l) and all(t == 0 for t, _, _ in l))
    one = p.quote_basket_orders([a], [0, 1], [b], [1.0], none, kind=OUT)
    cap = capacity([float(p.pool_state(0, k, 1)[0][0][0 if m.Ai[0][k][0] == b else 1]) for k in one.leg_pool])
    at = p.quote_basket_orders([a, a, a], [0, 1, 2, 3], [b, b, b], [cap, 2 * cap, np.nextafter(cap, 0.0)], none,
                               kind=OUT)
    assert at.status[0] == UNREACH and at.status[1] == UNREACH and at.status[2] != UNREACH
    # all-zero rows fill with zeros and run no solve; a zero sold entry beside a buy changes nothing
    zz = p.quote_basket_orders([a], [0, 1], [b], [0.0], none, kind=OUT)
    assert zz.status[0] == 0 and zz.solver_status[0] == -1 and zz.received[0] == 0.0 and not np.any(zz.paid)
    for r in range(3):
        if at.status[r] != 0:
            check_not_filled(at, r)
    same_state(before, state(p))


def test_unservable_buy_is_not_converged():
    # token 1 is deep in its pool with token 3, but 3 reaches the settlement token 2 only through a thin
    # pool: y < C, and no payment in 2 buys y
    p = cr.DevicePools(4, device=0)
    try:
        R = np.array([[1000.0, 1000.0], [1e-6, 1e-6], [50.0, 60.0]])
        p.add_product(R, np.full(3, 0.997), np.array([[1, 3], [3, 2], [3, 4]], np.int64))
        p.finalize()
        allowed = np.array([0, 0, 1, 0], bool)
        before = p.pool_state(0)[0]
        out = p.quote_basket_orders([2], [0, 2], [1, 4], [10.0, 1.0], allowed, kind=[OUT, 0])
        assert out.token.tolist() == [1, 2, 4, 3]
        assert out.status[0] == NC, (out.status[0], out.solver_status[0], out.merit[0])
        check_not_filled(out, 0)
        ex = p.execute_basket_orders([2], [0, 2], [1, 4], [10.0, 1.0], allowed, kind=[OUT, 0])
        assert ex.status[0] == NC
        assert np.array_equal(before, p.pool_state(0)[0])
    finally:
        p.close()


def test_rejections_change_nothing(mk_plain):
    p, _ = mk_plain
    lib = p._lib
    ip, dp, u8 = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    allowed = np.ones(N, np.uint8)
    before = state(p)

    def call(kind, limit, tout=(1,), off=(0, 2), bt=(2, 3), ba=(1.0, 1.0)):
        tout, off, bt = (np.asarray(x, np.int64) for x in (tout, off, bt))
        ba = np.asarray(ba, np.float64)
        k = None if kind is None else np.asarray(kind, np.uint8)
        lim = None if limit is None else np.asarray(limit, np.float64)
        return lib.cfmm_execute_basket_swap_orders(
            p._ctx, len(tout), tout.ctypes.data_as(ip), off.ctypes.data_as(ip), bt.ctypes.data_as(ip),
            None if k is None else k.ctypes.data_as(u8), ba.ctypes.data_as(dp),
            None if lim is None else lim.ctypes.data_as(dp), allowed.ctypes.data_as(u8), None,
            C.byref(cr._lib.BasketOut()))

    for kind, limit in (([0, 2], None), ([1, 1], [np.nan]), ([0, 1], [np.inf]), ([0, 0], [-1.0]),
                        ([0, 0], [-np.inf]), (None, [-1.0])):
        assert call(kind, limit) == cr._lib.CFMM_ERR_INVALID, (kind, limit)
    # the basket calls' own errors apply too
    assert call([0, 1], None, bt=(2, 2)) == cr._lib.CFMM_ERR_INVALID
    assert call([0, 1], None, bt=(2, 1)) == cr._lib.CFMM_ERR_INVALID
    assert call([0, 1], None, ba=(1.0, -1.0)) == cr._lib.CFMM_ERR_INVALID
    same_state(before, state(p))
    # the basket calls still reject negative limits
    with pytest.raises(cr.CFMMError):
        p.execute_basket_orders([1], [0, 1], [2], [1.0], np.ones(N, bool), limit=[-1.0])
    same_state(before, state(p))


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 21)
    try:
        n = 12
        allowed = np.zeros(n, bool)
        allowed[:6] = True
        tout = np.array([11, 12, 7])
        sells = [{7: 5.0, 8: 2.0}, ([9], [20.0]), {}]
        buys = [{9: 0.5}, ([10], [0.2]), {8: 0.3}]
        sold, bought, net, st, det = r.quote_basket_swap_orders(tout, sells, buys, allowed)
        assert [len(x) for x in sold] == [2, 1, 0] and [len(x) for x in bought] == [1, 1, 1]
        reach = st != UNREACH
        assert np.any(reach) and np.all(np.isin(st[reach], (0, NC)))
        want = [list(b.values()) if isinstance(b, dict) else list(b[1]) for b in buys]
        for k in np.flatnonzero(st == 0):
            assert np.all(bought[k] >= want[k]) and np.array_equal(net[k:k + 1], det.received[k:k + 1])
        with pytest.raises(ValueError):
            r.quote_basket_swap_orders(tout, sells, buys, None)
        sold2, bought2, net2, st2, det2 = r.execute_basket_swap_orders(tout, sells, buys, allowed,
                                                                       limits=np.full(len(tout), -np.inf))
        assert np.any(st2 == 0)
        for k in np.flatnonzero(st2 == 0):
            sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
            for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
                dev, _ = r._pools.pool_state(int(t), int(i), 1)
                c = r.cfmms[r._type_lists[int(t)][int(i)]]
                assert np.array_equal(np.asarray(c.R), dev[0])
    finally:
        r.close() if hasattr(r, "close") else None
