"""cfmm_quote_limit_orders / cfmm_execute_limit_orders (include/cfmm_b200.h) on the device.

On the five markets of test_gpu_subgraph_orders: zero limits give basket rows bit for bit (quote,
execute and the final state); limit rows list the basket rows' tokens and pools, their legs equal a
materialising cfmm_sweep at the row's ν and their Ψ the warp-tree sums; every filled row keeps the fill
promise (paid, intermediates, surplus floor) and the complementary-slackness reading.  On one pool
with an empty mask: paid is prod_arb_δ (ProductTwoCoin) or the oracle's find_arb! (UniV3) at the
row's ν, in both tender directions.  On the plain market: filled rows with K = 1, 2, 4, 16 pass the
50-digit certificate.  Over a ladder of limits paid does not increase and the average rate does not
fall; a limit above every pool's rate fills with zeros.  With every token allowed a row agrees with
cfmm_solve and the host route(LimitBasket).  Executes: a partially filled row leaves the pools at its
limit, a batch equals row-by-row executes, disjoint rows share a launch, min_received reverts (an equal
value fills), and quotes and rejected calls change no state."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import basket_oracle as bo
import limit_order_oracle as lo
import order_certificate as oc
import solve_certificate as sc
from test_gpu_basket_orders import baskets
from test_gpu_subgraph_orders import (N, RTOL, STATES, Market, fields, fresh, global_index, mask, row_slices,
                                      same_state, state)

pytestmark = pytest.mark.gpu


def limits_around(p, tout, off, bt, ba, allowed, rng, factors=(0.98, 1.0, 1.02)):
    """Limits drawn around each entry's marginal rate in i at the start (ν_k/ν_i of the same rows
    quoted as basket rows at a millionth of their amounts), times one of `factors`."""
    tiny = p.quote_basket_orders(tout, off, bt, ba * 1e-6, allowed)
    c = np.zeros(len(bt))
    for r in range(len(tout)):
        ts, _ = row_slices(tiny, r)
        loc = {int(t): k for k, t in enumerate(tiny.token[ts])}
        nu = tiny.nu[ts]
        for k in range(off[r], off[r + 1]):
            if int(bt[k]) in loc and tiny.status[r] == 0 and nu[0] > 0:
                c[k] = nu[loc[int(bt[k])]] / nu[0] * rng.choice(factors)
    return c


def check_fill(out, r, bt, ba, c):
    """The header's promise for filled row r: paid within δ + rtol·V/ν_k, intermediates at least
    −rtol·V/ν_b, the surplus in its operation order and above its floor, and the complementary-
    slackness reading within the stop's tolerance.  Returns the number of partially filled entries."""
    ts, _ = row_slices(out, r)
    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
    paid = out.paid[out.basket_off[r]:out.basket_off[r + 1]]
    assert out.surplus[r] == lo.surplus(out.received[r], paid, c)
    floor, V = lo.surplus_floor(toks.tolist(), bt, ba, c, nu, psi, RTOL)
    assert out.surplus[r] >= floor * (1 + 1e-9), (out.surplus[r], floor)
    lower = lo.box(toks.tolist(), bt, c)
    loc = {int(t): k for k, t in enumerate(toks)}
    tol = RTOL * V / nu * (1 + 1e-9)
    ent = set()
    n_part = 0
    for k, t in enumerate(bt):
        if int(t) not in loc:
            assert paid[k] == 0.0
            continue
        j = loc[int(t)]
        ent.add(j)
        assert paid[k] <= ba[k] + tol[j]
        on = nu[j] <= lower[j]
        if not on:                                   # off its limit: sold in full
            assert abs(paid[k] - ba[k]) <= tol[j]
        elif paid[k] < ba[k] - tol[j]:               # partially filled: on its limit
            n_part += 1
    for j in range(1, len(toks)):
        if j not in ent:
            assert psi[j] >= -tol[j]
    return n_part


# ---- zero limits are basket rows ------------------------------------------------------------------
@pytest.mark.parametrize("state_", STATES)
def test_zero_limits_are_basket_rows(state_):
    m1, m2 = Market(state_), Market(state_)
    try:
        rng = np.random.default_rng(1)
        for k in (0, 3, 10):
            allowed = mask(rng, k)
            tout, off, bt, ba = baskets(rng, 10, 5)
            zero = np.zeros(len(bt))
            a = m1.p.quote_basket_orders(tout, off, bt, ba, allowed)
            b = m1.p.quote_limit_orders(tout, off, bt, ba, zero, allowed)
            for x, y in zip(fields(a), fields(b)):
                assert np.array_equal(x, y)
            assert np.array_equal(b.surplus, b.received)   # 0·paid subtracted
            a = m1.p.execute_basket_orders(tout, off, bt, ba, allowed)
            b = m2.p.execute_limit_orders(tout, off, bt, ba, zero, allowed)
            for x, y in zip(fields(a), fields(b)):
                assert np.array_equal(x, y)
            same_state(state(m1.p), state(m2.p))
    finally:
        m1.close()
        m2.close()


# ---- lists, legs, sums and the fill promise on every state --------------------------------------
@pytest.mark.parametrize("state_", STATES)
def test_lists_legs_and_fill_promise_on_every_state(state_):
    m = Market(state_)
    try:
        p = m.p
        rng = np.random.default_rng(2)
        n_filled = n_part = 0
        for k in (0, 3, 6, 10):
            allowed = mask(rng, k)
            tout, off, bt, ba = baskets(rng, 10, 5)
            c = limits_around(p, tout, off, bt, ba, allowed, rng)
            base = p.quote_basket_orders(tout, off, bt, ba, allowed)
            out = p.quote_limit_orders(tout, off, bt, ba, c, allowed)
            assert np.array_equal(out.tok_off, base.tok_off) and np.array_equal(out.token, base.token)
            assert np.array_equal(out.leg_off, base.leg_off) and np.array_equal(out.leg_type, base.leg_type)
            assert np.array_equal(out.leg_pool, base.leg_pool)
            for r in range(len(tout)):
                sl = slice(off[r], off[r + 1])
                if out.status[r] == 0 and out.solver_status[r] == 0:
                    # the legs, Ψ and paid of basket_oracle, at the limit row's box
                    ts, _ = row_slices(out, r)
                    toks, nu, psi = out.token[ts], out.nu[ts], out.psi[ts]
                    v = np.ones(N)
                    v[toks - 1] = nu
                    p.sweep(v, materialize=True)
                    D, L = p.trades()
                    _, lsl = row_slices(out, r)
                    g = np.array([global_index(int(t), int(i)) for t, i in zip(out.leg_type[lsl], out.leg_pool[lsl])],
                                 np.int64)
                    assert np.array_equal(D[g], out.leg_delta[lsl]) and np.array_equal(L[g], out.leg_lambda[lsl])
                    A = bo.ingest_tokens(m.Ai, out.leg_type[lsl], out.leg_pool[lsl])
                    assert np.array_equal(bo.warp_psi(A, out.leg_delta[lsl], out.leg_lambda[lsl], toks), psi)
                    assert out.received[r] == psi[0] and out.merit[r] <= RTOL
                    n_part += check_fill(out, r, bt[sl], ba[sl], c[sl])
                    n_filled += 1
                elif out.status[r] == 0:
                    assert out.solver_status[r] == -1 and out.received[r] == 0.0 and out.surplus[r] == 0.0
                else:
                    assert out.status[r] in (cr._lib.ORDER_UNREACHABLE, cr._lib.ORDER_NOT_CONVERGED)
                    assert out.received[r] == 0.0 and not np.any(out.paid[sl]) and out.surplus[r] == 0.0
        assert n_filled >= 15 and n_part >= 1, (n_filled, n_part)
    finally:
        m.close()


# ---- known answers on one pool, empty mask --------------------------------------------------------
def one_pool(kind, rng):
    p = cr.DevicePools(2, device=0)
    if kind == "product":
        R = np.array([[rng.uniform(500, 2000), rng.uniform(500, 2000)]])
        p.add_product(R, np.array([0.997]), np.array([[1, 2]], np.int64))
        spec = R[0]
    else:
        u = synth.univ3_pools(1, 2, seed=int(rng.integers(1 << 30)))
        u = (u[0], u[1], np.array([[1, 2]], np.int64)) + tuple(u[3:])
        p.add_univ3(*u)
        spec = u
    p.finalize()
    return p, spec


@pytest.mark.parametrize("kind", ["product", "univ3"])
def test_known_answers_on_one_pool(kind, oracle):
    rng = np.random.default_rng(17)
    none = np.zeros(2, bool)
    n_part = 0
    for trial in range(8):
        p, spec = one_pool(kind, rng)
        try:
            for i, j in ((1, 2), (2, 1)):       # both tender directions
                rate = p.quote_limit_orders([i], [0, 1], [j], [1e-6], [0.0], none)
                nu0 = rate.nu
                mrate = nu0[1] / nu0[0]
                d = float(rng.uniform(5, 60))
                c = mrate * float(rng.choice([0.9, 0.97, 0.99, 1.01]))
                out = p.quote_limit_orders([i], [0, 1], [j], [d], [c], none)
                assert out.status[0] == 0
                nu = out.nu
                V = d * nu[1]
                tol = RTOL * V / nu[1] * (1 + 1e-9)
                paid = out.paid[0]
                if kind == "product":
                    Ri, Rj = (spec[0], spec[1]) if i == 1 else (spec[1], spec[0])
                    g = 0.997

                    def arb(ratio):   # prod_arb_δ: the tender of j at ν_j/ν_i = ratio
                        return max(np.sqrt(g * Rj * Ri / ratio) - Rj, 0.0) / g
                    assert abs(paid - min(d, arb(nu[1] / nu[0]))) <= tol + 1e-12 * d
                    if c > mrate:                     # above the pool's rate: at most the stop's tolerance
                        assert paid <= tol
                    elif paid < d - tol:
                        n_part += 1
                        assert abs(paid - arb(c)) <= tol + 1e-9 * d
                else:
                    v = np.zeros(2)
                    v[i - 1], v[j - 1] = nu[0], nu[1]
                    D, L = oracle.sweep_univ3(*spec, v)
                    want = D[0, j - 1]
                    assert abs(paid - min(d, want)) <= tol + 1e-9 * max(d, 1.0)
                    if paid < d - tol:
                        n_part += 1
                        assert nu[1] <= max(c, lo.SQRT_EPS)
        finally:
            p.close()
    assert n_part >= 2


# ---- the 50-digit certificate, K = 1, 2, 4, 16 ---------------------------------------------------------
@pytest.fixture(scope="module")
def mk_plain():
    m = Market()
    yield m.p, m
    m.close()


def test_certificate_k_1_to_16(mk_plain):
    p, m = mk_plain
    rng = np.random.default_rng(7)
    done = {}
    for K in (1, 2, 4, 16):
        allowed = mask(rng, 3)
        tout, bt = [], []
        for _ in range(4):
            pick = rng.choice(np.arange(1, N + 1), size=K + 1, replace=False)
            tout.append(int(pick[0]))
            bt += pick[1:].tolist()
        tout, bt = np.array(tout, np.int64), np.array(bt, np.int64)
        ba = rng.uniform(1.0, 20.0, size=len(bt))
        off = np.arange(0, len(bt) + 1, K, dtype=np.int64)
        c = limits_around(p, tout, off, bt, ba, allowed, rng)
        out = p.quote_limit_orders(tout, off, bt, ba, c, allowed)
        for r in np.flatnonzero((out.status == 0) & (out.solver_status == 0))[:2]:
            ts, sl = row_slices(out, r)
            toks, nu_r, psi = out.token[ts], out.nu[ts], out.psi[ts]
            pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
            q, order, cert = fresh(m, pools)
            try:
                nu = np.ones(N)
                nu[toks - 1] = nu_r
                D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
                D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
                e = slice(off[r], off[r + 1])
                lin, cc = np.zeros(N), np.zeros(N)
                lin[bt[e] - 1], cc[bt[e] - 1] = ba[e], c[e]
                out_T = np.setdiff1d(np.arange(N), toks - 1)    # tokens outside the row: ν = 1, no flow
                lin[out_T], cc[out_T] = 0.0, 0.0                # (a dropped entry is not in the problem)
                obj = cr.LimitBasket(int(tout[r]), lin, cc)
                ref = cc.copy()
                ref[int(tout[r]) - 1] = 1.0
                lower = obj.lower_limit()
                box = sc.Box(obj.linear_term(), lower, ref=ref)
                V = float(np.sum(lin[toks - 1] * nu_r))
                pgtol = float(np.max(out.merit[r] * V / nu_r)) * (1 + 1e-9)
                res = sc.certify(cert, box, nu, D, L, pgtol=pgtol)
                floor, _ = lo.surplus_floor(toks.tolist(), bt[e], ba[e], c[e], nu_r, psi, RTOL)
                assert res["gap"] <= -floor + res["allowance"], (res, floor)
                done[K] = done.get(K, 0) + 1
            finally:
                q.close()
    assert all(done.get(K, 0) >= 1 for K in (1, 2, 4, 16)), done


# ---- monotone in the limit ---------------------------------------------------------------------------
def ladder_rows(p, i, j, d, ladder, allowed):
    q = len(ladder)
    out = p.quote_limit_orders(np.full(q, i), np.arange(q + 1), np.full(q, j), np.full(q, d), ladder, allowed)
    V = d * out.nu[out.tok_off[:-1] + 1]
    return out, np.diff(out.tok_off) * RTOL * V     # |T|·rtol·V per row


def test_monotone_in_the_limit(mk_plain):
    """Paid does not increase along a ladder of limits (S*(c) is convex in c with slope Ψ_k), on the
    market with its cycles; on one pool, where the received is a concave function of the amount sold,
    the average rate does not fall either, and a limit above the pool's rate sells at most the stop's
    tolerance.  Both within the rows' certified gaps (twice them for the rate: a row may sit its gap
    below the frontier, or above it by the intermediates it may owe)."""
    p, _ = mk_plain
    rng = np.random.default_rng(9)
    n_rows = 0
    for _ in range(16):
        allowed = mask(rng, 4)
        i, j = (int(x) for x in rng.choice(np.arange(1, N + 1), size=2, replace=False))
        d = float(rng.uniform(5, 20))
        rate = limits_around(p, np.array([i]), np.array([0, 1]), np.array([j]), np.array([d]), allowed, rng, (1.0,))
        if not rate[0] > 0:
            continue
        ladder = rate[0] * np.linspace(0.6, 1.05, 10)
        out, gap = ladder_rows(p, i, j, d, ladder, allowed)
        if not np.all((out.status == 0) & (out.solver_status == 0)):
            continue
        n_rows += 1
        for a in range(len(ladder) - 1):
            assert out.paid[a + 1] <= out.paid[a] + (gap[a] + gap[a + 1]) / ladder[a]
    assert n_rows >= 1
    rng = np.random.default_rng(19)
    for _ in range(4):
        q1, _ = one_pool("product", rng)
        try:
            none = np.zeros(2, bool)
            rate = q1.quote_limit_orders([1], [0, 1], [2], [1e-6], [0.0], none).nu
            ladder = rate[1] / rate[0] * np.linspace(0.7, 1.05, 12)
            out, gap = ladder_rows(q1, 1, 2, float(rng.uniform(50, 200)), ladder, none)
            assert np.all(out.status == 0)
            for a in range(len(ladder) - 1):
                b = a + 1
                assert out.paid[b] <= out.paid[a] + (gap[a] + gap[b]) / ladder[a]
                if out.paid[b] > 1e-3 * out.paid[0]:
                    ra, rb = out.received[a] / out.paid[a], out.received[b] / out.paid[b]
                    assert rb >= ra - 2 * (gap[a] + gap[b]) / out.paid[b]
            assert out.paid[-1] <= gap[-1] / ladder[-1]
        finally:
            q1.close()


# ---- every token allowed: the row, cfmm_solve and the host route() ----------------------------------
def test_whole_set_agrees_with_cfmm_solve_and_route():
    n = 8
    rng = np.random.default_rng(43)
    R, g, A = synth.product_pools(40, n, seed=44)
    spec = list(zip(R, g, A))
    cert = [oc.product(Rk, gk, Ak) for Rk, gk, Ak in spec]
    p = cr.DevicePools(n, device=0)
    p.add_product(R, g, A)
    p.finalize()
    try:
        i, bt = 1, np.array([3, 5, 6], np.int64)
        ba = np.array([8.0, 15.0, 4.0])
        allowed = np.ones(n, bool)
        c = limits_around(p, np.array([i]), np.array([0, 3]), bt, ba, allowed, rng, (0.97, 1.0, 1.01))
        out = p.quote_limit_orders([i], [0, 3], bt, ba, c, allowed)
        assert out.status[0] == 0
        d, cc = np.zeros(n), np.zeros(n)
        d[bt - 1], cc[bt - 1] = ba, c
        obj = cr.LimitBasket(i, d, cc)
        const = float(d @ cc)
        ref = cc.copy()
        ref[i - 1] = 1.0
        box = sc.Box(obj.linear_term(), obj.lower_limit(), ref=ref)
        toks = out.token
        nu = np.ones(n)
        nu[toks - 1] = out.nu
        V = float(np.sum(d[toks - 1] * out.nu))
        floor, _ = lo.surplus_floor(toks.tolist(), bt, ba, c, out.nu, out.psi, RTOL)
        pgtol = float(np.max(out.merit[0] * V / out.nu)) * (1 + 1e-9)
        rd = sc.certify(cert, box, nu, out.leg_delta, out.leg_lambda, pgtol=pgtol)
        xs, info = p.solve(lower=obj.lower_limit(), lin=obj.linear_term())
        Ds, Ls = p.trades()
        rs = sc.certify(cert, box, xs, Ds, Ls, check_stop=False)
        r = cr.Router(obj, [cr.ProductTwoCoin(*s) for s in spec], n)
        cr.route(r)
        rh = sc.certify(cert, box, r.v, r.Δs, r.Λs, check_stop=False)
        for other in (rs, rh):
            slack = abs(rd["gap"]) + rd["allowance"] + abs(other["gap"]) + other["allowance"]
            assert abs((rd["g50"] - const) - (other["g50"] - const)) <= slack + 1e-9 * abs(rd["g50"]), (rd, other)
        # the surplus is the dual value (constant included) within the row's certified gap
        assert abs(out.surplus[0] - (rd["g50"] - const)) <= abs(rd["gap"]) + rd["allowance"] + 1e-9 * V
        assert out.surplus[0] >= floor
    finally:
        p.close()


# ---- execute -----------------------------------------------------------------------------------------
def test_execute_leaves_the_pools_at_the_limit_and_batches_row_by_row():
    rng = np.random.default_rng(5)
    m = Market()
    try:
        p = m.p
        n_part = 0
        for _ in range(12):
            allowed = mask(rng, 3)
            i, j = (int(x) for x in rng.choice(np.arange(1, N + 1), size=2, replace=False))
            d = float(rng.uniform(50, 500))
            # a limit halfway between the marginal rate before and after selling all of d
            r0 = limits_around(p, np.array([i]), np.array([0, 1]), np.array([j]), np.array([d]), allowed, rng, (1.0,))
            full = p.quote_limit_orders([i], [0, 1], [j], [d], [0.0], allowed)
            if full.status[0] != 0 or full.solver_status[0] != 0 or len(full.nu) < 2 or full.token[1] != j:
                continue
            r1 = full.nu[1] / full.nu[0]
            if not r0[0] > r1 * (1 + 1e-3):
                continue
            c = np.array([0.5 * (r0[0] + r1)])
            out = p.execute_limit_orders([i], [0, 1], [j], [d], c, allowed)
            if out.status[0] != 0 or out.solver_status[0] != 0 or not (0.01 * d < out.paid[0] < d * (1 - 1e-3)):
                continue
            n_part += 1
            V = d * out.nu[1]
            again = p.quote_limit_orders([i], [0, 1], [j], [d], c, allowed)
            assert again.status[0] == 0
            assert again.paid[0] <= RTOL * V / again.nu[1] * (1 + 1e-9) + RTOL * V / out.nu[1], (again.paid, V)
        assert n_part >= 2
    finally:
        m.close()
    allowed = mask(rng, 5)
    tout, off, bt, ba = baskets(rng, 6, 4)
    m1, m2 = Market(), Market()
    try:
        c = limits_around(m1.p, tout, off, bt, ba, allowed, rng)
        batch = m1.p.execute_limit_orders(tout, off, bt, ba, c, allowed)
        for r in range(len(tout)):
            e = slice(off[r], off[r + 1])
            o1 = np.array([0, off[r + 1] - off[r]], np.int64)
            one = m2.p.execute_limit_orders(tout[r:r + 1], o1, bt[e], ba[e], c[e], allowed)
            ts, sl = row_slices(batch, r)
            assert batch.received[r] == one.received[0] and batch.status[r] == one.status[0]
            assert batch.surplus[r] == one.surplus[0] and np.array_equal(batch.paid[e], one.paid)
            assert np.array_equal(batch.leg_delta[sl], one.leg_delta) and np.array_equal(batch.nu[ts], one.nu)
        same_state(state(m1.p), state(m2.p))
        assert np.any(batch.status == 0)
    finally:
        m1.close()
        m2.close()


def test_min_received_launches_and_no_state_change(mk_plain):
    p, _ = mk_plain
    rng = np.random.default_rng(6)
    allowed = mask(rng, 5)
    tout, off, bt, ba = baskets(rng, 9, 6)
    c = limits_around(p, tout, off, bt, ba, allowed, rng)
    before = state(p)
    a = p.quote_limit_orders(tout, off, bt, ba, c, allowed)
    b = p.quote_limit_orders(tout, off, bt, ba, c, allowed)
    for x, y in zip(fields(a) + [a.surplus], fields(b) + [b.surplus]):
        assert np.array_equal(x, y)
    same_state(before, state(p))
    m = Market()
    try:
        r = int(np.flatnonzero((a.status == 0) & (a.solver_status == 0) & (a.received > 0))[0])
        e = slice(off[r], off[r + 1])
        args = (tout[r:r + 1], np.array([0, off[r + 1] - off[r]], np.int64), bt[e], ba[e], c[e], allowed)
        before = state(m.p)
        rev = m.p.execute_limit_orders(*args, min_received=np.nextafter(a.received[r:r + 1], np.inf))
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.received[0] == 0.0 and not np.any(rev.paid)
        assert rev.surplus[0] == 0.0
        same_state(before, state(m.p))
        ok = m.p.execute_limit_orders(*args, min_received=a.received[r:r + 1])
        assert ok.status[0] == 0 and ok.received[0] == a.received[r] and ok.surplus[0] == a.surplus[r]
        # rows on disjoint tokens with an empty mask run in one launch; rows sharing a token do not
        none = np.zeros(N, bool)
        lp = np.full(6, 0.01)
        dis = (np.array([1, 4, 7], np.int64), np.array([0, 2, 4, 6], np.int64),
               np.array([2, 3, 5, 6, 8, 9], np.int64), np.full(6, 3.0))
        n0 = m.p.launch_count
        m.p.execute_limit_orders(*dis, lp, none)
        n_dis = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_limit_orders(dis[0][:1], dis[1][:2], dis[2][:2], dis[3][:2], lp[:2], none)
        n_one = m.p.launch_count - n0
        n0 = m.p.launch_count
        m.p.execute_limit_orders(np.array([1, 4], np.int64), np.array([0, 2, 4], np.int64),
                                 np.array([2, 3, 5, 3], np.int64), np.full(4, 3.0), lp[:4], none)
        n_two = m.p.launch_count - n0
        assert n_dis == n_one and n_two == n_one + 1
    finally:
        m.close()


def test_rejections_change_nothing(mk_plain):
    p, _ = mk_plain
    lib = p._lib
    ip, dp, u8 = C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_uint8)
    allowed = np.ones(N, np.uint8)
    before = state(p)

    def call(tout, off, bt, ba, lp, execute=True, minr=None, out=None):
        tout, off, bt = (np.asarray(x, np.int64) for x in (tout, off, bt))
        ba = np.asarray(ba, np.float64)
        lpp = None if lp is None else np.asarray(lp, np.float64).ctypes.data_as(dp)
        o = out or cr._lib.LimitOut()
        if execute:
            mr = None if minr is None else np.asarray(minr, np.float64).ctypes.data_as(dp)
            return lib.cfmm_execute_limit_orders(p._ctx, len(tout), tout.ctypes.data_as(ip), off.ctypes.data_as(ip),
                                                 bt.ctypes.data_as(ip), ba.ctypes.data_as(dp), lpp, mr,
                                                 allowed.ctypes.data_as(u8), None, C.byref(o))
        return lib.cfmm_quote_limit_orders(p._ctx, len(tout), tout.ctypes.data_as(ip), off.ctypes.data_as(ip),
                                           bt.ctypes.data_as(ip), ba.ctypes.data_as(dp), lpp,
                                           allowed.ctypes.data_as(u8), None, C.byref(o))

    assert call([1], [0, 2], [2, 3], [1.0, 1.0], [0.5, 0.5], execute=False) == 0
    bad = [
        ([1], [0, 2], [2, 3], [1.0, 1.0], None),                  # a null limit_price
        ([1], [0, 2], [2, 3], [1.0, 1.0], [0.5, -0.5]),           # a negative limit
        ([1], [0, 2], [2, 3], [1.0, 1.0], [0.5, float("nan")]),
        ([1], [0, 2], [2, 3], [1.0, 1.0], [float("inf"), 0.5]),
        ([1], [0, 2], [2, 2], [1.0, 1.0], [0.5, 0.5]),            # the basket calls' errors
        ([1], [0, 1], [2], [-1.0], [0.5]),
        ([1], [1, 2], [2, 3], [1.0, 1.0], [0.5, 0.5]),
    ]
    for args in bad:
        assert call(*args) == cr._lib.CFMM_ERR_INVALID, args
        assert call(*args, execute=False) == cr._lib.CFMM_ERR_INVALID, args
    assert call([1], [0, 1], [2], [1.0], [0.5], minr=[-1.0]) == cr._lib.CFMM_ERR_INVALID
    assert call([1], [0, 1], [2], [1.0], [0.5], minr=[float("inf")]) == cr._lib.CFMM_ERR_INVALID
    small = cr._lib.LimitOut()
    tokbuf = np.zeros(1, np.int64)
    small.token, small.tok_cap = tokbuf.ctypes.data_as(ip), 1
    assert call([1], [0, 2], [2, 3], [1.0, 1.0], [0.5, 0.5], out=small) == cr._lib.CFMM_ERR_INVALID
    same_state(before, state(p))
    # the surplus alone is an output: it runs the rows
    sur = np.full(1, np.nan)
    o = cr._lib.LimitOut()
    o.surplus = sur.ctypes.data_as(dp)
    assert call([1], [0, 2], [2, 3], [1.0, 1.0], [0.0, 0.0], execute=False, out=o) == 0
    full = p.quote_limit_orders([1], [0, 2], [2, 3], [1.0, 1.0], [0.0, 0.0], allowed.astype(bool))
    assert sur[0] == full.surplus[0] and np.isfinite(sur[0])
    same_state(before, state(p))


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 21)
    try:
        n = 12
        allowed = np.zeros(n, bool)
        allowed[:6] = True
        tout = np.array([11, 12, 7])
        sells = [{7: (5.0, 0.0), 8: (2.0, 0.0)}, ([9, 10], [20.0, 1.0], [0.0, 0.0]), {8: (3.0, 0.0)}]
        sold, recv, sur, st, det = r.quote_limit_orders(tout, sells, allowed)
        bsk = [{7: 5.0, 8: 2.0}, ([9, 10], [20.0, 1.0]), {8: 3.0}]
        paid, recv_b, st_b, _ = r.quote_basket_orders(tout, bsk, allowed)
        assert all(np.array_equal(x, y) for x, y in zip(sold, paid)) and np.array_equal(recv, recv_b)
        assert np.array_equal(st, st_b) and np.array_equal(sur, recv)
        sold2, recv2, sur2, st2, det2 = r.execute_limit_orders(tout, sells, allowed, min_received=np.zeros(3))
        assert np.any(st2 == 0)
        for k in np.flatnonzero(st2 == 0):
            sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
            for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
                dev, _ = r._pools.pool_state(int(t), int(i), 1)
                c = r.cfmms[r._type_lists[int(t)][int(i)]]
                assert np.array_equal(np.asarray(c.R), dev[0])
    finally:
        r.close() if hasattr(r, "close") else None
