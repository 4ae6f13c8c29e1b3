"""cfmm_quote_price_arbitrage_rows / cfmm_execute_price_arbitrage_rows (include/cfmm_b200.h) on the device.

Rows with no holdings and every listed price > 0 equal the one-mask price call with the list as its mask,
bit for bit, on every field, for unsorted lists and on the wide set's 258-token shapes.  On the market
states of test_gpu_subgraph_orders, with price-0 intermediates and holdings: each row lists the oracle's
tokens and pools, its legs equal a materialising cfmm_sweep at its ν bit for bit, its Ψ the warp-tree
sums, and filled rows meet the fill promise and gap bound; on the plain market they pass the 50-digit
certificate.  A one-pool row sells min(h, x*).  A c = e_i row agrees with the basket row and a limit-shaped
row with the limit row's surplus within their gaps.  With atol > 0 a tree row with nothing to do fills
where the one-mask call does not converge.  A batch execute equals one row per call, rows on disjoint
lists share a launch, and an executed row leaves no trade worth more than its stop tolerance.  Every
input error is rejected before anything changes, and the Router refreshes the pools it traded with."""
import ctypes as C

import numpy as np
import pytest

import cfmmrouter_b200 as cr
from cfmmrouter_b200 import synth
import price_arb_rows_oracle as ia
import row_certificate_sets as rc
import solve_certificate as sc
import subgraph_oracle as so
from test_gpu_price_arbitrage import product_context
from test_gpu_subgraph_orders import N, RTOL, Market, fresh, global_index, pair_lists, row_slices, same_state, state

pytestmark = pytest.mark.gpu

NC = cr._lib.ORDER_NOT_CONVERGED
SQRT_EPS = float(np.sqrt(np.finfo(float).eps))
FIELDS = ("profit", "status", "solver_status", "iterations", "fun_evals", "merit")
TOKEN_FIELDS = ("token", "nu", "psi")
LEG_FIELDS = ("leg_type", "leg_pool", "leg_delta", "leg_lambda")


def csr(lists):
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return off, np.concatenate([np.asarray(x, np.int64) for x in lists])


def quote(p, lists, prices, holdings=None, opts=None, execute=False, min_profit=None):
    off, tok = csr(lists)
    pr = np.concatenate([np.asarray(c, float) for c in prices])
    h = None if holdings is None else np.concatenate([np.asarray(x, float) for x in holdings])
    if execute:
        return p.execute_price_arbitrage_rows(off, tok, pr, h, min_profit, opts)
    return p.quote_price_arbitrage_rows(off, tok, pr, h, opts)


def same_row(a, r, b, k):
    """Row r of a equals row k of b on every field."""
    ta, la = row_slices(a, r)
    tb, lb = row_slices(b, k)
    for f in FIELDS:
        x, y = getattr(a, f)[r], getattr(b, f)[k]
        assert x == y or (np.isnan(x) and np.isnan(y)), (f, r, x, y)
    for f in TOKEN_FIELDS:
        assert np.array_equal(getattr(a, f)[ta], getattr(b, f)[tb]), (f, r)
    for f in LEG_FIELDS:
        assert np.array_equal(getattr(a, f)[la], getattr(b, f)[lb]), (f, r)


def random_rows(rng, q, k_lo=4, k_hi=12, zero=0.0, held=0.0, scale=20.0):
    lists, prices, holds = [], [], []
    for _ in range(q):
        k = int(rng.integers(k_lo, k_hi + 1))
        toks = rng.choice(np.arange(1, N + 1), size=k, replace=False)
        c = rng.uniform(0.5, 2.0, k)
        c[rng.random(k) < zero] = 0.0
        c[rng.integers(0, k)] = rng.uniform(0.5, 2.0)
        h = np.where(rng.random(k) < held, rng.uniform(0.0, scale, k), 0.0)
        lists.append(toks.tolist())
        prices.append(c)
        holds.append(h)
    return lists, prices, holds


def local_values(out, r, lists, vals):
    ts, _ = row_slices(out, r)
    return ia.local(lists[r], vals[r], out.token[ts].tolist())


def check_fill(out, r, c, h, cb, rtol=RTOL, atol=0.0):
    """The fill promise of filled row r (c, h in local order; cb the least positive price of its list):
    the stop, the floor Ψ_t >= −h_t − ε/max(ν_t, c̄) (no token overdrawn by more than ε/c̄ units), the
    profit's order and the gap bound.  Returns (P̄, ε)."""
    ts, _ = row_slices(out, r)
    nu, psi = out.nu[ts], out.psi[ts]
    assert out.status[r] == 0 and out.solver_status[r] == 0
    assert np.all(nu >= ia.box(c))
    assert out.profit[r] == ia.profit(c, psi)
    P = ia.pbar(nu, psi, h, c)
    e = ia.eps(P, rtol, atol) * 1.01 + 1e-12 * max(abs(P), 1.0)
    assert out.merit[r] <= rtol or ia.mx(nu, psi, h, c, cb) <= atol * 1.01 + 1e-12, (out.merit[r], r)
    assert np.all(psi >= ia.fill_floor(nu, h, e, cb) - 1e-9 * (np.abs(psi) + h)), r
    assert np.all(np.maximum(-(psi + h), 0.0) <= e / cb * (1 + 1e-9) + 1e-9 * (np.abs(psi) + h)), r
    assert P - out.profit[r] <= ia.gap_bound(nu, psi, h, c, e) + 1e-9 * max(abs(P), 1.0), (P, out.profit[r])
    return P, e


# ---- no holdings: the one-mask price row, bit for bit ---------------------------------------------
def test_no_holdings_equal_the_price_row_on_the_market():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(61)
        lists, prices, _ = random_rows(rng, 8)
        for holds in (None, [np.zeros(len(x)) for x in lists]):
            out = quote(p, lists, prices, holds)
            for r, (lst, c) in enumerate(zip(lists, prices)):
                msk = np.zeros(N, bool)
                msk[np.asarray(lst) - 1] = True
                order = np.argsort(lst)
                one = p.quote_price_arbitrage(np.asarray(c)[order][None, :], msk)
                same_row(out, r, one, 0)
        assert np.any(out.status == 0)
    finally:
        m.close()


def test_no_holdings_equal_the_price_row_on_the_wide_shapes():
    ws = rc.wide_set(cr).build()
    try:
        rng = np.random.default_rng(62)
        opts = {"rtol": 5e-4}
        lists, prices = [], []
        for name, (i, j, B) in rc.shapes(price=True).items():
            toks = sorted({i, j} | set(B))
            c = np.array([ws.nu[t] * np.exp(rng.uniform(-0.05, 0.05)) for t in toks])
            perm = rng.permutation(len(toks))
            lists.append([toks[k] for k in perm])
            prices.append(c[perm])
        assert max(len(x) for x in lists) == 258
        out = quote(ws.p, lists, prices, opts=dict(opts, atol=0.0))
        for r, (lst, c) in enumerate(zip(lists, prices)):
            order = np.argsort(lst)
            one = ws.p.quote_price_arbitrage(c[order][None, :], ws.mask(lst), opts=opts)
            same_row(out, r, one, 0)
        assert np.any(out.status == 0)
    finally:
        ws.p.close()


# ---- lists, legs, sums, fill promise and certificate ------------------------------------------
@pytest.mark.parametrize("state_", ("plain", "retire_after_adjacency"))
def test_lists_legs_sums_and_fill(state_):
    m = Market(state_)
    try:
        p = m.p
        rng = np.random.default_rng(63)
        lists = pair_lists(p)
        rows, prices, holds = random_rows(rng, 12, zero=0.25, held=0.3)
        out = quote(p, rows, prices, holds)
        filled = 0
        for r in range(len(rows)):
            T, pools = ia.row_order(lists, rows[r])
            ts, sl = row_slices(out, r)
            assert out.token[ts].tolist() == T, (r, out.token[ts], T)
            assert list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist())) == sorted(
                pools, key=lambda h: global_index(*h))
            toks, nu = out.token[ts], out.nu[ts]
            v = np.ones(N)
            v[toks - 1] = nu
            p.sweep(v, materialize=True)
            D, L = p.trades()
            g = np.array([global_index(int(t), int(i)) for t, i in zip(out.leg_type[sl], out.leg_pool[sl])], np.int64)
            if out.status[r] == 0:
                filled += 1
                assert np.array_equal(D[g], out.leg_delta[sl]) and np.array_equal(L[g], out.leg_lambda[sl])
                A = so.ingest_tokens(m.Ai, out.leg_type[sl], out.leg_pool[sl])
                assert np.array_equal(so.warp_psi(A, out.leg_delta[sl], out.leg_lambda[sl], toks), out.psi[ts])
                check_fill(out, r, local_values(out, r, rows, prices), local_values(out, r, rows, holds),
                           ia.cbar(prices[r]))
            else:
                assert out.status[r] == NC and out.profit[r] == 0.0 and not np.any(out.leg_delta[sl])
        assert filled >= len(rows) // 2, filled
    finally:
        m.close()


def test_certificate_with_intermediates_and_sold_holdings():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(64)
        rows, prices, holds = random_rows(rng, 8, k_lo=5, k_hi=9, zero=0.3, held=0.5)
        out = quote(p, rows, prices, holds)
        done = sold = inter = 0
        for r in np.flatnonzero(out.status == 0):
            ts, sl = row_slices(out, r)
            if sl.stop == sl.start:
                continue
            c, h = local_values(out, r, rows, prices), local_values(out, r, rows, holds)
            cb = ia.cbar(prices[r])
            P, e = check_fill(out, r, c, h, cb)
            pools = list(zip(out.leg_type[sl].tolist(), out.leg_pool[sl].tolist()))
            q, order, cert = fresh(m, pools)
            q.close()
            D, L = np.zeros((len(cert), 2)), np.zeros((len(cert), 2))
            D[order], L[order] = out.leg_delta[sl], out.leg_lambda[sl]
            toks, nu = out.token[ts], out.nu[ts]
            fc, fh, fnu = np.ones(N), np.zeros(N), np.ones(N) + ia.BOX
            fc[toks - 1], fh[toks - 1], fnu[toks - 1] = c, h, nu
            pgtol = float(np.max(e / ia.scale(nu, cb))) * (1 + 1e-9)  # at most ε/c̄ in token units
            assert pgtol <= e / cb * (1 + 1e-9)
            res = sc.certify(cert, ia.cert_box(fc, fh), fnu, D, L, pgtol=max(pgtol, 1e-300))
            assert res["gap"] <= ia.gap_bound(nu, out.psi[ts], h, c, e) + res["allowance"], res
            sold += bool(np.any((h > 0) & (out.psi[ts] < 0)))
            inter += bool(np.any(c == 0.0))
            done += 1
        assert done >= 3 and sold >= 1 and inter >= 1, (done, sold, inter)
    finally:
        m.close()


# ---- closed form and special cases ----------------------------------------------------------------
@pytest.mark.parametrize("h", [0.0, 0.5, 5.0, 1e6])
def test_one_pool_closed_form(h):
    """A one-pool tree: nothing is self-funding, so the row sells min(h, x*) of the held token (atol
    stops the h = 0 row, whose relative stop is 0 / 0)."""
    R, gam, ca, cb, atol = (1000.0, 1000.0), 0.997, 1.0, 1.02, 1e-6
    p = product_context(2, [(list(R), gam, [1, 2])])
    try:
        out = quote(p, [[2, 1]], [[cb, ca]], [[0.0, h]], opts={"atol": atol})
        assert out.status[0] == 0 and out.token.tolist() == [1, 2]
        sold = -out.psi[0]
        want = ia.product_sold(R, gam, ca, cb, h)
        shifted = ia.product_sold(R, gam, ca + ia.BOX, cb + ia.BOX, h)  # the box's 1e-8 when h does not bind
        P = ia.pbar(out.nu, out.psi, np.array([h, 0.0]), np.array([ca, cb]))
        e = ia.eps(P, RTOL, atol)
        tol = abs(shifted - want) + e / out.nu[0] + 1e-9 * max(want, 1.0)
        assert abs(sold - want) <= tol, (sold, want, tol)
        assert out.psi[1] >= 0.0
        if h == 0.0:
            assert out.profit[0] == 0.0 or abs(out.profit[0]) <= e
    finally:
        p.close()


def agree(a, b, lists, prices, holds):
    """Row 0 of a (an inventory row) and row 0 of b (the basket or limit row of the same problem) agree
    within the sum of their certified gaps.  Each row's certified gap is P̄ − cᵀΨ (its dual bound
    P̄ = νᵀΨ + hᵀ(ν − c) less its value) plus its overdraft Σ_t ν̂_t·max(−Ψ_t − h_t, 0), ν̂ the larger
    of the two rows' ν: by weak duality cᵀΨ_a <= P̄_b + Σ_t (ν_b − c)_t·overdraft_a,t, so
    |cᵀΨ_a − cᵀΨ_b| <= gap_a + gap_b.  The inventory row also meets its fill promise, and the two gaps
    together stay below 1 % of the value, so the agreement is tight.  Returns False (nothing compared)
    when either did not fill or their token sets differ."""
    ta, _ = row_slices(a, 0)
    tb, _ = row_slices(b, 0)
    if a.status[0] != 0 or b.status[0] != 0 or sorted(a.token[ta].tolist()) != sorted(b.token[tb].tolist()):
        return False
    check_fill(a, 0, local_values(a, 0, lists, prices), local_values(a, 0, lists, holds), ia.cbar(prices[0]))
    rows = []
    for o, t in ((a, ta), (b, tb)):
        order = np.argsort(o.token[t])  # both in token order
        tok = o.token[t][order].tolist()
        c, h = ia.local(lists[0], prices[0], tok), ia.local(lists[0], holds[0], tok)
        nu, psi = o.nu[t][order], o.psi[t][order]
        rows.append((c, h, nu, psi, ia.pbar(nu, psi, h, c), ia.profit(c, psi)))
    nu_hat = np.maximum(rows[0][2], rows[1][2])
    gaps = [max(P - v, 0.0) + float(np.sum(nu_hat * np.maximum(-(psi + h), 0.0))) for c, h, nu, psi, P, v in rows]
    va, vb = rows[0][5], rows[1][5]
    rounding = 1e-12 * float(sum(np.sum(nu_hat * np.abs(r[3])) for r in rows)) + 1e-9 * max(abs(vb), 1.0)
    assert abs(va - vb) <= gaps[0] + gaps[1] + rounding, (va, vb, gaps)
    assert gaps[0] + gaps[1] <= 1e-2 * max(abs(vb), 1.0), (va, vb, gaps)
    return True


def test_basket_and_limit_shaped_rows():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(65)
        done_b = done_l = 0
        for _ in range(8):
            toks = rng.choice(np.arange(1, N + 1), size=8, replace=False).tolist()
            i, ents = toks[0], toks[1:4]
            amt = rng.uniform(1.0, 10.0, 3)
            h = np.zeros(8)
            h[1:4] = amt
            # c = e_i, h = Δin: the basket row's received
            c = np.zeros(8)
            c[0] = 1.0
            inv = quote(p, [toks], [c], [h])
            bk = p.quote_basket_orders([i], [0, 3], ents, amt, [toks])
            if agree(inv, bk, [toks], [c], [h]):
                assert inv.profit[0] == ia.profit(local_values(inv, 0, [toks], [c]), inv.psi)
                done_b += 1
            # c = (1 at i, limit_k at the entries), h = Δin: the limit row's surplus
            c2 = np.zeros(8)
            c2[0] = 1.0
            c2[1:4] = rng.uniform(0.5, 1.0, 3)
            inv = quote(p, [toks], [c2], [h])
            lo = p.quote_limit_orders([i], [0, 3], ents, amt, c2[1:4], [toks])
            if agree(inv, lo, [toks], [c2], [h]):
                assert abs(lo.surplus[0] - lo.received[0] - float(c2[1:4] @ -lo.paid)) <= 1e-9 * (1 + abs(lo.received[0]))
                done_l += 1
        assert done_b >= 2 and done_l >= 2, (done_b, done_l)
    finally:
        m.close()


# ---- no opportunity: the absolute stop ----------------------------------------------------------
def test_atol_stops_a_tree_row_with_nothing_to_do():
    """Stars of seven pools around token 1 whose prices disagree with the outside prices (as the headline
    set's): a tree has no self-funding arbitrage, so a row without holdings has nothing to do.  The
    one-mask call's relative stop is 0 / 0 there; with atol > 0 the row fills with a profit within
    |T|·atol of 0."""
    rng = np.random.default_rng(70)
    atol, nc = 1e-3, 0
    for _ in range(6):
        spec = [([1000.0, 1000.0 * float(np.exp(rng.uniform(-1.5, 1.5)))], 0.997, [1, k]) for k in range(2, 9)]
        c = np.exp(rng.uniform(-0.02, 0.02, 8))
        p = product_context(8, spec)
        try:
            one = p.quote_price_arbitrage(c[None, :], np.ones(8, bool))
            perm = rng.permutation(8)
            out = quote(p, [(perm + 1).tolist()], [c[perm]], opts={"atol": atol})
            assert out.status[0] == 0 and out.solver_status[0] == 0, (out.solver_status[0], out.merit[0])
            assert abs(out.profit[0]) <= 8 * atol, out.profit[0]
            assert ia.mx(out.nu, out.psi, np.zeros(8), c, ia.cbar(c)) <= atol * 1.01 or out.merit[0] <= RTOL
            if one.status[0] == NC:
                # the same row without atol (every price > 0, nothing held: the one-mask call's operations)
                # spends more evaluations and ends unfilled
                nc += 1
                assert out.fun_evals[0] < one.fun_evals[0], (out.fun_evals[0], one.fun_evals[0])
            # with a holding the same tree has trades: sell the held token into pools that pay more
            h = np.zeros(8)
            h[1:] = 50.0
            out = quote(p, [(perm + 1).tolist()], [c[perm]], [h[perm]], opts={"atol": atol})
            assert out.status[0] == 0 and out.profit[0] > 0.0
            check_fill(out, 0, c, h, ia.cbar(c), atol=atol)
        finally:
            p.close()
    assert nc >= 1, nc


# ---- execute --------------------------------------------------------------------------------------
def test_batch_equals_sequence_and_leaves_no_trade():
    rng = np.random.default_rng(66)
    rows, prices, holds = random_rows(rng, 6, zero=0.2, held=0.4)
    m1, m2 = Market(), Market()
    try:
        batch = quote(m1.p, rows, prices, holds, execute=True)
        for r in range(len(rows)):
            one = quote(m2.p, rows[r:r + 1], prices[r:r + 1], holds[r:r + 1], execute=True)
            same_row(batch, r, one, 0)
        same_state(state(m1.p), state(m2.p))
        assert np.any(batch.status == 0)
        # the last filled row: no pool of it trades at its ν beyond the stop's tolerance
        r = int(np.flatnonzero(batch.status == 0)[-1])
        later = [k for k in range(r + 1, len(rows)) if set(rows[k]) & set(rows[r])]
        if not later:
            ts, sl = row_slices(batch, r)
            c, h = local_values(batch, r, rows, prices), local_values(batch, r, rows, holds)
            P, e = check_fill(batch, r, c, h, ia.cbar(prices[r]))
            v = np.ones(N)
            v[batch.token[ts] - 1] = batch.nu[ts]
            m1.p.sweep(v, materialize=True)
            D, L = m1.p.trades()
            gi = np.array([global_index(int(t), int(i)) for t, i in zip(batch.leg_type[sl], batch.leg_pool[sl])],
                          np.int64)
            A = np.asarray(so.ingest_tokens(m1.Ai, batch.leg_type[sl], batch.leg_pool[sl]), np.int64)
            after = float(np.sum(v[A - 1] * (L[gi] - D[gi])))
            assert abs(after) <= len(c) * e + 1e-9 * max(P, 1.0), (after, e)
    finally:
        m1.close()
        m2.close()


def test_disjoint_lists_share_a_launch():
    n = 10
    spec = list(zip(*synth.product_pools(200, n, seed=46)))
    rng = np.random.default_rng(67)
    a, b = [1, 2, 3, 4, 5], [6, 7, 8, 9, 10]
    ca, cb = rng.uniform(0.5, 2.0, 5), rng.uniform(0.5, 2.0, 5)
    ha, hb = np.r_[3.0, np.zeros(4)], np.r_[0.0, 2.0, np.zeros(3)]
    launches, outs, states = [], [], []
    for lists, prices, holds in (([a], [ca], [ha]), ([a, b], [ca, cb], [ha, hb]), ([a, a], [ca, ca * 1.1], [ha, ha])):
        p = product_context(n, spec)
        try:
            n0 = p.launch_count
            outs.append(quote(p, lists, prices, holds, execute=True))
            launches.append(p.launch_count - n0)
            states.append(state(p))
        finally:
            p.close()
    assert np.all(outs[1].status == 0) and outs[2].status[0] == 0
    assert launches[1] == launches[0] and launches[2] == launches[0] + 1, launches
    p = product_context(n, spec)
    try:
        ea = quote(p, [a], [ca], [ha], execute=True)
        eb = quote(p, [b], [cb], [hb], execute=True)
        same_row(outs[1], 0, ea, 0)
        same_row(outs[1], 1, eb, 0)
        same_state(states[1], state(p))
    finally:
        p.close()


def test_min_profit_and_rejections_change_nothing():
    m = Market("plain")
    try:
        p = m.p
        rng = np.random.default_rng(68)
        rows, prices, holds = random_rows(rng, 3, held=0.4)
        before = state(p)
        a = quote(p, rows, prices, holds)
        b = quote(p, rows, prices, holds)
        for r in range(3):
            same_row(a, r, b, r)
        same_state(before, state(p))
        r = int(np.flatnonzero((a.status == 0) & (a.profit > 0))[0])
        one = (rows[r:r + 1], prices[r:r + 1], holds[r:r + 1])
        rev = quote(p, *one, execute=True, min_profit=np.nextafter(a.profit[r], np.inf))
        assert rev.status[0] == cr._lib.ORDER_LIMIT and rev.profit[0] == 0.0 and not np.any(rev.leg_delta)
        same_state(before, state(p))
        ok = quote(p, *one, execute=True, min_profit=a.profit[r])
        assert ok.status[0] == 0 and ok.profit[0] == a.profit[r]
        after = state(p)
        lib, ctx = p._lib, p._ctx
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int64)

        def arr(x, t):
            return None if x is None else np.ascontiguousarray(x, dtype=t).ctypes.data_as(dp if t == float else ip)

        good = dict(q=1, off=[0, 3], tok=[1, 2, 3], pr=[1.0, 0.0, 2.0], h=[0.0, 1.0, 0.0], mp=None, opts=None)
        bad = [dict(q=-1), dict(off=None), dict(tok=None), dict(pr=None), dict(off=[0, 0]),
               dict(off=[1, 3]), dict(q=1, off=[0, 259], tok=list(range(1, 260)), pr=[1.0] * 259, h=None),
               dict(tok=[1, 2, N + 1]), dict(tok=[0, 2, 3]), dict(tok=[1, 2, 1]), dict(pr=[1.0, -1.0, 2.0]),
               dict(pr=[1.0, np.nan, 2.0]), dict(pr=[1.0, np.inf, 2.0]), dict(pr=[0.0, 0.0, 0.0]),
               dict(h=[0.0, -1.0, 0.0]), dict(h=[0.0, np.nan, 0.0]), dict(h=[0.0, np.inf, 0.0]),
               dict(mp=[-1.0]), dict(mp=[np.nan]), dict(mp=[np.inf]),
               dict(opts=(0, 4000, 1e-4, 0.0, 0.0)), dict(opts=(1000, 4000, 0.0, 0.0, 0.0)),
               dict(opts=(1000, 4000, 1e-4, -1.0, 0.0)), dict(opts=(1000, 4000, 1e-4, 0.0, -1.0)),
               dict(opts=(1000, 4000, 1e-4, 0.0, np.inf)), dict(opts=(1000, 4000, 1e-4, 0.0, np.nan))]
        for d in bad:
            a_ = dict(good, **d)
            o = None if a_["opts"] is None else C.byref(cr._lib.PriceArbOpts(*a_["opts"]))
            out = cr._lib.PriceArbOut()
            rc_ = lib.cfmm_execute_price_arbitrage_rows(ctx, a_["q"], arr(a_["off"], np.int64), arr(a_["tok"], np.int64),
                                                        arr(a_["pr"], float), arr(a_["h"], float), arr(a_["mp"], float),
                                                        o, C.byref(out))
            assert rc_ == cr._lib.CFMM_ERR_INVALID, d
        assert lib.cfmm_execute_price_arbitrage_rows(ctx, 0, arr([0], np.int64), None, None, None, None, None,
                                                     None) == 0
        same_state(after, state(p))
    finally:
        m.close()


def test_router_quote_execute_and_refresh():
    from test_gpu_order_hubs import router_market
    r = router_market(cr, 22)
    rng = np.random.default_rng(69)
    lists = [[3, 1, 2, 5], [4, 6, 7, 8]]
    prices = [rng.uniform(0.5, 2.0, 4), rng.uniform(0.5, 2.0, 4)]
    holds = [[1.0, 0.0, 2.0, 0.0], [0.0, 0.0, 0.0, 3.0]]
    profit, st, det = r.quote_inventory_arbitrage(lists, prices, holds, opts={"atol": 1e-9})
    assert np.array_equal(profit, det.profit) and np.any(st == 0)
    profit2, st2, det2 = r.execute_inventory_arbitrage(lists, prices, holds)
    assert np.any(st2 == 0)
    for k in np.flatnonzero(st2 == 0):
        sl = slice(det2.leg_off[k], det2.leg_off[k + 1])
        for t, i in zip(det2.leg_type[sl], det2.leg_pool[sl]):
            dev, _ = r._pools.pool_state(int(t), int(i), 1)
            pool = r.cfmms[r._type_lists[int(t)][int(i)]]
            assert np.array_equal(np.asarray(pool.R), dev[0])
