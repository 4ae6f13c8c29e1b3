"""cfmm_quote_swaps_exact_out / cfmm_execute_swap_orders (include/cfmm_b200.h) on the device.

Exact-output quotes are checked for the crossing property through cfmm_quote_swaps at x* and at
pred(x*), and bit for bit against the host mirror (swap_order_oracle.py) for ProductTwoCoin and
UniV3.  Order batches are checked against the host replay, and against a fresh context on which
cfmm_execute_swaps runs the filled rows' paid tenders.  Every set has appended pools (a tail) and
retired pools; the ProductTwoCoin sets are laid out with orient_by_degree, so some of their pools
are stored with their tokens exchanged."""
import numpy as np
import pytest

import swap_order_oracle as oo
from test_gpu_parity import check_psi, make_pools
from test_gpu_swaps import product_set, univ3_ref_pool

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
DBL_MAX = np.finfo(np.float64).max


def pred(x):
    return np.nextafter(x, 0.0)


class Set:
    """A pool set of one type on the device (main + tail, some pools retired) and its host copy."""

    def __init__(self, cr, synth, t, seed, m=3000, mt=500, n=64):
        self._cr, self.t, self.n, self.m = cr, t, n, m + mt
        if t == P:
            R, g, A = product_set(m + mt, n, seed=seed, wide=False)
            self.args = (R, g, A)
            main, tail = (R[:m], g[:m], A[:m]), (R[m:], g[m:], A[m:])
            pre = {"orient_by_degree": 1}
        elif t == G:
            R, g, A, w = synth.geomean_pools(m + mt, n, seed=seed)
            self.args = (R, g, A, w)
            main, tail = (R[:m], g[:m], A[:m], w[:m]), (R[m:], g[m:], A[m:], w[m:])
            pre = {}
        else:
            cp, g, A, off, lt, lq = synth.univ3_pools(m, n, seed=seed, ragged=True)
            cpt, gt, At, offt, ltt, lqt = synth.univ3_pools(mt, n, seed=seed + 1, ragged=True)
            main, tail = (cp, g, A, off, lt, lq), (cpt, gt, At, offt, ltt, lqt)
            self.args = (np.concatenate([cp, cpt]), np.concatenate([g, gt]), np.concatenate([A, At]),
                         np.concatenate([off, off[-1] + offt[1:]]), np.concatenate([lt, ltt]),
                         np.concatenate([lq, lqt]))
            assert np.any(self.args[5] == 0.0) and set(np.diff(self.args[3])) >= {1, 16}
            pre = {}
        self.main, self.tail, self.pre = main, tail, pre
        self.retired = set(range(100, 140)) | set(range(m + 20, m + 40))
        self.p = self.fresh()

    def fresh(self):
        cr = self._cr
        kw = {("product", "geomean", "univ3")[self.t]: self.main}
        p = make_pools(cr, self.n, pre=self.pre, **kw)
        getattr(p, ("append_product", "append_geomean", "append_univ3")[self.t])(*self.tail)
        act = np.ones(self.m, bool)
        act[sorted(self.retired)] = False
        p.set_active(self.t, 0, act)
        return p

    def host_pools(self, p=None):
        """The mirror's pool objects at the device's current state (ladders read back)."""
        p = p or self.p
        if self.t == U:
            return univ3_host_pools(p, self.args[1])
        state, _ = p.pool_state(self.t)
        g = self.args[1]
        if self.t == P:
            return [oo.ProductPool(state[i], g[i]) for i in range(self.m)]
        return [oo.GeoMeanPool(state[i], g[i], self.args[3][i]) for i in range(self.m)]

    def out_scale(self):
        """Per pool, the output each side can give (R for two-coin; the walk's capacity for UniV3)."""
        if self.t != U:
            return np.asarray(self.args[0], dtype=float)
        hp = self.host_pools()
        return np.array([[hp[i].f(DBL_MAX, False), hp[i].f(DBL_MAX, True)] for i in range(self.m)])


def univ3_host_pools(p, g):
    """The mirror's UniV3 pools at the device's current state, ladders read back."""
    state, _ = p.pool_state(U)
    off, lt, lq = p.univ3_ticks()
    return [oo.Univ3Pool(state[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], g[i]) for i in range(len(state))]


@pytest.fixture(params=[P, G, U], ids=["product", "geomean", "univ3"])
def pset(request, cr, synth):
    s = Set(cr, synth, request.param, seed=100 + request.param)
    yield s
    s.p.close()


def wants_for(scale, rng, lo=-10.0, hi=0.3, zero_every=13):
    """One wanted output per row of scale [q, 2] (output capacity per side): a random side, y =
    10^U(lo, hi) times that side's capacity (hi > 0 gives unreachable rows)."""
    q = len(scale)
    side = rng.integers(0, 2, size=q)
    W = np.zeros((q, 2))
    W[np.arange(q), side] = scale[np.arange(q), side] * 10.0 ** rng.uniform(lo, hi, size=q)
    W[::zero_every] = 0.0
    return W


def tender_of(W, x):
    """The tender rows (x, 0) / (0, x) that go with wanted rows W (0, y) / (y, 0)."""
    T = np.zeros_like(W)
    tok1 = W[:, 1] > 0
    T[tok1, 0] = x[tok1]
    T[~tok1 & (W[:, 0] > 0), 1] = x[~tok1 & (W[:, 0] > 0)]
    return T


# ---- 1. exact-output quotes ----------------------------------------------------------------
def test_exact_out_quotes(pset):
    s, p = pset, pset.p
    rng = np.random.default_rng(1)
    scale = s.out_scale()
    W = wants_for(scale, rng)
    W[1] = [0.0, scale[1, 1]]            # exactly the capacity
    W[2] = [pred(scale[2, 0]), 0.0]       # one ulp below it
    W[3] = [0.0, 5e-324]                  # the least positive double
    pools = np.arange(s.m)
    T = p.quote_swaps_exact_out(s.t, pools, W)
    y = W.max(axis=1)
    x = T.max(axis=1)
    active = np.array([i not in s.retired for i in pools])
    assert np.all(T.min(axis=1) == 0.0)
    assert np.all(x[y == 0] == 0.0)
    assert np.all(np.isinf(x[(y > 0) & ~active]))
    live = (y > 0) & active
    reach = live & np.isfinite(x)
    unreach = live & ~np.isfinite(x)
    assert reach.sum() > s.m // 2 and unreach.sum() > 20
    side_out = np.where(W[:, 1] > 0, 1, 0)
    # crossing: f(x*) >= y and f(pred(x*)) < y, through cfmm_quote_swaps
    r_at = p.quote_swaps(s.t, pools[reach], T[reach])[np.arange(reach.sum()), side_out[reach]]
    assert np.all(r_at >= y[reach]), np.flatnonzero(r_at < y[reach])[:5]
    Tp = tender_of(W[reach], pred(x[reach]))
    r_pred = p.quote_swaps(s.t, pools[reach], Tp)[np.arange(reach.sum()), side_out[reach]]
    assert np.all(r_pred < y[reach]), np.flatnonzero(r_pred >= y[reach])[:5]
    # unreachable: even DBL_MAX falls short
    Tm = tender_of(W[unreach], np.full(unreach.sum(), DBL_MAX))
    r_max = p.quote_swaps(s.t, pools[unreach], Tm)[np.arange(unreach.sum()), side_out[unreach]]
    assert np.all(r_max < y[unreach])
    # bit for bit against the host mirror (ProductTwoCoin: every row; UniV3: a sample)
    if s.t != G:
        hp = s.host_pools()
        rows = pools if s.t == P else rng.choice(pools, size=600, replace=False)
        for i in rows:
            want = oo.quote_exact_out(hp[i], W[i], retired=i in s.retired)
            assert T[i].tolist() == list(want), (i, W[i], T[i], want)
    # ProductTwoCoin: the least tender (f is monotone, so the crossing is unique)
    if s.t == P:
        for i in np.flatnonzero(reach)[:200]:
            tok1 = W[i, 1] > 0
            lower = [oo.from_ordinal(oo.ordinal(x[i]) - k) for k in (1, 2, 7, 1000, 2 ** 20)]
            lower = [v for v in lower if v > 0]
            Tl = np.array([(v, 0.0) if tok1 else (0.0, v) for v in lower])
            r = p.quote_swaps(P, np.full(len(lower), i), Tl)[:, side_out[i]]
            assert np.all(r < y[i])
    # rows repeated in a shuffled batch are quoted on their own
    idx = rng.integers(0, s.m, size=2000)
    assert np.array_equal(p.quote_swaps_exact_out(s.t, idx, W[idx]), T[idx])


def test_geomean_exact_out_against_mpmath(cr, synth):
    import mpmath as mp
    m, n = 1000, 40
    R, g, A, w = synth.geomean_pools(m, n, seed=7)
    p = make_pools(cr, n, geomean=(R, g, A, w))
    rng = np.random.default_rng(8)
    W = wants_for(R, rng, lo=-10, hi=-0.01, zero_every=10 ** 9)
    x = p.quote_swaps_exact_out(G, np.arange(m), W).max(axis=1)
    eps = np.finfo(float).eps
    with mp.workdps(50):
        for i in range(m):
            o = 1 if W[i, 1] > 0 else 0
            eta = mp.mpf(w[i, 1 - o]) / mp.mpf(w[i, o])
            B = (4.5 + 2 * float(eta)) * eps * R[i, o]  # the forward bound, plus eps/2·R_out for γ·x

            def inv(yy):
                return mp.mpf(R[i, 1 - o]) * ((1 - mp.mpf(yy) / mp.mpf(R[i, o])) ** (-1 / eta) - 1) / mp.mpf(g[i])
            y = W[i, o]
            assert x[i] >= inv(y - B) and pred(x[i]) <= inv(min(y + B, np.nextafter(R[i, o], 0))), i
    p.close()


# ---- 2. mixed order batches ----------------------------------------------------------------
def order_batch(s, rng, q=6000, hot=200):
    """Rows on pools with many repeats: kinds mixed; exact-in tenders and exact-out wants sized to
    the pool; limits around the isolated quote, so some rows fill and some revert."""
    pools = rng.integers(0, s.m, size=q)
    pools[: q // 2] = rng.integers(0, hot, size=q // 2)  # repeats, retired pools among them
    rng.shuffle(pools)
    scale = s.out_scale()[pools]
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    W = wants_for(scale, rng, lo=-6, hi=0.05, zero_every=29)
    T = wants_for(np.maximum(scale, 1e-3), rng, lo=-6, hi=-0.5, zero_every=31)
    amount = np.where(kind[:, None] == 1, W, T)
    x_iso = s.p.quote_swaps_exact_out(s.t, pools, W).max(axis=1)
    r_iso = s.p.quote_swaps(s.t, pools, T).max(axis=1)
    f = 10.0 ** rng.uniform(-0.02, 0.02, size=q)
    limit = np.where(kind == 1, np.where(np.isfinite(x_iso), x_iso * f, 1.0), r_iso * f)
    limit[::17] = np.where(kind[::17] == 1, np.inf, 0.0)
    return pools, kind, amount, limit


def test_execute_orders(pset):
    s, p = pset, pset.p
    rng = np.random.default_rng(2)
    pools, kind, amount, limit = order_batch(s, rng)
    hp = s.host_pools() if s.t != G else None
    paid, rec, st = p.execute_swap_orders(s.t, pools, kind, amount, limit)
    counts = np.bincount(st, minlength=4)
    assert counts[0] > 1000 and counts[1] > 100 and counts[3] > 10, counts
    assert np.all(st[np.isin(pools, sorted(s.retired))] == oo.RETIRED)
    bad = st != 0
    assert not paid[bad].any() and not rec[bad].any()
    # exact-out fills receive at least what they wanted, and pay within their limit
    fo = (st == 0) & (kind == 1)
    assert np.all(rec[fo].max(axis=1) >= amount[fo].max(axis=1)) and np.all(paid[fo].max(axis=1) <= limit[fo])
    # the host replay, bit for bit (ProductTwoCoin and UniV3)
    if s.t != G:
        P2, R2, S2, _ = oo.replay_orders(hp, pools, kind, amount, limit, retired=s.retired)
        assert np.array_equal(st, S2), np.flatnonzero(st != S2)[:5]
        assert np.array_equal(paid, P2) and np.array_equal(rec, R2)
        state, _ = p.pool_state(s.t)
        want = np.array([h.price for h in hp]) if s.t == U else np.array([h.R for h in hp])
        act = np.array([i not in s.retired for i in range(s.m)])
        assert np.array_equal(state[act], want[act])
    # a fresh context executing only the filled rows' paid tenders: same state, same received
    f = s.fresh()
    ok = st == 0
    got = f.execute_swaps(s.t, pools[ok], paid[ok])
    assert np.array_equal(got, rec[ok])
    assert np.array_equal(f.pool_state(s.t)[0], p.pool_state(s.t)[0])
    if s.t == U:
        for a, b in zip(f.univ3_ticks(), p.univ3_ticks()):
            assert np.array_equal(a, b)
    f.close()


def test_limits_at_the_boundary(pset):
    s, p = pset, pset.p
    scales = s.out_scale()
    i = next(k for k in range(s.m) if k not in s.retired and scales[k].min() > 0)
    st0 = p.pool_state(s.t)[0].copy()
    scale = scales[i]
    y = 0.01 * scale[1]
    x = p.quote_swaps_exact_out(s.t, [i], [[0.0, y]])[0, 0]
    assert 0 < x < np.inf
    # one ulp under x* reverts and leaves the state; x* itself then fills, against the same state
    paid, rec, st = p.execute_swap_orders(s.t, [i, i], [1, 1], [[0.0, y], [0.0, y]], [pred(x), x])
    assert st.tolist() == [oo.LIMIT, oo.FILLED] and paid[1].tolist() == [x, 0.0] and not paid[0].any()
    assert rec[1, 1] >= y
    st1 = p.pool_state(s.t)[0].copy()
    assert not np.array_equal(st1, st0)
    # an exact-in row: a minimum one ulp above what arrives reverts, the exact amount fills
    r = p.quote_swaps(s.t, [i], [[0.0, 0.3 * scale[0]]])[0, 0]
    paid, rec, st = p.execute_swap_orders(s.t, [i, i], [0, 0], [[0.0, 0.3 * scale[0]]] * 2,
                                          [np.nextafter(r, np.inf), r])
    assert st.tolist() == [oo.LIMIT, oo.FILLED] and rec[1, 0] == r and rec[0].tolist() == [0.0, 0.0]
    # an exact-out row past what the pool can give is unreachable, and changes nothing
    st2 = p.pool_state(s.t)[0].copy()
    cap = s.out_scale()[i, 1] if s.t == U else st2[i, 1]
    _, _, st = p.execute_swap_orders(s.t, [i], [1], [[0.0, 2 * cap + 1.0]])
    assert st.tolist() == [oo.UNREACHABLE]
    assert np.array_equal(p.pool_state(s.t)[0], st2)


def test_all_exact_in_equals_execute_swaps(pset):
    s = pset
    rng = np.random.default_rng(3)
    q = 4000
    pools = rng.integers(0, s.m, size=q)
    pools[::3] = rng.integers(0, 50, size=len(pools[::3]))
    T = wants_for(np.maximum(s.out_scale()[pools], 1e-3), rng, lo=-6, hi=0, zero_every=23)
    a, b = s.fresh(), s.fresh()
    paid, rec, st = a.execute_swap_orders(s.t, pools, np.zeros(q, np.uint8), T)
    got = b.execute_swaps(s.t, pools, T)
    active = ~np.isin(pools, sorted(s.retired))
    assert np.array_equal(rec, got) and np.array_equal(paid[active], T[active])
    assert np.all(st[active] == 0) and np.all(st[~active] == oo.RETIRED)
    assert np.array_equal(a.pool_state(s.t)[0], b.pool_state(s.t)[0])
    a.close()
    b.close()


# ---- 3. rejected calls ---------------------------------------------------------------------
def test_rejected_calls_change_nothing(cr, synth):
    n = 30
    Rp, gp, Ap = synth.product_pools(500, n, seed=71)
    Rg, gg, Ag, wg = synth.geomean_pools(400, n, seed=72)
    cu = synth.univ3_pools(300, n, seed=73, ragged=True)
    p = make_pools(cr, n, product=(Rp, gp, Ap), geomean=(Rg, gg, Ag, wg), univ3=cu)
    s0 = [p.pool_state(t)[0].copy() for t in (P, G, U)]
    one = [[0.0, 1.0]]
    bad = [  # (type, pools, kind, amount, limit)
        (5, [0], [1], one, None), (P, [500], [1], one, None), (U, [-1], [0], one, None),
        (P, [0], [2], one, None), (G, [0, 1], [0, 7], one * 2, None),
        (P, [0], [1], [[np.nan, 0.0]], None), (U, [0], [0], [[np.inf, 0.0]], None),
        (G, [0], [1], [[-1.0, 0.0]], None), (P, [0], [1], [[1.0, 1.0]], None),
        (P, [0], [1], one, [np.nan]), (U, [0], [1], one, [-1.0]), (G, [0], [0], one, [np.inf]),
        (P, [0, 1], [1, 0], one * 2, [1.0, np.inf]),
    ]
    for t, pools, kind, amount, limit in bad:
        with pytest.raises(cr.CFMMError) as e:
            p.execute_swap_orders(t, pools, kind, np.array(amount), limit)
        assert e.value.code == -1, (t, pools, kind, amount, limit)
    for t, pools, W in ((5, [0], one), (P, [500], one), (G, [0], [[np.nan, 0.0]]), (U, [0], [[1.0, 1.0]])):
        with pytest.raises(cr.CFMMError) as e:
            p.quote_swaps_exact_out(t, pools, np.array(W))
        assert e.value.code == -1
    for t in (P, G, U):
        assert np.array_equal(p.pool_state(t)[0], s0[t])
    # an exact-out row with an infinite limit is fine, and q == 0 does nothing
    p.execute_swap_orders(P, [0], [1], one, [np.inf])
    paid, rec, st = p.execute_swap_orders(U, [], [], np.zeros((0, 2)))
    assert paid.shape == (0, 2) and st.shape == (0,)
    assert p.quote_swaps_exact_out(G, [], np.zeros((0, 2))).shape == (0, 2)
    p.close()
    q = cr.DevicePools(n)
    q.add_product(Rp, gp, Ap)
    with pytest.raises(cr.CFMMError) as e:
        q.quote_swaps_exact_out(P, [0], np.array(one))
    assert e.value.code == -3
    with pytest.raises(cr.CFMMError) as e:
        q.execute_swap_orders(P, [0], [1], np.array(one))
    assert e.value.code == -3
    q.close()


# ---- 4. sweeps after execute ---------------------------------------------------------------
def test_sweeps_after_orders(cr, oracle, synth):
    m = 20000
    R, g, A, v = synth.disjoint_product(m, seed=81, adversarial=False)
    n = 2 * m
    p = make_pools(cr, n, product=(R, g, A))
    for _ in range(3):  # the second call captures the sweep graph, the third replays it
        p.sweep(v)
    info0 = p.pool_set_info(P)
    assert info0["fast_range"] == 1 and info0["fixed_point"] == 1
    rng = np.random.default_rng(82)
    q = 8000
    pools = rng.integers(0, m, size=q)
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    side = rng.integers(0, 2, size=q)
    amount = np.zeros((q, 2))
    amount[np.arange(q), side] = R[pools, side] * 10.0 ** rng.uniform(-4, -0.5, size=q)
    paid, rec, st = p.execute_swap_orders(P, pools, kind, amount)
    assert set(st.tolist()) <= {0, 2} and (st == 0).sum() > q - 100  # (repeated rows can drain a pool)
    state, _ = p.pool_state(P)
    assert not np.array_equal(state, R)
    psi, acc = p.sweep(v)
    f = make_pools(cr, n, product=(state, g, A))
    psi_f, acc_f = f.sweep(v)
    assert np.array_equal(psi, psi_f) and abs(acc - acc_f) <= 1e-12 * abs(acc_f)
    D, L = oracle.sweep_product(state, g, A, v)
    check_psi(oracle, A, D, L, v, n, psi, acc, R=state, g=g)
    i1, i2 = p.pool_set_info(P), f.pool_set_info(P)
    assert i1["fixed_point"] == i2["fixed_point"] and i1["fast_range"] == i2["fast_range"]
    f.close()
    # an exact-out row that nearly drains a pool, then an exact-in row that leaves the guard-free range
    _, _, st = p.execute_swap_orders(P, [7, 8], [1, 0], [[0.0, pred(state[7, 1])], [2.0 ** 110, 0.0]])
    assert st.tolist() == [0, 0]
    state, _ = p.pool_state(P)
    assert state[8, 0] > 2.0 ** 100
    f = make_pools(cr, n, product=(state, g, A))
    i1, i2 = p.pool_set_info(P), f.pool_set_info(P)
    assert i1["fast_range"] == i2["fast_range"] == 0 and i1["fixed_point"] == i2["fixed_point"]
    psi, acc = p.sweep(v)
    psi_f, acc_f = f.sweep(v)
    assert np.array_equal(psi, psi_f) and abs(acc - acc_f) <= 1e-12 * abs(acc_f)
    f.close()
    p.close()


# ---- 5. with liquidity changes and compact --------------------------------------------------
def test_orders_after_liquidity_and_compact(cr, synth):
    n, m, mt = 40, 1500, 300
    cp, g, A, off, lt, lq = synth.univ3_pools(m, n, seed=91, ragged=True)
    tail = synth.univ3_pools(mt, n, seed=92, ragged=True)
    p = make_pools(cr, n, univ3=(cp, g, A, off, lt, lq))
    p.append_univ3(*tail)
    rng = np.random.default_rng(93)
    # mint on new ranges around the current price: the ladders grow
    rows = rng.integers(0, m + mt, size=400)
    price, _ = p.pool_state(U)
    lo = price[rows] * rng.uniform(0.5, 0.99, size=400)
    hi = price[rows] * rng.uniform(1.01, 1.5, size=400)
    ticks0 = p.univ3_ticks(ladders=False)[0]
    p.modify_univ3_liquidity(rows, lo, hi, rng.uniform(1, 20, size=400))
    off1, lt1, lq1 = p.univ3_ticks()
    assert off1[-1] > ticks0[-1]
    hp = univ3_host_pools(p, np.concatenate([g, tail[1]]))
    q = 3000
    pools = np.concatenate([rows, rng.integers(0, m + mt, size=q - len(rows))])
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    amount = np.zeros((q, 2))
    amount[np.arange(q), rng.integers(0, 2, size=q)] = 10.0 ** rng.uniform(-4, 1, size=q)
    limit = np.where(kind == 1, 10.0 ** rng.uniform(-4, 2, size=q), 10.0 ** rng.uniform(-6, 0, size=q))
    paid, rec, st = p.execute_swap_orders(U, pools, kind, amount, limit)
    P2, R2, S2, _ = oo.replay_orders(hp, pools, kind, amount, limit)
    assert np.array_equal(st, S2) and np.array_equal(paid, P2) and np.array_equal(rec, R2)
    assert (st == 0).sum() > 100 and (st == 1).sum() > 100
    # compact folds the tail in: the same state quotes the same tenders
    W = wants_for(np.ones((m + mt, 2)), rng, lo=-4, hi=0.5)
    before = p.quote_swaps_exact_out(U, np.arange(m + mt), W)
    p.compact()
    assert p.pool_set_info(U)["tail"] == 0
    after = p.quote_swaps_exact_out(U, np.arange(m + mt), W)
    assert np.array_equal(before, after)
    paid2, rec2, st2 = p.execute_swap_orders(U, pools, kind, amount, limit)
    P3, R3, S3, _ = oo.replay_orders(hp, pools, kind, amount, limit)
    assert np.array_equal(st2, S3) and np.array_equal(paid2, P3) and np.array_equal(rec2, R3)
    p.close()


def test_reference_pool_orders(cr):
    """test/cfmms.jl's UniV3 pool: exact-out rows across every tick, against the mirror."""
    cp, lt, lq, g = univ3_ref_pool(0.997)
    p = make_pools(cr, 2, univ3=(np.array([cp]), np.array([g]), np.array([[1, 2]]), np.array([0, 4]), lt, lq))
    pool = oo.Univ3Pool(cp, lt, lq, g)
    ys = np.concatenate([np.geomspace(1e-9, 1, 30) * pool.f(DBL_MAX, True), [pool.f(DBL_MAX, True)]])
    W = np.concatenate([np.stack([0 * ys, ys], 1), np.stack([ys * 10, 0 * ys], 1)])
    T = p.quote_swaps_exact_out(U, np.zeros(len(W), dtype=np.int64), W)
    for j, w in enumerate(W):
        assert T[j].tolist() == list(oo.quote_exact_out(pool, w)), (w, T[j])
    p.close()


def test_router_orders_device(cr):
    rng = np.random.default_rng(95)
    n = 8
    pools = []
    for k in range(30):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 0:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        elif k % 3 == 1:
            pools.append(cr.GeometricMeanTwoCoin(100 + 900 * rng.random(2), [0.3, 0.7], 0.997, [a, b]))
        else:
            c = float(np.exp(rng.uniform(-1, 1)))
            pools.append(cr.UniV3(c, c * 1.5 * np.cumprod([1.0, 0.8, 0.7, 0.6]), [100.0, 50.0, 0.0, 80.0], 0.997, [a, b]))
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n)
    ids = rng.integers(0, 30, size=60)
    W = wants_for(np.ones((60, 2)) * 20, rng, lo=-2, hi=0)
    x = r.quote_swaps_exact_out(ids, W)
    kind = np.ones(60, np.uint8)
    paid, rec, st = r.execute_swap_orders(ids, kind, W)
    assert np.array_equal(paid[0], x[0])  # the first row sees no earlier row
    for i, c in enumerate(pools):
        t = (P, G, U)[i % 3]
        k = r._type_lists[t].index(i)
        state = r._pools.pool_state(t, k, 1)[0]
        if t == U:
            assert c.current_price == state[0]
        else:
            assert np.array_equal(c.R, state[0])
    r._pools.close()
