"""cfmm_quote_swaps / cfmm_execute_swaps (include/cfmm_b200.h) on the device.

ProductTwoCoin and UniV3 results are checked bit for bit against host restatements of the
reference's forward trade (swap_oracle.py) and against oracle_univ3_forward_trade; GeometricMean
quotes against a 50-digit truth within the bound the header states.  Execution is checked against
host replays of the rows in batch order, and the state it leaves against fresh contexts and the
sweep oracle."""
import numpy as np
import pytest

import swap_oracle as so
from test_gpu_parity import EPS, check_psi, make_pools

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2


def tenders_for(R_in_scale, rng, lo=-12.0, hi=6.0, zero_every=17):
    """One tender per pool: a random side, x = 10^U(lo, hi) times that side's scale; every
    zero_every-th row (0, 0)."""
    m = len(R_in_scale)
    side = rng.integers(0, 2, size=m)
    x = R_in_scale[np.arange(m), side] * 10.0 ** rng.uniform(lo, hi, size=m)
    T = np.zeros((m, 2))
    T[np.arange(m), side] = x
    T[::zero_every] = 0.0
    return T


def product_set(m, n, seed, wide):
    rng = np.random.default_rng(seed)
    R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=(m, 2)))
    g = rng.uniform(0.99, 1.0, size=m) if wide else rng.choice([0.997, 0.999, 1.0], size=m)
    a = rng.integers(1, n + 1, size=m)
    b = (a + rng.integers(1, n, size=m) - 1) % n + 1
    if n > 8:  # a hub token: orient_by_degree has something to turn
        a[::5] = 1
        b[::5] = np.where(b[::5] == 1, 2, b[::5])
    return R, g, np.stack([a, b], axis=1).astype(np.int64)


def univ3_ref_pool(gamma):
    # test/cfmms.jl:117-120
    return 15.0, np.array([30.0, 20, 10, 5]), np.array([1.0, 2.0, 1.5, 0.0]), gamma


# ---- 1. ProductTwoCoin quotes ----------------------------------------------------------
@pytest.mark.parametrize("orient", [1, 0])
@pytest.mark.parametrize("wide", [False, True])
def test_product_quotes(cr, orient, wide):
    n, m, mt = 64, 4000, 700
    R, g, A = product_set(m + mt, n, seed=3 + orient + 2 * wide, wide=wide)
    p = make_pools(cr, n, product=(R[:m], g[:m], A[:m]), pre={"orient_by_degree": orient})
    p.append_product(R[m:], g[m:], A[m:])
    info = p.pool_set_info(P)
    assert info["tail"] == mt and info["compact_stream"] == (0 if wide else 1)
    rng = np.random.default_rng(1)
    T = tenders_for(R, rng)
    T[1] = [R[1, 0] * 1e-12, 0.0]
    T[2] = [0.0, R[2, 1] * 1e6]
    pools = np.arange(m + mt)
    got = p.quote_swaps(P, pools, T)
    want = np.array([so.product_forward(R[i], g[i], T[i]) for i in pools])
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    # a shuffled batch with repeats: each row on its own
    idx = rng.integers(0, m + mt, size=3000)
    got = p.quote_swaps(P, idx, T[idx])
    assert np.array_equal(got, want[idx])
    p.close()


# ---- 2. UniV3 quotes -----------------------------------------------------------------------
@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_univ3_quotes_reference_pool(cr, oracle, gamma):
    cp, lt, lq, g = univ3_ref_pool(gamma)
    p = make_pools(cr, 2, univ3=(np.array([cp]), np.array([g]), np.array([[1, 2]]), np.array([0, 4]), lt, lq))
    xs = np.concatenate([[0.0, 1e-12, 1e-3, 0.1, 0.5, 1.0], np.geomspace(1e-3, 1e6, 40), [1e12, 1e300]])
    T = np.concatenate([np.stack([xs, 0 * xs], 1), np.stack([0 * xs, xs], 1)])
    got = p.quote_swaps(U, np.zeros(len(T), dtype=np.int64), T)
    for j, t in enumerate(T):
        lam = oracle.univ3_forward_trade(cp, lt, lq, g, t)
        want = [0.0, lam] if t[0] > 0 else [lam, 0.0]
        assert got[j].tolist() == want, (t, got[j], want)
        assert so.univ3_swap(cp, lt, lq, g, t)[0] == lam
    # draining: a token-2 tender of 1e300 takes every token 1 of ticks 1..current
    assert got[-1, 0] > 0 and got[-1, 1] == 0.0
    p.close()


def test_univ3_quotes_ragged(cr, oracle, synth):
    m, n = 3000, 40
    cp, g, A, off, lt, lq = synth.univ3_pools(m, n, seed=21, ragged=True)
    mt = 400
    cpt, gt, At, offt, ltt, lqt = synth.univ3_pools(mt, n, seed=22, ragged=True)
    p = make_pools(cr, n, univ3=(cp, g, A, off, lt, lq))
    p.append_univ3(cpt, gt, At, offt, ltt, lqt)
    cpa, ga = np.concatenate([cp, cpt]), np.concatenate([g, gt])
    offa = np.concatenate([off, off[-1] + offt[1:]])
    lta, lqa = np.concatenate([lt, ltt]), np.concatenate([lq, lqt])
    assert np.any(lqa == 0.0) and set(np.diff(offa)) >= {1, 16}
    rng = np.random.default_rng(5)
    scale = np.stack([np.sqrt(lqa[offa[:-1]] + 1), np.sqrt(lqa[offa[:-1]] + 1)], 1)
    T = tenders_for(scale, rng, lo=-8, hi=4)
    T[3::11] = np.where(T[3::11] > 0, 1e30, 0.0)  # drain every tick in that direction
    pools = np.arange(m + mt)
    got = p.quote_swaps(U, pools, T)
    for i in pools:
        s = slice(offa[i], offa[i + 1])
        lam = oracle.univ3_forward_trade(cpa[i], lta[s], lqa[s], ga[i], T[i])
        want = [0.0, lam] if T[i, 0] > 0 else ([lam, 0.0] if T[i, 1] > 0 else [0.0, 0.0])
        assert got[i].tolist() == want, (i, T[i], got[i], want)
    p.close()


# ---- 3. GeometricMean quotes ---------------------------------------------------------------
def test_geomean_quotes(cr):
    import mpmath as mp
    m, n = 1500, 50
    rng = np.random.default_rng(8)
    R = np.exp(rng.uniform(np.log(1e-2), np.log(1e4), size=(m, 2)))
    w1 = rng.choice([1 / 25, 24 / 25, 0.5, 0.3], size=m)
    w1[::7] = rng.uniform(0.05, 0.95, size=len(w1[::7]))
    w = np.stack([w1, 1 - w1], 1)
    g = rng.choice([0.997, 1.0], size=m)
    a = rng.integers(1, n + 1, size=m)
    A = np.stack([a, a % n + 1], 1)
    p = make_pools(cr, n, geomean=(R, g, A, w))
    T = tenders_for(R, rng, lo=-12, hi=6)
    got = p.quote_swaps(G, np.arange(m), T)
    worst = 0.0
    for i in range(m):
        truth = so.geomean_truth(R[i], w[i], g[i], T[i])
        o = 1 if T[i, 0] > 0 else 0
        assert got[i, 1 - o] == 0.0
        if T[i].max() == 0:
            assert got[i].tolist() == [0.0, 0.0]
            continue
        eta = w[i, 1 - o] / w[i, o]
        err = abs(mp.mpf(float(got[i, o])) - truth[o]) / (EPS * R[i, o])
        worst = max(worst, float(err) / (4 + 2 * eta))
        assert 0.0 <= got[i, o] <= R[i, o]
        assert err <= 4 + 2 * eta, (i, float(err), eta)
        # ϕ(R + γΔ − Λ) ≥ ϕ(R) − √eps (test/cfmms.jl:18), on ϕ normalised to ϕ(R) = 1, for rows that
        # leave at least 1e-6 of R_out: nearer a drain the bound's few ulp of λ alone exceed √eps of ϕ
        if truth[o] > R[i, o] * (1 - 1e-6):
            continue
        with mp.workdps(50):
            Rn = [mp.mpf(float(R[i, k])) + mp.mpf(float(g[i])) * mp.mpf(float(T[i, k])) - mp.mpf(float(got[i, k]))
                  for k in (0, 1)]
            phi = (Rn[0] / mp.mpf(float(R[i, 0]))) ** mp.mpf(float(w[i, 0])) * \
                  (Rn[1] / mp.mpf(float(R[i, 1]))) ** mp.mpf(float(w[i, 1]))
            assert phi >= 1 - mp.sqrt(mp.mpf(EPS)), (i, phi)
    print(f"\ngeomean quote error: max {worst:.3f} of the (4 + 2η)·eps·R_out bound")
    p.close()


# ---- 4. the reference's predicate on routed trades -----------------------------------------
def test_quote_own_trades(cr, synth):
    n = 30
    Rp, gp, Ap = synth.product_pools(2000, n, seed=31)
    Rg, gg, Ag, wg = synth.geomean_pools(1500, n, seed=32)
    cp, gu, Au, off, lt, lq = synth.univ3_pools(1500, n, seed=33, ragged=True)
    p = make_pools(cr, n, product=(Rp, gp, Ap), geomean=(Rg, gg, Ag, wg), univ3=(cp, gu, Au, off, lt, lq))
    v = synth.dual_prices(n, "wide")
    p.sweep(v, materialize=True)
    D, L = p.trades()
    k0, k1 = 2000, 3500
    for t, lo, hi, R in ((P, 0, k0, Rp), (G, k0, k1, Rg)):
        q = p.quote_swaps(t, np.arange(hi - lo), D[lo:hi])
        tol = (64 if t == G else 8) * EPS * (R[:, 0] + R[:, 1])
        assert np.all(np.abs(q - L[lo:hi]) <= tol[:, None]), np.max(np.abs(q - L[lo:hi]) / tol[:, None])
    q = p.quote_swaps(U, np.arange(1500), D[k1:])
    Lu, Du = L[k1:], D[k1:]
    for i in range(1500):
        s = slice(off[i], off[i + 1])
        pr = v[Au[i, 0] - 1] / v[Au[i, 1] - 1]
        if pr > lt[s][0] or (pr < lt[s][-1] and lq[s][-1] == 0.0):  # out of liquidity (test/cfmms.jl:37-42)
            assert Lu[i].min() == 0.0
            assert np.allclose(q[i], Lu[i], rtol=1e-12, atol=0), (i, q[i], Lu[i])
        else:
            assert np.allclose(q[i], Lu[i], rtol=1e-9, atol=64 * EPS * (np.abs(Lu[i]).max() + 1)), (i, q[i], Lu[i])
        assert (q[i] == 0).tolist() == (Du[i][::-1] == 0).tolist() or Du[i].max() == 0
    p.close()


# ---- 5. execute, two-coin ------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["product", "geomean"])
def test_execute_two_coin(cr, synth, kind):
    n, m = 40, 3000
    rng = np.random.default_rng(12)
    if kind == "product":
        R, g, A = product_set(m, n, seed=13, wide=False)
        p = make_pools(cr, n, product=(R, g, A), pre={"orient_by_degree": 1})
        t = P
    else:
        R, g, A, w = synth.geomean_pools(m, n, seed=14)
        p = make_pools(cr, n, geomean=(R, g, A, w))
        t = G
    q = 5000
    pools = rng.integers(0, m, size=q)
    T = tenders_for(R[pools], rng, lo=-6, hi=0)
    got = p.execute_swaps(t, pools, T)
    Rh = R.copy()
    for j, i in enumerate(pools):  # replay in batch order with the returned Λ
        if kind == "product":
            assert got[j].tolist() == list(so.product_forward(Rh[i], g[i], T[j])), j
        if T[j].max() > 0:
            Rh[i] = (Rh[i] + g[i] * T[j]) - got[j]
    state, _ = p.pool_state(t)
    assert np.array_equal(state, Rh), np.argwhere(state != Rh)[:5]
    p.close()


# ---- 6. execute, UniV3 ---------------------------------------------------------------------
def test_execute_univ3(cr, oracle, synth):
    n, m = 40, 2000
    cp, g, A, off, lt, lq = synth.univ3_pools(m, n, seed=41, ragged=True)
    p = make_pools(cr, n, univ3=(cp, g, A, off, lt, lq))
    rng = np.random.default_rng(42)
    q = 6000
    pools = rng.integers(0, m, size=q)
    scale = np.sqrt(lq[off[:-1]] + 1)[pools]
    T = tenders_for(np.stack([scale, scale], 1), rng, lo=-6, hi=2)
    T[5::13] = np.where(T[5::13] > 0, 1e30, 0.0)
    got = p.execute_swaps(U, pools, T)
    cph = cp.copy()
    for j, i in enumerate(pools):
        s = slice(off[i], off[i + 1])
        lam, qn = so.univ3_swap(cph[i], lt[s], lq[s], g[i], T[j])
        want = [0.0, lam] if T[j, 0] > 0 else ([lam, 0.0] if T[j, 1] > 0 else [0.0, 0.0])
        assert got[j].tolist() == want, (j, i, got[j], want)
        assert lt[s][-1] * 0 <= qn <= lt[s][0]
        cph[i] = qn
    state, _ = p.pool_state(U)
    assert np.array_equal(state, cph), np.argwhere(state != cph)[:5]
    moved = np.flatnonzero(cph != cp)
    assert len(moved) > m // 2
    for v in (synth.dual_prices(n, "wide"), synth.dual_prices(n, "near")):
        p.sweep(v, materialize=True)
        D, L = p.trades()
        Do, Lo = oracle.sweep_univ3(cph, g, A, off, lt, lq, v)
        assert np.array_equal(D, Do) and np.array_equal(L, Lo)
        f = make_pools(cr, n, univ3=(state, g, A, off, lt, lq))
        f.sweep(v, materialize=True)
        Df, Lf = f.trades()
        assert np.array_equal(Df, D) and np.array_equal(Lf, L)
        f.close()
    p.close()


# ---- 7. consistency with cfmm_apply_trades -------------------------------------------------
def test_execute_matches_apply_trades(cr, synth):
    n, m = 30, 2000
    cp, g, A, off, lt, lq = synth.univ3_pools(m, n, seed=51)
    a = make_pools(cr, n, univ3=(cp, g, A, off, lt, lq))
    b = make_pools(cr, n, univ3=(cp, g, A, off, lt, lq))
    rng = np.random.default_rng(52)
    v = np.exp(rng.uniform(np.log(0.3), np.log(3.0), size=n))
    a.sweep(v, materialize=True)
    D, L = a.trades()
    a.apply_trades()
    qa, _ = a.pool_state(U)
    got = b.execute_swaps(U, np.arange(m), D)
    qb, _ = b.pool_state(U)
    # pools whose walk target lies inside the ladder (apply_trades clamps only at T₁; a walk past
    # the last non-empty tick ends on its boundary instead)
    pr = v[A[:, 0] - 1] / v[A[:, 1] - 1]
    inside = (pr >= lt[off[:-1] + 2] / g) & (pr <= lt[off[:-1]] * g)
    traded = D.max(axis=1) > 0
    sel = inside & traded
    assert sel.sum() > m // 10
    assert np.all(np.abs(qb[sel] - qa[sel]) <= 1e-12 * qa[sel]), np.max(np.abs(qb[sel] / qa[sel] - 1))
    assert np.allclose(got[sel], L[sel], rtol=1e-9, atol=0)
    a.close()
    b.close()


# ---- 8. batch order ------------------------------------------------------------------------
@pytest.mark.parametrize("t", [P, G, U])
def test_batch_order(cr, synth, t):
    n, m = 20, 300
    rng = np.random.default_rng(60 + t)
    if t == P:
        args = synth.product_pools(m, n, seed=61)
    elif t == G:
        args = synth.geomean_pools(m, n, seed=62)
    else:
        args = synth.univ3_pools(m, n, seed=63, ragged=True)

    def fresh():
        return make_pools(cr, n, **{("product", "geomean", "univ3")[t]: args})
    q = 900
    pools = rng.integers(0, m // 10, size=q)  # many repeats
    scale = args[0][pools] if t != U else np.full((q, 2), 10.0)
    T = tenders_for(scale, rng, lo=-3, hi=0)
    a, b = fresh(), fresh()
    ga = a.execute_swaps(t, pools, T)
    gb = np.concatenate([b.execute_swaps(t, pools[j:j + 1], T[j:j + 1]) for j in range(q)])
    assert np.array_equal(ga, gb)
    assert np.array_equal(a.pool_state(t)[0], b.pool_state(t)[0])
    # a→b then b→a against the reverse order on one pool
    c, d = fresh(), fresh()
    rows = np.array([[5.0, 0.0], [0.0, 5.0]])
    gc = c.execute_swaps(t, [0, 0], rows)
    gd = d.execute_swaps(t, [0, 0], rows[::-1])
    assert not np.array_equal(gc, gd[::-1])
    # quotes in one batch do not see each other
    qq = c.quote_swaps(t, [1, 1, 1], [[5.0, 0.0]] * 3)
    assert np.array_equal(qq[0], qq[1]) and np.array_equal(qq[0], qq[2])
    for x in (a, b, c, d):
        x.close()


# ---- 9. no-ops and errors ------------------------------------------------------------------
def test_noops_retired_and_errors(cr, synth):
    n = 30
    Rp, gp, Ap = synth.product_pools(1000, n, seed=71)
    Rg, gg, Ag, wg = synth.geomean_pools(800, n, seed=72)
    cu = synth.univ3_pools(600, n, seed=73, ragged=True)
    p = make_pools(cr, n, product=(Rp, gp, Ap), geomean=(Rg, gg, Ag, wg), univ3=cu)
    v = synth.dual_prices(n, "wide")
    p.sweep(v, materialize=True)
    trades0 = p.trades()

    def states():
        return [p.pool_state(t)[0].copy() for t in (P, G, U)]
    s0 = states()
    rng = np.random.default_rng(74)
    for t, m in ((P, 1000), (G, 800), (U, 600)):
        p.quote_swaps(t, np.arange(m), tenders_for(np.ones((m, 2)) * 50, rng))
        z = p.execute_swaps(t, np.arange(m), np.zeros((m, 2)))
        assert not z.any()
    for x, y in zip(states(), s0):
        assert np.array_equal(x, y)
    p.sweep(v, materialize=True)
    assert all(np.array_equal(x, y) for x, y in zip(p.trades(), trades0))
    # retired pools: receive zero, keep their parked state, live again after restore
    for t in (P, G, U):
        p.set_active(t, 10, np.zeros(20, bool))
        T = np.tile([[3.0, 0.0], [0.0, 3.0]], (10, 1))
        assert not p.quote_swaps(t, np.arange(10, 30), T).any()
        assert not p.execute_swaps(t, np.arange(10, 30), T).any()
        st, act = p.pool_state(t, 10, 20)
        assert np.array_equal(st, s0[t][10:30]) and not act.any()
        p.set_active(t, 10, np.ones(20, bool))
        assert p.quote_swaps(t, [10], [[3.0, 0.0]]).any()
    for x, y in zip(states(), s0):
        assert np.array_equal(x, y)
    # rejected inputs: the code, and no change
    bad = [(5, [0], [[1.0, 0.0]]), (P, [1000], [[1.0, 0.0]]), (P, [-1], [[1.0, 0.0]]),
           (G, [0], [[np.nan, 0.0]]), (U, [0], [[np.inf, 0.0]]), (P, [0], [[-1.0, 0.0]]),
           (G, [0], [[1.0, 1.0]]), (P, [0, 1], [[1.0, 0.0], [0.0, -0.5]])]
    for t, pools, T in bad:
        for fn in (p.quote_swaps, p.execute_swaps):
            with pytest.raises(cr.CFMMError) as e:
                fn(t, pools, np.array(T))
            assert e.value.code == -1
    for x, y in zip(states(), s0):
        assert np.array_equal(x, y)
    with pytest.raises(ValueError):
        p.quote_swaps(P, [0, 1], [[1.0, 0.0]])
    p.close()
    q = cr.DevicePools(n)
    q.add_product(Rp, gp, Ap)
    for fn in (q.quote_swaps, q.execute_swaps):
        with pytest.raises(cr.CFMMError) as e:
            fn(P, [0], np.array([[1.0, 0.0]]))
        assert e.value.code == -3
    q.close()


# ---- 10. sweeps after execute --------------------------------------------------------------
def test_sweeps_after_execute(cr, oracle, synth):
    m = 20000
    R, g, A, v = synth.disjoint_product(m, seed=81, adversarial=False)
    n = 2 * m
    p = make_pools(cr, n, product=(R, g, A))
    for _ in range(3):  # the second call captures the sweep graph, the third replays it
        p.sweep(v)
    info0 = p.pool_set_info(P)
    assert info0["fast_range"] == 1 and info0["fixed_point"] == 1
    rng = np.random.default_rng(82)
    pools = rng.integers(0, m, size=8000)
    T = tenders_for(R[pools], rng, lo=-4, hi=1)
    p.execute_swaps(P, pools, T)
    state, _ = p.pool_state(P)
    psi, acc = p.sweep(v)
    f = make_pools(cr, n, product=(state, g, A))
    psi_f, acc_f = f.sweep(v)
    assert np.array_equal(psi, psi_f) and abs(acc - acc_f) <= 1e-12 * abs(acc_f)  # (acc: fp64 atomics, any order)
    D, L = oracle.sweep_product(state, g, A, v)
    check_psi(oracle, A, D, L, v, n, psi, acc, R=state, g=g)
    f.close()
    # push one pool's reserves out of the guard-free range
    p.execute_swaps(P, [7], [[2.0 ** 110, 0.0]])
    state, _ = p.pool_state(P)
    assert state[7, 0] > 2.0 ** 100
    f = make_pools(cr, n, product=(state, g, A))
    i1, i2 = p.pool_set_info(P), f.pool_set_info(P)
    assert i1["fast_range"] == 0 and i1["fast_range"] == i2["fast_range"] and i1["fixed_point"] == i2["fixed_point"]
    psi, acc = p.sweep(v)
    psi_f, acc_f = f.sweep(v)
    assert np.array_equal(psi, psi_f) and abs(acc - acc_f) <= 1e-12 * abs(acc_f)  # (acc: fp64 atomics, any order)
    f.close()
    p.close()


def test_router_swaps_device(cr, synth):
    rng = np.random.default_rng(91)
    n = 8
    pools = []
    for k in range(30):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 0:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        elif k % 3 == 1:
            pools.append(cr.GeometricMeanTwoCoin(100 + 900 * rng.random(2), [0.3, 0.7], 0.997, [a, b]))
        else:
            cp = float(np.exp(rng.uniform(-1, 1)))
            lt = cp * 1.5 * np.cumprod([1.0, 0.8, 0.7, 0.6])
            pools.append(cr.UniV3(cp, lt, [100.0, 50.0, 0.0, 80.0], 0.997, [a, b]))
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n)
    ids = rng.integers(0, 30, size=60)
    T = tenders_for(np.ones((60, 2)) * 20, rng, lo=-2, hi=0)
    q = r.quote_swaps(ids, T)
    got = r.execute_swaps(ids, T)
    assert np.array_equal(q[0], got[0])  # the first row sees no earlier row
    for i, c in enumerate(pools):
        t = (P, G, U)[i % 3]
        k = r._type_lists[t].index(i)
        st = r._pools.pool_state(t, k, 1)[0]
        if t == U:
            assert c.current_price == st[0] and c.current_tick == so.current_tick(c.lower_ticks, c.current_price)
        else:
            assert np.array_equal(c.R, st[0])
    r._pools.close()
