"""cfmm_modify_univ3_liquidity / cfmm_get_univ3_ticks (include/cfmm_b200.h) on the device.

Every ladder the device reports is compared bit for bit with the row-by-row host restatement
(liquidity_oracle.py); trades with the oracle on the restated ladders, bit for bit, and quotes with
swap_oracle.univ3_swap.  Both commit paths run: batches whose boundaries all exist already (tick
counts unchanged, the liquidities are rewritten in place) and batches that grow ladders (the set's
tick arrays are spliced)."""
import numpy as np
import pytest

import liquidity_oracle as lo_
import swap_oracle as so
from test_gpu_parity import check_psi, make_pools
from test_gpu_univ3_state import Univ3Mirror, moved_prices, new_prices

pytestmark = pytest.mark.gpu

U = 2


class Mirror(Univ3Mirror):
    """Univ3Mirror with retired flags and liquidity rows replayed on the host."""

    def __init__(self, *args):
        super().__init__(*args)
        self.retired = np.zeros(len(self.cp), dtype=bool)

    def modify(self, pools, lo, hi, dL):
        off, lt, lq, bad = lo_.replay(self.off, self.lt, self.lq, pools, lo, hi, dL)
        if bad is None:
            self.off, self.lt, self.lq = off, lt, lq
        return bad

    def append(self, cp, g, Ai, off, lt, lq):
        self.off = np.concatenate([self.off, self.off[-1] + off[1:]])
        self.cp, self.g, self.Ai = np.concatenate([self.cp, cp]), np.concatenate([self.g, g]), np.concatenate([self.Ai, Ai])
        self.lt, self.lq = np.concatenate([self.lt, lt]), np.concatenate([self.lq, lq])
        self.retired = np.concatenate([self.retired, np.zeros(len(cp), dtype=bool)])

    def trades(self, oracle, v):
        D, L = self.sweep(oracle, v)
        D[self.retired] = 0.0
        L[self.retired] = 0.0
        return D, L


def check_ladders(p, mir):
    off, lt, lq = p.univ3_ticks()
    assert np.array_equal(off, mir.off), np.flatnonzero(np.diff(off) != np.diff(mir.off))[:5]
    assert np.array_equal(lt, mir.lt) and np.array_equal(lq, mir.lq)
    cp, active = p.pool_state(U)
    assert np.array_equal(cp, mir.cp) and np.array_equal(~active, mir.retired)


def check_trades(p, oracle, mir, n, vs):
    for v in vs:
        psi, acc = p.sweep(v, materialize=True)
        D, L = p.trades()
        Do, Lo = mir.trades(oracle, v)
        assert np.array_equal(D, Do), np.argwhere(D != Do)[:5]
        assert np.array_equal(L, Lo), np.argwhere(L != Lo)[:5]
        check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)


def apply(p, mir, pools, lo, hi, dL):
    pools, lo, hi, dL = (np.asarray(x) for x in (pools, lo, hi, dL))
    assert mir.modify(pools, lo, hi, dL) is None
    p.modify_univ3_liquidity(pools, lo, hi, dL)


# ---- 1. the reference pool --------------------------------------------------------------
REF_ROWS = [
    ("existing boundaries", 10.0, 20.0, 0.5),
    ("split tick 2 (holds the price)", 12.0, 18.0, 1.0),
    ("boundary at the current price", 15.0, 25.0, 0.75),
    ("above T1", 28.0, 40.0, 2.0),
    ("split the last tick", 1.0, 5.0, 0.3),
    ("burn back to zero", 1.0, 5.0, -0.3),
    ("burn above T1 back to zero", 28.0, 40.0, -2.0),
]


@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_reference_pool_rows(cr, oracle, gamma):
    cp = 15.0
    mir = Mirror(np.array([cp]), np.array([gamma]), np.array([[1, 2]]), np.array([0, 4]),
                 np.array([30.0, 20, 10, 5]), np.array([1.0, 2.0, 1.5, 0.0]))
    p = make_pools(cr, 2, univ3=mir.args)
    vs = [np.array(v, dtype=float) for v in ([15, 1], [15 * (1 + gamma) / 2, 1], [16, 1], [14, 1], [25, 1],
                                             [7.5, 1], [4, 1], [35, 1], [45, 1], [0.5, 1])]
    xs = np.concatenate([[1e-6, 0.01, 0.3, 1.0], np.geomspace(1e-3, 1e3, 12), [1e30]])
    T = np.concatenate([np.stack([xs, 0 * xs], 1), np.stack([0 * xs, xs], 1)])
    for what, a, b, d in REF_ROWS:
        ticks_before = len(mir.lt)
        apply(p, mir, [0], [a], [b], [d])
        check_ladders(p, mir)
        if what == "existing boundaries":
            assert len(mir.lt) == ticks_before
        if what.startswith("burn"):
            assert np.any(mir.lq[(mir.lt > a) & (mir.lt <= b)] == 0.0)
        assert oracle.univ3_current_tick(mir.lt, mir.cp[0]) == so.current_tick(mir.lt, mir.cp[0])
        for v in vs:
            p.sweep(v, materialize=True)
            D, L = p.trades()
            Do, Lo = oracle.univ3_arb(mir.cp[0], mir.lt, mir.lq, gamma, v)
            assert np.array_equal(D[0], Do) and np.array_equal(L[0], Lo), (what, v, D[0], Do, L[0], Lo)
        got = p.quote_swaps(U, np.zeros(len(T), dtype=np.int64), T)
        for j, t in enumerate(T):
            lam = so.univ3_swap(mir.cp[0], mir.lt, mir.lq, gamma, t)[0]
            assert got[j].tolist() == ([0.0, lam] if t[0] > 0 else [lam, 0.0]), (what, t)
        if what == "above T1":  # the new T₁ is the price bound of cfmm_update_univ3
            p.update_univ3(0, [40.0])
            mir.cp[0] = 40.0
            check_trades(p, oracle, mir, 2, vs[:3])
            with pytest.raises(cr.CFMMError) as e:
                p.update_univ3(0, [np.nextafter(40.0, np.inf)])
            assert e.value.code == -1
            p.update_univ3(0, [cp])
            mir.cp[0] = cp
    assert mir.lt.tolist() == [40, 30, 28, 25, 20, 18, 15, 12, 10, 5, 1]
    p.close()


# ---- 2. a ragged set with a tail and retired pools ------------------------------------------
def ragged_set(cr, synth, m=20_000, mt=3_000, n=60):
    mir = Mirror(*synth.univ3_pools(m, n, seed=71, ragged=True))
    p = make_pools(cr, n, univ3=mir.args)
    tail = synth.univ3_pools(mt, n, seed=72, ragged=True)
    p.append_univ3(*tail)
    mir.append(*tail)
    flags = np.ones(m + mt, dtype=bool)
    flags[::97] = False
    flags[m + 5::89] = False
    p.set_active(U, 0, flags)
    mir.retired = ~flags
    return p, mir, n


def burn_of(rows, rng, burned):
    """A burn of an earlier mint of the batch: exactly what it minted the first time its pool is
    burned (the header's guarantee holds: only mints before it on those ticks), half of it after
    that (a second exact burn could meet a tick that an earlier exact burn rounded down).  Each
    mint is burned at most once."""
    k = int(rng.integers(0, len(rows)))
    i, a, b, d = rows[k]
    if d <= 0 or ("row", k) in burned:
        return None
    row = (i, a, b, -d if ("pool", i) not in burned else -0.5 * d)
    burned.update({("pool", i), ("row", k)})
    return row


def rows_on_boundaries(mir, rng, q):
    """Rows whose lo and hi are boundaries of the pool's ladder already; every third row burns an
    earlier mint."""
    multi = np.flatnonzero(np.diff(mir.off) >= 2)
    rows, burned = [], set()
    while len(rows) < q:
        if rows and len(rows) % 3 == 2:
            row = burn_of(rows, rng, burned)
            if row:
                rows.append(row)
                continue
        i = int(rng.choice(multi[:200])) if rng.random() < 0.3 else int(rng.choice(multi))
        lt = mir.lt[mir.ticks(i)]
        x, y = np.sort(rng.choice(len(lt), size=2, replace=False))
        rows.append((i, lt[y], lt[x], float(rng.uniform(0.5, 50.0))))
    return rows


def rows_mixed(mir, rng, q):
    """Rows with new boundaries: inside ticks, at the current price, above T₁, below the last tick,
    on existing boundaries; burns of earlier mints; a few pools with many rows."""
    m = len(mir.cp)
    hot = [3 % m, 11 % m, m - 2, max(m - 700, 0)]  # (the last two: appended pools, when there are any)
    rows, burned = [], set()
    while len(rows) < q:
        k = len(rows) % 7
        if rows and k == 6:
            row = burn_of(rows, rng, burned)
            if row:
                rows.append(row)
                continue
        i = int(rng.choice(hot)) if rng.random() < 0.25 else int(rng.integers(0, m))
        lt = mir.lt[mir.ticks(i)]
        cp = mir.cp[i]
        if k == 0:
            a, b = lt[-1] * rng.uniform(0.1, 0.9), lt[0] * rng.uniform(0.2, 0.95)   # inside / below
        elif k == 1:
            a, b = cp, lt[0] * rng.uniform(1.01, 3.0)                                # at the price, above T₁
        elif k == 2:
            a, b = lt[-1] * rng.uniform(0.1, 0.9), lt[-1]                             # below the last tick
        elif k == 3:
            a, b = np.sort(lt[rng.integers(0, len(lt), size=2)]) if len(lt) > 1 else (lt[0] * 0.5, lt[0])
            if a == b:
                a = a * 0.5
        elif k == 4:
            a, b = lt[0] * rng.uniform(1.01, 2.0), lt[0] * rng.uniform(2.5, 4.0)     # wholly above T₁
        else:
            a, b = np.sort(np.exp(rng.uniform(np.log(lt[-1] * 0.5), np.log(lt[0] * 1.5), size=2)))
        if not a < b:
            continue
        rows.append((i, float(a), float(b), float(rng.uniform(0.1, 100.0))))
    return rows


def run_rows(p, mir, rows):
    pools, lo, hi, dL = (np.array(c) for c in zip(*rows))
    apply(p, mir, pools.astype(np.int64), lo, hi, dL)


def test_ragged_set_in_place_then_splice(cr, oracle, synth):
    p, mir, n = ragged_set(cr, synth)
    vs = [synth.dual_prices(n, k, seed=s) for k, s in (("near", 1), ("wide", 2), ("wide", 3))]
    rng = np.random.default_rng(5)
    cp0, off0 = mir.cp.copy(), mir.off.copy()
    run_rows(p, mir, rows_on_boundaries(mir, rng, 20_000))
    assert np.array_equal(mir.off, off0)          # tick counts unchanged: the in-place path
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, vs)
    run_rows(p, mir, rows_mixed(mir, rng, 20_000))
    assert mir.off[-1] > off0[-1] + 10_000         # grown ladders: the splice path
    assert np.array_equal(mir.cp, cp0)
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, vs)
    # a context built afresh from the read-back state trades the same
    off, lt, lq = p.univ3_ticks()
    cp, active = p.pool_state(U)
    fresh = make_pools(cr, n, univ3=(cp, mir.g, mir.Ai, off, lt, lq))
    fresh.set_active(U, 0, active)
    for v in vs:
        p.sweep(v, materialize=True)
        fresh.sweep(v, materialize=True)
        D, L = p.trades()
        Df, Lf = fresh.trades()
        assert np.array_equal(D, Df) and np.array_equal(L, Lf)
    # retired pools take the change and trade once restored
    p.set_active(U, 0, np.ones(len(mir.cp), dtype=bool))
    mir.retired[:] = False
    check_trades(p, oracle, mir, n, vs[:1])
    p.close()
    fresh.close()


# ---- 3. rejections --------------------------------------------------------------------------
def test_rejections_change_nothing(cr, oracle, synth):
    p, mir, n = ragged_set(cr, synth, m=4000, mt=500)
    v = synth.dual_prices(n, "wide", seed=4)
    p.sweep(v, materialize=True)
    D0, L0 = p.trades()
    psi0, acc0 = p.sweep(v)
    off0, lt0, lq0 = p.univ3_ticks()
    cp0, _ = p.pool_state(U)
    t = 4000 + 17  # an appended pool
    lt_t = mir.lt[mir.ticks(t)]
    lt_3 = mir.lt[mir.ticks(3)]
    rows = [(3, lt_3[-1] * 0.5, lt_3[0] * 2, 5.0),          # 0 grows pool 3
            (8, mir.cp[8], mir.lt[mir.off[8]] * 1.5, 1.0),    # 1 another pool
            (t, lt_t[-1] * 0.3, lt_t[0] * 1.2, 2.0),          # 2 the tail
            (3, lt_3[-1] * 0.7, lt_3[0] * 1.5, -5.0),         # 3 fine: burns what row 0 minted
            (t, lt_t[-1] * 0.3, lt_t[0] * 1.2, -1e9),         # 4 the first row that fails (tail)
            (3, lt_3[-1] * 0.5, lt_3[0] * 2, -1e9),           # 5 fails too (main set)
            (9, 1.0, 2.0, 1.0)]
    pools, lo, hi, dL = (np.array(c) for c in zip(*rows))
    assert mir.modify(pools.astype(np.int64), lo, hi, dL) == 4
    with pytest.raises(cr.CFMMError) as e:
        p.modify_univ3_liquidity(pools, lo, hi, dL)
    assert e.value.code == -1 and "row 4 " in e.value.message, e.value.message
    # every invalid argument, each inside an otherwise valid batch
    m = len(mir.cp)
    good = (np.array([1, 2, 3]), np.array([1.0, 2.0, 3.0]), np.array([2.0, 3.0, 4.0]), np.array([1.0, 1.0, 1.0]))
    bad_cases = [("pool", -1), ("pool", m), ("lo", np.nan), ("lo", np.inf), ("hi", np.inf), ("hi", np.nan),
                 ("lo", 0.0), ("lo", -1.0), ("lo", 3.0), ("lo", 3.5), ("dL", 0.0), ("dL", np.nan), ("dL", -np.inf)]
    for field, val in bad_cases:
        args = [a.copy() for a in good]
        k = ["pool", "lo", "hi", "dL"].index(field)
        args[k] = args[k].astype(np.int64 if k == 0 else float)
        args[k][1] = val
        with pytest.raises(cr.CFMMError) as e:
            p.modify_univ3_liquidity(*args)
        assert e.value.code == -1 and "row 1" in e.value.message, (field, val, e.value.message)
    p.modify_univ3_liquidity([], [], [], [])  # q == 0: nothing happens
    off, lt, lq = p.univ3_ticks()
    cp, _ = p.pool_state(U)
    assert np.array_equal(off, off0) and np.array_equal(lt, lt0) and np.array_equal(lq, lq0)
    assert np.array_equal(cp, cp0)
    psi, acc = p.sweep(v)
    Do, Lo = mir.trades(oracle, v)
    check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)
    assert np.allclose(psi, psi0, rtol=1e-12, atol=1e-12 * np.max(np.abs(psi0)))
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, D0) and np.array_equal(L, L0)
    p.close()
    q = cr.DevicePools(4)
    q.add_univ3(*synth.univ3_pools(10, 4, seed=1))
    with pytest.raises(cr.CFMMError) as e:
        q.modify_univ3_liquidity([0], [1.0], [2.0], [1.0])
    assert e.value.code == -3
    q.close()


# ---- 4. interactions --------------------------------------------------------------------------
def test_interactions(cr, oracle, synth):
    mir = Mirror(*synth.univ3_pools(6000, 40, seed=81, ragged=True))
    n = 40
    p = make_pools(cr, n, univ3=mir.args)
    v = synth.dual_prices(n, "wide", seed=8)
    rng = np.random.default_rng(8)
    # a graph captured before the change replays the new ladders
    for _ in range(6):
        psi0, _ = p.sweep(v)
    run_rows(p, mir, rows_mixed(mir, rng, 3000))
    psi, acc = p.sweep(v)
    Do, Lo = mir.trades(oracle, v)
    check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)
    assert not np.array_equal(psi, psi0)
    # a cfmm_update_univ3 liquidity push in the new CSR order
    lo, hi = 1000, 3000
    t0, t1 = mir.off[lo], mir.off[hi]
    lq = mir.lq[t0:t1] * rng.uniform(0.5, 1.5, size=t1 - t0)
    p.update_univ3(lo, liquidity=lq, count=hi - lo)
    mir.lq[t0:t1] = lq
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, [v])
    # cfmm_apply_trades clamps to the new T₁: pools whose T₁ grew, driven far above it
    grown = np.arange(0, 6000, 50)
    apply(p, mir, grown, mir.t1[grown] * 1.5, mir.t1[grown] * 3.0, np.full(len(grown), 5.0))
    v2 = v.copy()
    v2[mir.Ai[grown[0], 0] - 1] *= 1e6
    p.sweep(v2, materialize=True)
    p.apply_trades()
    q0 = mir.cp.copy()
    mir.cp = np.where(mir.retired, mir.cp, moved_prices(mir.cp, mir.g, mir.t1, v2[mir.Ai[:, 0] - 1],
                                                        v2[mir.Ai[:, 1] - 1]))
    assert np.any(mir.cp[grown] == mir.t1[grown]) and np.any(mir.cp[grown] > q0[grown])
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, [v])
    # cfmm_execute_swaps after a change
    run_rows(p, mir, rows_mixed(mir, rng, 500))
    pools = rng.integers(0, 6000, size=2000)
    T = np.zeros((2000, 2))
    T[np.arange(2000), rng.integers(0, 2, size=2000)] = 10.0 ** rng.uniform(-3, 2, size=2000)
    got = p.execute_swaps(U, pools, T)
    for j, i in enumerate(pools):
        s = mir.ticks(i)
        lam, q = so.univ3_swap(mir.cp[i], mir.lt[s], mir.lq[s], mir.g[i], T[j])
        assert got[j].tolist() == ([0.0, lam] if T[j, 0] > 0 else [lam, 0.0]), (j, i)
        mir.cp[i] = q
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, [v])
    # cfmm_compact keeps ladders and trades, tails included
    tail = synth.univ3_pools(700, n, seed=82, ragged=True)
    p.append_univ3(*tail)
    mir.append(*tail)
    run_rows(p, mir, rows_mixed(mir, rng, 2000))
    check_trades(p, oracle, mir, n, [v])
    p.compact()
    assert p.pool_set_info(U)["tail"] == 0
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, [v])
    run_rows(p, mir, rows_mixed(mir, rng, 2000))
    check_ladders(p, mir)
    check_trades(p, oracle, mir, n, [v])
    p.close()


def test_solve_after_change(cr):
    """Router.modify_liquidity, then route! on the device and on the host reach the same optimum."""
    rng = np.random.default_rng(12)
    n = 8
    pools = []
    for _ in range(60):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        pools.append(cr.ProductTwoCoin(1000 * rng.random(2) + 10, 0.997, [a, b]))
    for _ in range(12):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        cp = float(np.exp(rng.uniform(-0.5, 0.5)))
        pools.append(cr.UniV3(cp, cp * np.array([2.0, 1.3, 0.8, 0.5]), [20.0, 50.0, 40.0, 10.0], 0.997, [a, b]))
    c = rng.random(n) + 0.5
    ids = np.arange(60, 72)
    lt0 = np.array([pools[i].lower_ticks[0] for i in ids])
    rs = []
    for optimizer in ("device", "host"):
        cs = []
        for q in pools:
            if isinstance(q, cr.UniV3):
                cs.append(cr.UniV3(q.current_price, q.lower_ticks, q.liquidity, q.gamma, q.Ai))
            else:
                cs.append(cr.ProductTwoCoin(q.R, q.gamma, q.Ai))
        r = cr.Router(cr.LinearNonnegative(c), cs, n)
        r.modify_liquidity(ids, lt0 * 0.6, lt0 * 1.7, np.full(len(ids), 30.0))
        r.modify_liquidity(ids[::2], lt0[::2] * 0.6, lt0[::2] * 1.7, np.full(len(ids[::2]), -30.0))
        assert len(cs[60].lower_ticks) == 6 and cs[60].lower_ticks[0] == lt0[0] * 1.7
        cr.route(r, optimizer=optimizer)
        psi, acc = r._pools.sweep(r.v)
        rs.append((r, r.objective.f(r.v) + acc, float(c @ cr.netflows(r))))
    (rd, gd, pd), (rh, gh, ph) = rs
    assert abs(gd - gh) <= 1e-5 * max(1.0, abs(gh)), (gd, gh)
    assert abs(pd - ph) <= 1e-3 * max(1.0, abs(ph)), (pd, ph)
    for r in (rd, rh):  # the device ladders are the host objects' after the refresh
        off, lt, lq = r._pools.univ3_ticks()
        assert np.array_equal(lt, np.concatenate([r.cfmms[i].lower_ticks for i in ids]))
        assert np.array_equal(lq, np.concatenate([r.cfmms[i].liquidity for i in ids]))


# ---- 5. state-machine fuzz --------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_operation_sequences(cr, oracle, synth, seed):
    rng = np.random.default_rng(2000 + seed)
    n = int(rng.integers(10, 80))
    mir = Mirror(*synth.univ3_pools(int(rng.integers(200, 3000)), n, seed=600 + seed, ragged=True))
    p = make_pools(cr, n, univ3=mir.args)
    v = synth.dual_prices(n, "wide", seed=seed)
    ops = ["modify", "modify", "modify", "price", "liq", "execute", "apply", "append", "retire", "compact"]
    check_trades(p, oracle, mir, n, [v])
    for step in range(14):
        op = str(rng.choice(ops))
        m = len(mir.cp)
        if op == "modify":
            run_rows(p, mir, rows_mixed(mir, rng, int(rng.integers(1, 600))))
        elif op == "price":
            lo = int(rng.integers(0, m))
            hi = int(rng.integers(lo, m)) + 1
            cp = new_prices(mir, lo, hi, rng)
            p.update_univ3(lo, cp)
            mir.cp[lo:hi] = cp
        elif op == "liq":
            lo = int(rng.integers(0, m))
            hi = int(rng.integers(lo, m)) + 1
            t0, t1 = mir.off[lo], mir.off[hi]
            lq = mir.lq[t0:t1] * rng.uniform(0.5, 1.5, size=t1 - t0)
            lq[rng.random(t1 - t0) < 0.1] = 0.0
            p.update_univ3(lo, liquidity=lq, count=hi - lo)
            mir.lq[t0:t1] = lq
        elif op == "execute":
            q = int(rng.integers(1, 300))
            pools = rng.integers(0, m, size=q)
            T = np.zeros((q, 2))
            T[np.arange(q), rng.integers(0, 2, size=q)] = 10.0 ** rng.uniform(-3, 2, size=q)
            got = p.execute_swaps(U, pools, T)
            for j, i in enumerate(pools):
                if mir.retired[i]:
                    assert got[j].tolist() == [0.0, 0.0]
                    continue
                s = mir.ticks(i)
                lam, mir.cp[i] = so.univ3_swap(mir.cp[i], mir.lt[s], mir.lq[s], mir.g[i], T[j])
                assert got[j].tolist() == ([0.0, lam] if T[j, 0] > 0 else [lam, 0.0])
        elif op == "apply":  # by the ν of the last check's materialising sweep
            p.apply_trades()
            mir.cp = np.where(mir.retired, mir.cp, moved_prices(mir.cp, mir.g, mir.t1, v[mir.Ai[:, 0] - 1],
                                                                v[mir.Ai[:, 1] - 1]))
        elif op == "append":
            tail = synth.univ3_pools(int(rng.integers(1, 300)), n, seed=700 + 10 * seed + step, ragged=True)
            p.append_univ3(*tail)
            mir.append(*tail)
        elif op == "retire":
            lo = int(rng.integers(0, m))
            flags = rng.random(min(m - lo, 200)) < 0.5
            p.set_active(U, lo, flags)
            mir.retired[lo:lo + len(flags)] = ~flags
        else:
            p.compact()
        check_ladders(p, mir)
        v = synth.dual_prices(n, str(rng.choice(["near", "wide"])), seed=int(rng.integers(1 << 30)))
        check_trades(p, oracle, mir, n, [v])
    p.close()
