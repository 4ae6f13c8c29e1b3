"""UniV3 pool state on the device: cfmm_update_univ3 (price / liquidity pushes), the device
rebuild of the tick records, and cfmm_apply_trades on sets that hold UniV3 pools.

Every check runs the oracle on a host mirror of the pool state: materialising sweeps must give
the oracle's Δ, Λ bit for bit, gradient-only sweeps pass check_psi (on token-disjoint sets Ψ is
compared per pool, bit for bit).  The mirror moves UniV3 prices by the rule documented at
cfmm_apply_trades (include/cfmm_b200.h), written out here in numpy."""
import numpy as np
import pytest

from test_gpu_parity import EPS, check_psi, make_pools

pytestmark = pytest.mark.gpu


def moved_prices(cp, g, t1, va, vb):
    """q′ of cfmm_apply_trades, elementwise (one IEEE operation per step, as on the device)."""
    with np.errstate(all="ignore"):
        p = va / vb
        lo = g * cp
        band = (lo <= p) & (p <= cp / g)
        target = np.where(p < lo, p / g, g * p)
        move = ~band & (target > 0.0)  # (NaN > 0 is False)
        return np.where(move, np.minimum(np.where(move, target, 0.0), t1), cp)


class Univ3Mirror:
    """Host copy of a UniV3 pool set (insertion order, ingest CSR)."""

    def __init__(self, cp, g, Ai, off, lt, lq):
        self.cp, self.g, self.Ai = cp.astype(float).copy(), g.astype(float).copy(), Ai.copy()
        self.off, self.lt, self.lq = off.copy(), lt.astype(float).copy(), lq.astype(float).copy()

    @property
    def args(self):
        return self.cp, self.g, self.Ai, self.off, self.lt, self.lq

    @property
    def t1(self):
        return self.lt[self.off[:-1]]

    def ticks(self, i):
        return slice(self.off[i], self.off[i + 1])

    def sweep(self, oracle, v):
        return oracle.sweep_univ3(*self.args, v, threads=8)

    def move(self, v):
        self.cp = moved_prices(self.cp, self.g, self.t1, v[self.Ai[:, 0] - 1], v[self.Ai[:, 1] - 1])

    def totals(self, oracle, i, cp=None):
        """(token totals (R1, R2) over pool i's ticks, Σ of R + α / R + β over its ticks)."""
        cp = self.cp[i] if cp is None else cp
        lt, lq = self.lt[self.ticks(i)], self.lq[self.ticks(i)]
        tot, vir = np.zeros(2), np.zeros(2)
        for idx in range(1, len(lt) + 1):
            k, a, b, R1, R2 = oracle.univ3_tick(cp, lt, lq, idx)
            tot += [R1, R2]
            vir += [abs(R1) + abs(a), abs(R2) + abs(b)]
        return tot, vir


def univ3_set(synth, kind, m):
    """(mirror, n_tokens, ν list) of one of the three test sets."""
    if kind == "disjoint":
        cp, g, Ai, off, lt, lq, v = synth.disjoint_univ3(m, seed=7, ragged=True)
        n = 2 * m
        rng = np.random.default_rng(8)
        vs = [v, v * np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n))]
    else:
        n = 60
        cp, g, Ai, off, lt, lq = synth.univ3_pools(m, n, seed=11, ragged=kind == "ragged")
        rng = np.random.default_rng(9)
        vs = [np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n)) for _ in range(2)] + [synth.dual_prices(n, "wide")]
    return Univ3Mirror(cp, g, Ai, off, lt, lq), n, vs


def check_state(p, oracle, mir, n, vs, disjoint=False):
    for v in vs:
        psi, acc = p.sweep(v, materialize=True)
        D, L = p.trades()
        Do, Lo = mir.sweep(oracle, v)
        assert np.array_equal(D, Do), np.argwhere(D != Do)[:5]
        assert np.array_equal(L, Lo), np.argwhere(L != Lo)[:5]
        check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)
        psi, acc = p.sweep(v)
        if disjoint:  # Ψ[2i+1], Ψ[2i+2] are pool i's own Λ − Δ: no summation order involved
            assert np.array_equal(psi, (Lo - Do).reshape(-1))
        check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)


def new_prices(mir, lo, hi, rng):
    """Prices for pools [lo, hi): ties with a lower tick, exactly T₁, inside an empty tick,
    random inside the ladder, cycling."""
    out = np.empty(hi - lo)
    for j, i in enumerate(range(lo, hi)):
        lt, lq = mir.lt[mir.ticks(i)], mir.lq[mir.ticks(i)]
        case = j % 4
        if case == 0:
            out[j] = lt[rng.integers(0, len(lt))]                  # tie: counts as >= (that tick is current)
        elif case == 1:
            out[j] = lt[0]                                          # exactly T₁
        elif case == 2 and np.any(lq == 0.0):
            k = int(np.flatnonzero(lq == 0.0)[0])                   # inside an empty tick
            out[j] = 0.5 * (lt[k] + lt[k + 1]) if k + 1 < len(lt) else 0.5 * lt[k]
        else:
            out[j] = lt[-1] * np.exp(rng.uniform(np.log(0.3), np.log(lt[0] / lt[-1])))
    return np.minimum(out, mir.t1[lo:hi])


@pytest.mark.parametrize("kind,m", [("regular", 3000), ("ragged", 3000), ("disjoint", 400)])
def test_price_and_liquidity_pushes(cr, oracle, synth, kind, m):
    mir, n, vs = univ3_set(synth, kind, m)
    p = make_pools(cr, n, univ3=mir.args)
    check_state(p, oracle, mir, n, vs[:1], disjoint=kind == "disjoint")
    rng = np.random.default_rng(len(kind))
    # prices of a sub-range
    lo, hi = m // 5, m // 5 + m // 2
    cp = new_prices(mir, lo, hi, rng)
    p.update_univ3(lo, cp)
    mir.cp[lo:hi] = cp
    check_state(p, oracle, mir, n, vs, disjoint=kind == "disjoint")
    # liquidity of another sub-range: zero some ticks, refill the empty ones, rescale the rest
    lo, hi = m // 3, m - 7
    t0, t1 = mir.off[lo], mir.off[hi]
    lq = mir.lq[t0:t1].copy()
    empty = lq == 0.0
    lq[empty] = rng.uniform(1.0, 500.0, size=int(empty.sum()))
    lq[~empty] *= rng.uniform(0.5, 2.0, size=int((~empty).sum()))
    lq[rng.random(len(lq)) < 0.2] = 0.0
    p.update_univ3(lo, liquidity=lq, count=hi - lo)
    mir.lq[t0:t1] = lq
    check_state(p, oracle, mir, n, vs, disjoint=kind == "disjoint")
    # both at once, the whole set
    cp = new_prices(mir, 0, m, rng)
    lq = mir.lq * rng.uniform(0.8, 1.25, size=len(mir.lq))
    p.update_univ3(0, cp, lq)
    mir.cp[:], mir.lq[:] = cp, lq
    check_state(p, oracle, mir, n, vs, disjoint=kind == "disjoint")
    p.close()


def test_fresh_context_equivalence(cr, oracle, synth):
    """After pushes and trade applications, trades equal those of a context built afresh."""
    mir, n, vs = univ3_set(synth, "ragged", 5000)
    p = make_pools(cr, n, univ3=mir.args)
    rng = np.random.default_rng(3)
    for step in range(3):
        lo = int(rng.integers(0, 2000))
        cp = new_prices(mir, lo, lo + 2500, rng)
        p.update_univ3(lo, cp)
        mir.cp[lo:lo + 2500] = cp
        p.sweep(vs[step], materialize=True)
        p.apply_trades()
        mir.move(vs[step])
        t0, t1 = mir.off[lo], mir.off[lo + 1000]
        lq = mir.lq[t0:t1] * rng.uniform(0.5, 1.5, size=t1 - t0)
        p.update_univ3(lo, liquidity=lq, count=1000)
        mir.lq[t0:t1] = lq
    fresh = make_pools(cr, n, univ3=mir.args)
    for v in vs:
        p.sweep(v, materialize=True)
        fresh.sweep(v, materialize=True)
        D, L = p.trades()
        Df, Lf = fresh.trades()
        assert np.array_equal(D, Df) and np.array_equal(L, Lf)
        Do, Lo = mir.sweep(oracle, v)
        assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    p.close()
    fresh.close()


def test_rejected_pushes_change_nothing(cr, oracle, synth):
    mir, n, vs = univ3_set(synth, "ragged", 2000)
    p = make_pools(cr, n, univ3=mir.args)
    v = vs[0]
    p.sweep(v, materialize=True)
    D0, L0 = p.trades()
    good = mir.cp[100:200] * 0.9
    bad_cases = []
    above = good.copy()
    above[57] = np.nextafter(mir.t1[157], np.inf)      # one pool just above its T₁
    bad_cases.append((100, above, "pool 157"))
    nan = good.copy()
    nan[3] = np.nan
    bad_cases.append((100, nan, "pool 103"))
    for first, cp, what in bad_cases:
        with pytest.raises(cr.CFMMError) as e:
            p.update_univ3(first, cp, mir.lq[mir.off[first]:mir.off[first + len(cp)]] * 2)
        assert e.value.code == -1 and what in e.value.message
    for first, count in ((-1, 5), (1990, 11), (2001, 0)):
        with pytest.raises(cr.CFMMError) as e:
            p.update_univ3(first, np.full(count, 1e-9))
        assert e.value.code == -1
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, D0) and np.array_equal(L, L0)
    check_state(p, oracle, mir, n, vs)
    p.close()


def table_nu(mir, rng):
    """Per-pool prices of a token-disjoint set covering every row of the table."""
    m = len(mir.cp)
    v = np.ones(2 * m)
    cases = ["band", "band_lo", "band_hi", "up", "down", "above_T1", "drain", "nan", "zero_a", "zero_b"]
    kinds = []
    for i in range(m):
        c = cases[i % len(cases)]
        q, g, lt = mir.cp[i], mir.g[i], mir.lt[mir.ticks(i)]
        if c == "band":
            pa = q
        elif c == "band_lo":
            pa = g * q
        elif c == "band_hi":
            pa = q / g
        elif c == "up":
            pa = q * rng.uniform(0.4, 0.95)
        elif c == "down":
            pa = q * rng.uniform(1.05, 2.5)
        elif c == "above_T1":
            pa = lt[0] * 1e3                     # the lower walk drains tick 1: clamp to T₁
        elif c == "drain":
            pa = lt[-1] * 1e-3                   # the upper walk runs into the trailing ticks
        elif c == "nan":
            pa = np.nan
        elif c == "zero_a":
            pa = 0.0                             # target 0: unchanged
        else:
            pa, v[2 * i + 1] = 1.0, 0.0          # p = inf: the lower walk, clamped to T₁
        v[2 * i] = pa
        kinds.append(c)
    return v, np.array(kinds)


def test_apply_trades_table_rows(cr, oracle, synth):
    """Every row of the table on a token-disjoint set, the consistency of the moved state with
    the reference's reserve update, and idempotence."""
    m = 600
    cp, g, Ai, off, lt, lq, _ = synth.disjoint_univ3(m, seed=21, ragged=True, adversarial=False)
    lq[off[1:] - 1] = 0.0  # trailing empty ticks: a downward walk drains into them
    mir = Univ3Mirror(cp, g, Ai, off, lt, lq)
    n = 2 * m
    p = make_pools(cr, n, univ3=mir.args)
    v, kinds = table_nu(mir, np.random.default_rng(4))
    p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = mir.sweep(oracle, v)
    real = kinds != "nan"  # (a NaN ν is only asked to leave the price alone)
    assert np.array_equal(D[real], Do[real]) and np.array_equal(L[real], Lo[real])
    before = Univ3Mirror(*mir.args)
    p.apply_trades()
    mir.move(v)
    q0, q1 = before.cp, mir.cp
    t1 = mir.t1
    assert np.all(q1[np.isin(kinds, ["band", "band_lo", "band_hi", "nan", "zero_a"])] ==
                  q0[np.isin(kinds, ["band", "band_lo", "band_hi", "nan", "zero_a"])])
    assert np.all(q1[np.isin(kinds, ["above_T1", "zero_b"])] == t1[np.isin(kinds, ["above_T1", "zero_b"])])
    up = kinds == "up"
    assert np.array_equal(q1[up], v[2 * np.flatnonzero(up)] / g[up])
    down = kinds == "down"
    assert np.array_equal(q1[down], np.minimum(g[down] * v[2 * np.flatnonzero(down)], t1[down]))
    drain = kinds == "drain"
    assert np.all(q1[drain] < lt[off[1:][drain] - 1])  # below the last lower tick
    # the device moved exactly as the mirror: bit-exact trades at new prices
    rng = np.random.default_rng(5)
    v2 = np.nan_to_num(v, nan=1.0, posinf=1.0)
    v2[v2 == 0.0] = 1.0
    v2 = v2 * np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n))
    check_state(p, oracle, mir, n, [v2], disjoint=True)
    # consistency with R⁺ = R + γΔ − Λ (test/cfmms.jl:10): the token totals over the ticks move by
    # γΔ − Λ.  Rounding: every tick reserve R = sqrt(k/p) − α (or sqrt(k·p) − β) is within
    # 2 eps·(R + α) of its exact value, the tick sums add eps·Σ per tick, and Δ = dsum/γ, γ·Δ add
    # 2 eps·γ|Δ|: 4·nt·eps·(Σ(R + α) at q + Σ(R + α) at q′ + γ|Δ| + |Λ|) per token bounds the gap.
    # Not for ν[a] = 0: the walk to price 0 drains every tick, but the table keeps the price
    # (a target that is not > 0 names no price a pool can hold).
    moves = real & (kinds != "zero_a")
    for i in np.flatnonzero(moves & (np.any(D != 0, axis=1) | np.any(L != 0, axis=1))):
        T0, V0 = before.totals(oracle, i)
        T1, V1 = mir.totals(oracle, i)
        nt = mir.off[i + 1] - mir.off[i]
        flow = g[i] * D[i] - L[i]
        bound = 4 * nt * EPS * (V0 + V1 + np.abs(g[i] * D[i]) + np.abs(L[i]))
        gap = np.abs((T1 - T0) - flow)
        assert np.all(gap <= bound), (i, kinds[i], gap, bound)
        assert np.all(gap <= 1e-9 * (T0 + T1 + np.abs(flow)) + 1e-300), (i, kinds[i], gap)
    # idempotence: at the same ν the moved pools trade (almost) nothing
    vv = np.nan_to_num(v, nan=1.0)
    p.sweep(vv, materialize=True)
    D2, L2 = p.trades()
    for i in np.flatnonzero(moves):
        T, _ = mir.totals(oracle, i)
        cap = 1e-9 * max(T[0], T[1], 1e-300)
        assert np.all(D2[i] <= cap) and np.all(L2[i] <= cap), (i, kinds[i], D2[i], L2[i], T)
    p.close()


def test_apply_trades_mixed_set(cr, oracle, synth):
    """Product + GeometricMean + UniV3: the two-coin pools get R + γΔ − Λ, the UniV3 pools move;
    the next sweeps match the oracle on the mirror."""
    n = 50
    R, g, Ai = synth.product_pools(20_000, n, seed=31)
    Rg, gg, Ag, wg = synth.geomean_pools(5_000, n, seed=32)
    mir = Univ3Mirror(*synth.univ3_pools(8_000, n, seed=33, ragged=True))
    v = synth.dual_prices(n, "wide")
    v[7] = 1e6    # pools on token 8: far above / below every tick (T₁ clamp, drain)
    p = make_pools(cr, n, product=(R, g, Ai), geomean=(Rg, gg, Ag, wg), univ3=mir.args)
    p.sweep(v, materialize=True)
    D, L = p.trades()
    mp, mg = len(g), len(gg)
    p.apply_trades()
    R2 = R + g[:, None] * D[:mp] - L[:mp]
    Rg2 = Rg + gg[:, None] * D[mp:mp + mg] - L[mp:mp + mg]
    q0 = mir.cp.copy()
    mir.move(v)
    on8 = np.any(mir.Ai == 8, axis=1)
    assert np.any(mir.cp[on8] == mir.t1[on8]) and np.any(mir.cp[on8] < q0[on8])
    assert np.any(mir.cp != q0) and np.any(mir.cp == q0)
    for v2 in (synth.dual_prices(n, "near"), v):
        psi, acc = p.sweep(v2, materialize=True)
        Dn, Ln = p.trades()
        Do, Lo = oracle.sweep_product(R2, g, Ai, v2, threads=8)
        assert np.array_equal(Dn[:mp], Do) and np.array_equal(Ln[:mp], Lo)
        Dg, Lg = oracle.sweep_geomean(Rg2, gg, Ag, wg, v2, threads=8)
        tol = 1e-12 * (np.max(Rg2, axis=1) / gg)[:, None]
        assert np.all(np.abs(Dn[mp:mp + mg] - Dg) <= tol) and np.all(np.abs(Ln[mp:mp + mg] - Lg) <= tol)
        Du, Lu = mir.sweep(oracle, v2)
        assert np.array_equal(Dn[mp + mg:], Du) and np.array_equal(Ln[mp + mg:], Lu)
        check_psi(oracle, np.concatenate([Ai, Ag, mir.Ai]), Dn, Ln, v2, n, psi, acc)
    p.close()


def test_solve_then_apply(cr, oracle, synth):
    """cfmm_solve materialises at its final ν; cfmm_apply_trades moves the pools by that ν."""
    n = 20
    R, g, Ai = synth.product_pools(2000, n, seed=41)
    mir = Univ3Mirror(*synth.univ3_pools(1000, n, seed=42, ragged=True))
    p = make_pools(cr, n, product=(R, g, Ai), univ3=mir.args)
    c = synth.objective_prices(n)
    x, info = p.solve(c + 1e-8)
    D, L = p.trades()
    p.sweep(np.ones(n))  # a later gradient sweep does not change what apply_trades uses
    p.apply_trades()
    mir.move(x)
    R2 = R + g[:, None] * D[:2000] - L[:2000]
    v2 = synth.dual_prices(n, "wide")
    p.sweep(v2, materialize=True)
    Dn, Ln = p.trades()
    Do, Lo = oracle.sweep_product(R2, g, Ai, v2)
    Du, Lu = mir.sweep(oracle, v2)
    assert np.array_equal(Dn, np.concatenate([Do, Du])) and np.array_equal(Ln, np.concatenate([Lo, Lu]))
    p.close()


def test_sweep_device_then_overwrite_nu(cr, oracle, synth):
    """The caller's d_v may change between the materialising sweep and cfmm_apply_trades."""
    torch = pytest.importorskip("torch")
    mir, n, vs = univ3_set(synth, "ragged", 4000)
    p = make_pools(cr, n, univ3=mir.args)
    dev = torch.device("cuda", 0)
    d_v = torch.tensor(vs[0], dtype=torch.float64, device=dev)
    d_out = torch.zeros(n + 1, dtype=torch.float64, device=dev)
    torch.cuda.synchronize()
    p.sweep_device(d_v.data_ptr(), d_out.data_ptr(), materialize=True)
    p.trades()  # (synchronises the context's stream)
    d_v.fill_(123.0)
    torch.cuda.synchronize()
    p.apply_trades()
    mir.move(vs[0])
    check_state(p, oracle, mir, n, vs[1:])
    p.close()


def test_graph_replay_sees_updates(cr, oracle, synth):
    """Once cfmm_sweep replays a captured graph, a push or an apply shows in the very next sweep."""
    mir, n, vs = univ3_set(synth, "regular", 3000)
    p = make_pools(cr, n, univ3=mir.args)
    v = vs[0]
    for _ in range(6):
        psi0, acc0 = p.sweep(v)
    Do, Lo = mir.sweep(oracle, v)
    check_psi(oracle, mir.Ai, Do, Lo, v, n, psi0, acc0)
    cp = mir.cp * 0.8
    p.update_univ3(0, cp)
    mir.cp[:] = cp
    psi, acc = p.sweep(v)
    Do, Lo = mir.sweep(oracle, v)
    check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)
    assert not np.array_equal(psi, psi0)
    for _ in range(6):
        p.sweep(v)
    p.sweep(vs[1], materialize=True)
    p.apply_trades()
    mir.move(vs[1])
    psi, acc = p.sweep(v)
    Do, Lo = mir.sweep(oracle, v)
    check_psi(oracle, mir.Ai, Do, Lo, v, n, psi, acc)
    p.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_univ3_operation_sequences(cr, oracle, synth, seed):
    """State-machine fuzz over a mixed set: gradient / materialising sweeps, UniV3 price and
    liquidity pushes, two-coin pushes, trade application and option toggles, every step checked
    against the oracle on a host mirror."""
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(20, 400))
    mp_, mg_, mu_ = int(rng.integers(1, 20_000)), int(rng.integers(0, 3_000)), int(rng.integers(1, 6_000))
    R, g, Ai = synth.product_pools(mp_, n, seed=300 + seed)
    Rg, gg, Ag, wg = synth.geomean_pools(max(mg_, 1), n, seed=400 + seed)
    if mg_ == 0:
        Rg, gg, Ag, wg = Rg[:0], gg[:0], Ag[:0], wg[:0]
    mir = Univ3Mirror(*synth.univ3_pools(mu_, n, seed=500 + seed, ragged=bool(seed % 2 == 0)))
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    if mg_:
        p.add_geomean(Rg, gg, Ag, wg)
    p.add_univ3(*mir.args)
    p.finalize()
    R, Rg = R.copy(), Rg.copy()
    A = np.concatenate([Ai, Ag, mir.Ai])
    last_mat = None

    def reference(v):
        D1, L1 = oracle.sweep_product(R, g, Ai, v, threads=8)
        D2, L2 = oracle.sweep_geomean(Rg, gg, Ag, wg, v, threads=8) if mg_ else (D1[:0], L1[:0])
        D3, L3 = mir.sweep(oracle, v)
        return np.concatenate([D1, D2, D3]), np.concatenate([L1, L2, L3])

    ops = ["grad", "mat", "mat", "price", "liq", "push", "apply", "apply", "toggle"]
    for step in range(16):
        op = str(rng.choice(ops))
        v = synth.dual_prices(n, str(rng.choice(["near", "wide", "ones"])), seed=int(rng.integers(1 << 30)))
        if op == "grad":
            psi, acc = p.sweep(v)
            Do, Lo = reference(v)
            check_psi(oracle, A, Do, Lo, v, n, psi, acc, R=np.concatenate([R, Rg, np.zeros((mu_, 2))]) * 64,
                      g=np.concatenate([g, gg, mir.g]))
        elif op == "mat":
            psi, acc = p.sweep(v, materialize=True)
            D, L = p.trades()
            Do, Lo = reference(v)
            assert np.array_equal(D[:mp_], Do[:mp_]) and np.array_equal(L[:mp_], Lo[:mp_])
            assert np.array_equal(D[mp_ + mg_:], Do[mp_ + mg_:]) and np.array_equal(L[mp_ + mg_:], Lo[mp_ + mg_:])
            if mg_:
                tol = 1e-12 * (np.max(Rg, axis=1) / gg)[:, None]
                assert np.all(np.abs(D[mp_:mp_ + mg_] - Do[mp_:mp_ + mg_]) <= tol)
            check_psi(oracle, A, D, L, v, n, psi, acc)
            last_mat = (D, L, v)
        elif op == "price":
            lo = int(rng.integers(0, mu_))
            hi = int(rng.integers(lo, mu_)) + 1
            cp = new_prices(mir, lo, hi, rng)
            p.update_univ3(lo, cp)
            mir.cp[lo:hi] = cp
        elif op == "liq":
            lo = int(rng.integers(0, mu_))
            hi = int(rng.integers(lo, mu_)) + 1
            t0, t1 = mir.off[lo], mir.off[hi]
            lq = mir.lq[t0:t1] * rng.uniform(0.5, 1.5, size=t1 - t0)
            lq[rng.random(t1 - t0) < 0.1] = 0.0
            p.update_univ3(lo, liquidity=lq, count=hi - lo)
            mir.lq[t0:t1] = lq
        elif op == "push":
            lo = int(rng.integers(0, mp_))
            hi = int(rng.integers(lo, mp_)) + 1
            R[lo:hi] *= rng.uniform(0.5, 1.5, size=(hi - lo, 1))
            p.update_reserves(0, lo, R[lo:hi])
            last_mat = None  # (the library would apply the old trades to the pushed reserves)
        elif op == "apply" and last_mat is not None:
            D, L, vm = last_mat
            p.apply_trades()
            R = R + g[:, None] * D[:mp_] - L[:mp_]
            if mg_:
                Rg = Rg + gg[:, None] * D[mp_:mp_ + mg_] - L[mp_:mp_ + mg_]
            mir.move(vm)
            last_mat = None
        elif op == "toggle":
            key = str(rng.choice(["grid_waves", "use_tma"]))
            p.set_option(key, int(rng.integers(0, 2)))
    p.close()
