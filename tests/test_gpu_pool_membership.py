"""Changing the pool set after cfmm_finalize: cfmm_append_* (per-type tail sets), cfmm_set_active
(retire / restore), cfmm_get_pool_state and cfmm_compact (include/cfmm_b200.h).

A pool set is written as a list of add calls (type, arrays) in global insertion order; the first
n_main calls are ingested before finalize and the rest appended after it.  The references are a
context that ingested every call before finalize, a context built without the retired pools,
and the oracle on a host mirror of the pool state."""
import numpy as np
import pytest

from test_gpu_parity import check_psi
from test_gpu_univ3_state import moved_prices

pytestmark = pytest.mark.gpu

ADD = {0: "add_product", 1: "add_geomean", 2: "add_univ3"}
APPEND = {0: "append_product", 1: "append_geomean", 2: "append_univ3"}


def cut(t, a, lo, hi):
    """Pools [lo, hi) of one add call's arrays."""
    if t != 2:
        return tuple(x[lo:hi] for x in a)
    cp, g, Ai, off, lt, lq = a
    return cp[lo:hi], g[lo:hi], Ai[lo:hi], off[lo:hi + 1] - off[lo], lt[off[lo]:off[hi]], lq[off[lo]:off[hi]]


def build(cr, n, calls, n_main=None, opts=None):
    p = cr.DevicePools(n)
    for k, val in (opts or {}).items():
        p.set_option(k, val)
    n_main = len(calls) if n_main is None else n_main
    for i, (t, a) in enumerate(calls):
        if i == n_main:
            p.finalize()
        getattr(p, ADD[t] if i < n_main else APPEND[t])(*a)
    if n_main == len(calls):
        p.finalize()
    return p


def oracle_trades(oracle, calls, v):
    Ds, Ls = [], []
    for t, a in calls:
        D, L = (oracle.sweep_product, oracle.sweep_geomean, oracle.sweep_univ3)[t](*a, v)
        Ds.append(D)
        Ls.append(L)
    return np.concatenate(Ds), np.concatenate(Ls)


def flat(calls):
    """(Ai, R with zero rows for UniV3, γ, type, type-local index) of every pool, global order."""
    Ai, R, g, ty, loc = [], [], [], [], []
    count = {0: 0, 1: 0, 2: 0}
    for t, a in calls:
        m = len(a[1]) if t != 2 else len(a[0])
        Ai.append(a[2])
        g.append(a[1])
        R.append(a[0] if t != 2 else np.zeros((m, 2)))
        ty.append(np.full(m, t))
        loc.append(count[t] + np.arange(m))
        count[t] += m
    return np.concatenate(Ai), np.concatenate(R), np.concatenate(g), np.concatenate(ty), np.concatenate(loc)


def psi_ok(oracle, calls, v, n, psi, acc, retired=None):
    D, L = oracle_trades(oracle, calls, v)
    Ai, R, g, _, _ = flat(calls)
    if retired is not None:
        D[retired] = 0.0
        L[retired] = 0.0
    check_psi(oracle, Ai, D, L, v, n, psi, acc, R=R, g=g, Rq=R)


def retire(p, calls, retired):
    """Retire the pools flagged in `retired` (global order) through cfmm_set_active, type by type."""
    _, _, _, ty, loc = flat(calls)
    for t in (0, 1, 2):
        sel = ty == t
        if sel.any():
            p.set_active(t, 0, ~retired[sel])


def pool_sets(synth, kind, n):
    P = synth.product_pools(30_000, n, seed=11)
    G = synth.geomean_pools(6_000, n, seed=12)
    U = synth.univ3_pools(3_000, n, seed=13, ragged=True)
    if kind in ("product", "product_wide"):
        return [(0, cut(0, P, 0, 24_000)), (0, cut(0, P, 24_000, 25_000)), (0, cut(0, P, 25_000, 30_000))], 1
    if kind == "geomean":
        return [(1, cut(1, G, 0, 4_000)), (1, cut(1, G, 4_000, 4_500)), (1, cut(1, G, 4_500, 6_000))], 1
    if kind == "univ3":
        return [(2, cut(2, U, 0, 2_000)), (2, cut(2, U, 2_000, 2_100)), (2, cut(2, U, 2_100, 3_000))], 1
    return [(0, cut(0, P, 0, 24_000)), (1, cut(1, G, 0, 4_000)), (2, cut(2, U, 0, 2_000)),
            (2, cut(2, U, 2_000, 3_000)), (0, cut(0, P, 24_000, 30_000)), (1, cut(1, G, 4_000, 6_000))], 3


N = 1_500


@pytest.mark.parametrize("kind", ["product", "product_wide", "geomean", "univ3", "mixed"])
def test_append_equals_ingest(cr, oracle, synth, kind):
    calls, n_main = pool_sets(synth, kind, N)
    opts = {"compact_stream": 0} if kind == "product_wide" else {}
    a = build(cr, N, calls, opts=opts)
    b = build(cr, N, calls, n_main, opts=opts)
    assert b.num_pools == a.num_pools
    _, _, _, ty, _ = flat(calls)
    for vk in ("near", "wide"):
        v = synth.dual_prices(N, vk)
        a.sweep(v, materialize=True)
        b.sweep(v, materialize=True)
        (Da, La), (Db, Lb) = a.trades(), b.trades()
        assert np.array_equal(Da, Db) and np.array_equal(La, Lb)
        Do, Lo = oracle_trades(oracle, calls, v)
        exact = ty != 1  # (GeometricMean: pow differs from the oracle's in the last bits)
        assert np.array_equal(Db[exact], Do[exact]) and np.array_equal(Lb[exact], Lo[exact])
        assert np.allclose(Db, Do, rtol=1e-9, atol=1e-9) and np.allclose(Lb, Lo, rtol=1e-9, atol=1e-9)
        for _ in range(2):
            psi, acc = b.sweep(v)
            psi_ok(oracle, calls, v, N, psi, acc)
    a.close()
    b.close()


def test_retire_equals_absent_and_restore(cr, oracle, synth):
    calls, n_main = pool_sets(synth, "mixed", N)
    rng = np.random.default_rng(3)
    _, _, _, ty, _ = flat(calls)
    retired = rng.random(len(ty)) < 0.2
    b = build(cr, N, calls, n_main)
    retire(b, calls, retired)
    kept = []
    start = 0
    for t, a in calls:  # the same calls without the retired pools
        m = len(a[1]) if t != 2 else len(a[0])
        keep = np.flatnonzero(~retired[start:start + m])
        if t != 2:
            kept.append((t, tuple(x[keep] for x in a)))
        else:
            parts = [cut(2, a, i, i + 1) for i in keep]
            cp = np.concatenate([q[0] for q in parts])
            off = np.concatenate([[0], np.cumsum([len(q[4]) for q in parts])]).astype(np.int64)
            kept.append((2, (cp, a[1][keep], a[2][keep], off, np.concatenate([q[4] for q in parts]),
                             np.concatenate([q[5] for q in parts]))))
        start += m
    c = build(cr, N, kept)
    for vk in ("near", "wide"):
        v = synth.dual_prices(N, vk)
        psi, acc = b.sweep(v)
        psi_ok(oracle, calls, v, N, psi, acc, retired=retired)
        psic, accc = c.sweep(v)
        psi_ok(oracle, kept, v, N, psic, accc)
        b.sweep(v, materialize=True)
        c.sweep(v, materialize=True)
        (Db, Lb), (Dc, Lc) = b.trades(), c.trades()
        assert not Db[retired].any() and not Lb[retired].any()
        assert np.array_equal(Db[~retired], Dc) and np.array_equal(Lb[~retired], Lc)
    # restore: the trades of a context that never retired anything
    retire(b, calls, np.zeros(len(ty), dtype=bool))
    for t in (0, 1, 2):
        assert b.pool_state(t)[1].all()
    a = build(cr, N, calls)
    v = synth.dual_prices(N, "wide")
    a.sweep(v, materialize=True)
    b.sweep(v, materialize=True)
    (Da, La), (Db, Lb) = a.trades(), b.trades()
    assert np.array_equal(Da, Db) and np.array_equal(La, Lb)
    for p in (a, b, c):
        p.close()


def test_retire_every_pool_of_a_token(cr, synth):
    n = 400
    R, g, Ai = synth.product_pools(40_000, n, seed=21)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    before = p.pool_set_info(0)
    assert before["tma"] == 1 and before["fixed_point"] == 1 and before["fast_range"] == 1
    b = 17
    held = np.flatnonzero((Ai[:, 0] == b) | (Ai[:, 1] == b))
    active = np.ones(len(g), dtype=bool)
    active[held] = False
    p.set_active(0, 0, active)
    info = p.pool_set_info(0)
    assert info["retired"] == len(held)
    # the token's total reserve is now 0: it must not cost the set its fixed-point slice or range flag
    assert info["fixed_point"] == 1 and info["fast_range"] == 1 and info["compact_stream"] == before["compact_stream"]
    v = synth.dual_prices(n, "wide")
    for _ in range(3):
        psi, acc = p.sweep(v)
        assert psi[b - 1] == 0.0 and np.all(np.isfinite(psi)) and np.isfinite(acc)
    p.close()


def test_state_apply_and_parked_updates(cr, oracle, synth):
    calls, n_main = pool_sets(synth, "mixed", N)
    Ai, _, _, ty, loc = flat(calls)
    retired = np.random.default_rng(5).random(len(ty)) < 0.15
    p = build(cr, N, calls, n_main)
    retire(p, calls, retired)
    # the host mirror, per type in type-local order
    state = {t: [] for t in (0, 1, 2)}
    gam = {t: [] for t in (0, 1, 2)}
    t1 = []
    for t, a in calls:
        state[t].append(a[0].copy())
        gam[t].append(a[1])
        if t == 2:
            t1.append(a[4][a[3][:-1]])
    state = {t: np.concatenate(x) if x else None for t, x in state.items()}
    gam = {t: np.concatenate(x) if x else None for t, x in gam.items()}
    t1 = np.concatenate(t1)
    for t in (0, 1, 2):
        s, act = p.pool_state(t)
        assert np.array_equal(s, state[t]) and np.array_equal(act, ~retired[ty == t])
    v = synth.dual_prices(N, "wide")
    p.sweep(v, materialize=True)
    D, L = p.trades()
    p.apply_trades()
    for t in (0, 1):
        sel = ty == t
        ret = retired[sel]
        new = state[t] + gam[t][:, None] * D[sel] - L[sel]
        state[t] = np.where(ret[:, None], state[t], new)
    sel = ty == 2
    Au = Ai[sel]
    moved = moved_prices(state[2], gam[2], t1, v[Au[:, 0] - 1], v[Au[:, 1] - 1])
    would_move = moved != state[2]
    assert (would_move & retired[sel]).any()  # some retired pools would have moved
    state[2] = np.where(retired[sel], state[2], moved)
    for t in (0, 1, 2):
        assert np.array_equal(p.pool_state(t)[0], state[t])
    assert p.pool_state(0, first=3, count=5)[0].tolist() == state[0][3:8].tolist()
    # pushes to retired pools are kept and become live on restore
    ret0 = np.flatnonzero(retired[ty == 0])[:3]
    ret2 = np.flatnonzero(retired[ty == 2])[:2]
    for k in ret0:
        state[0][k] = state[0][k] * 1.5
        p.update_reserves(0, int(k), state[0][k:k + 1])
    for k in ret2:
        state[2][k] = t1[k] * 0.5
        p.update_univ3(int(k), state[2][k:k + 1])
    assert np.array_equal(p.pool_state(0)[0], state[0]) and np.array_equal(p.pool_state(2)[0], state[2])
    retire(p, calls, np.zeros(len(ty), dtype=bool))
    # a fresh context holding the mirror state (UniV3 liquidities never changed)
    fresh, k = [], {0: 0, 1: 0, 2: 0}
    for t, a in calls:
        m = len(a[1]) if t != 2 else len(a[0])
        fresh.append((t, (state[t][k[t]:k[t] + m],) + tuple(a[1:])))
        k[t] += m
    f = build(cr, N, fresh)
    for vk in ("near", "wide"):
        v = synth.dual_prices(N, vk)
        p.sweep(v, materialize=True)
        f.sweep(v, materialize=True)
        (Dp, Lp), (Df, Lf) = p.trades(), f.trades()
        assert np.array_equal(Dp, Df) and np.array_equal(Lp, Lf)
    p.close()
    f.close()


def test_compact(cr, oracle, synth):
    calls, n_main = pool_sets(synth, "mixed", N)
    _, _, _, ty, _ = flat(calls)
    retired = np.random.default_rng(9).random(len(ty)) < 0.1
    p = build(cr, N, calls, n_main)
    retire(p, calls, retired)
    v = synth.dual_prices(N, "wide")
    p.sweep(v, materialize=True)
    p.apply_trades()
    assert p.pool_set_info(0)["tail"] > 0
    states = {t: p.pool_state(t) for t in (0, 1, 2)}
    v2 = synth.dual_prices(N, "near", seed=3)
    p.sweep(v2, materialize=True)
    D0, L0 = p.trades()
    p.sweep(v2)  # (the first gradient sweep after a reserve change also repacks the TMA streams)
    l0 = p.launch_count
    p.sweep(v2)
    assert p.launch_count - l0 == 6  # three main sets + three tails
    p.compact()
    for t in (0, 1, 2):
        info = p.pool_set_info(t)
        assert info["tail"] == 0 and info["retired"] == int(retired[ty == t].sum())
        s, act = p.pool_state(t)
        assert np.array_equal(s, states[t][0]) and np.array_equal(act, states[t][1])
    assert p.pool_set_info(0)["tma"] == 1
    p.sweep(v2, materialize=True)
    D1, L1 = p.trades()
    assert np.array_equal(D0, D1) and np.array_equal(L0, L1)
    p.sweep(v2)
    l0 = p.launch_count
    psi, acc = p.sweep(v2)
    assert p.launch_count - l0 == 3  # one launch per pool type again
    # Ψ against the oracle on the read-back state
    now = []
    k = {0: 0, 1: 0, 2: 0}
    for t, a in calls:
        m = len(a[1]) if t != 2 else len(a[0])
        now.append((t, (states[t][0][k[t]:k[t] + m],) + tuple(a[1:])))
        k[t] += m
    psi_ok(oracle, now, v2, N, psi, acc, retired=retired)
    p.close()


def test_graph_replay_sees_membership_changes(cr, oracle, synth):
    calls, n_main = pool_sets(synth, "mixed", N)
    _, _, _, ty, _ = flat(calls)
    p = build(cr, N, calls[:n_main])
    v = synth.dual_prices(N, "wide")
    live = list(calls[:n_main])

    def sweeps(retired=None):
        for _ in range(4):  # the second call with the same pinned buffers captures, the rest replay
            psi, acc = p.sweep(v)
        psi_ok(oracle, live, v, N, psi, acc, retired=retired)
        return psi

    base = sweeps()
    for t, a in calls[n_main:]:
        getattr(p, APPEND[t])(*a)
        live.append((t, a))
        psi = sweeps()
        assert not np.array_equal(psi, base)
        base = psi
    retired = np.zeros(len(ty), dtype=bool)
    retired[::7] = True
    retire(p, calls, retired)
    psi_r = sweeps(retired)
    assert not np.array_equal(psi_r, base)
    retire(p, calls, np.zeros(len(ty), dtype=bool))
    sweeps()
    retire(p, calls, retired)
    p.compact()
    sweeps(retired)
    p.close()


def test_device_solver_with_tail_and_retired_pools(cr):
    rng = np.random.default_rng(1234)
    n = 10
    pools = []
    for _ in range(120):
        Ai = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        pools.append(cr.ProductTwoCoin(1000 * rng.random(2), 0.997, Ai))
    c = rng.random(n) + 1e-3
    r = cr.Router(cr.LinearNonnegative(c), pools[:80], n)
    r.add_cfmms(pools[80:])
    off = [3, 17, 85, 101]
    r.set_active(off, False)
    cr.route(r, optimizer="device")
    assert not r.Δs[off].any() and not r.Λs[off].any()
    kept = [q for i, q in enumerate(pools) if i not in off]
    f = cr.Router(cr.LinearNonnegative(c), kept, n)
    cr.route(f, optimizer="device")
    gr = r.objective.f(r.v) + r._pools.sweep(r.v)[1]
    gf = f.objective.f(f.v) + f._pools.sweep(f.v)[1]
    assert abs(gr - gf) <= 1e-6 * max(1.0, abs(gf)), (gr, gf)
    pr, pf = float(c @ cr.netflows(r)), float(c @ cr.netflows(f))
    assert abs(pr - pf) <= 1e-4 * max(1.0, abs(pf)), (pr, pf)


def test_errors_change_nothing(cr, synth):
    n = 50
    R, g, Ai = synth.product_pools(500, n, seed=2)
    p = cr.DevicePools(n)
    with pytest.raises(cr.CFMMError) as e:
        p.append_product(R[:3], g[:3], Ai[:3])  # before finalize
    assert e.value.code == -3
    p.add_product(R, g, Ai)
    p.finalize()
    with pytest.raises(cr.CFMMError) as e:
        p.add_product(R[:3], g[:3], Ai[:3])  # cfmm_add_* after finalize keeps its meaning
    assert e.value.code == -3
    v = synth.dual_prices(n, "wide")
    p.sweep(v, materialize=True)
    D0, _ = p.trades()
    bad = Ai[:3].copy()
    bad[1, 1] = n + 1
    with pytest.raises(cr.CFMMError) as e:
        p.append_product(R[:3], g[:3], bad)
    assert e.value.code == -1
    with pytest.raises(cr.CFMMError) as e:
        p.set_active(0, 499, [True, False])
    assert e.value.code == -1
    with pytest.raises(cr.CFMMError) as e:
        p.pool_state(0, first=-1, count=2)
    assert e.value.code == -1
    with pytest.raises(cr.CFMMError) as e:
        p.set_active(7, 0, [False])
    assert e.value.code == -1
    assert p.num_pools == 500 and p.pool_set_info(0)["tail"] == 0
    assert np.array_equal(p.trades()[0], D0)  # nothing changed: the trades are still readable
    p.set_active(0, 0, [True, True])  # restoring active pools changes nothing either
    assert np.array_equal(p.trades()[0], D0)
    for change in (lambda: p.append_product(R[:2], g[:2], Ai[:2]), lambda: p.set_active(0, 5, [False]),
                   lambda: p.compact()):
        p.sweep(v, materialize=True)
        change()
        for fn in (p.trades, p.apply_trades):
            with pytest.raises(cr.CFMMError) as e:
                fn()
            assert e.value.code == -3
    p.close()
