"""The host restatement of cfmm_modify_univ3_liquidity (liquidity_oracle.py) and
Router.modify_liquidity, without a GPU.

The restatement is checked against an independent evaluation of the liquidity step function, and
against the batch form the device uses (all boundaries merged first, then every tick's rows in
order).  The Router drives a stand-in for DevicePools backed by the restatement: the list-to-UniV3
mapping, the argument checks and the refresh of the host pool objects are checked against it."""
import numpy as np
import pytest

import liquidity_oracle as lo_

F = np.float64


def random_ladder(rng, t=None):
    t = int(rng.integers(1, 9)) if t is None else t
    cp = float(np.exp(rng.uniform(-1, 1)))
    lt = cp * 2.0 * np.cumprod(np.concatenate([[1.0], rng.uniform(0.5, 0.9, size=t - 1)]))
    lq = rng.uniform(0, 50, size=t)
    lq[rng.random(t) < 0.2] = 0.0
    return cp, lt, lq


def random_rows(rng, lt, n, burns=True):
    """Mints with bounds on, inside, above and below the ladder; with burns=True some rows burn
    exactly what an earlier mint on the same range added."""
    rows = []
    pts = np.concatenate([lt, lt * 1.5, lt * 0.7, [lt[0] * 3, lt[-1] * 0.2]])
    for _ in range(n):
        if burns and rows and rng.random() < 0.3:
            a, b, d = rows[int(rng.integers(0, len(rows)))]
            if d > 0:
                rows.append((a, b, -d))
                continue
        a, b = np.sort(rng.choice(pts, size=2, replace=False))
        if a == b:
            continue
        rows.append((float(a), float(b), float(rng.uniform(0.1, 40.0))))
    return rows


def batch(lt, lq, rows):
    """The device's form: merge every candidate boundary at once (inheriting the liquidity of the
    tick each falls in, 0 above T₁), then each new tick's rows in batch order."""
    cand = sorted({F(x) for a, b, _ in rows for x in (a, b)}, reverse=True)
    nl, nq, inherit = [], [], F(0.0)
    a = b = 0
    while a < len(lt) or b < len(cand):
        if b == len(cand) or (a < len(lt) and lt[a] >= cand[b]):
            if b < len(cand) and lt[a] == cand[b]:
                b += 1
            nl.append(F(lt[a]))
            inherit = F(lq[a])
            nq.append(inherit)
            a += 1
        else:
            nl.append(cand[b])
            nq.append(inherit)
            b += 1
    nq = np.array(nq)
    bad = None
    for t, T in enumerate(nl):
        for j, (x, y, d) in enumerate(rows):
            if F(x) < T <= F(y):
                nq[t] = nq[t] + F(d)
                if not (nq[t] >= 0 and np.isfinite(nq[t])):
                    bad = j if bad is None else min(bad, j)  # the device's atomicMin
                    break
    return np.array(nl), nq, bad


def test_restatement_is_the_step_function():
    rng = np.random.default_rng(1)
    for _ in range(300):
        _, lt, lq = random_ladder(rng)
        rows = random_rows(rng, lt, int(rng.integers(1, 12)), burns=False)
        nl, nq = lt, lq
        for a, b, d in rows:
            nl, nq, ok = lo_.apply_row(nl, nq, a, b, d)
            assert ok
        assert np.all(np.diff(nl) < 0)
        assert set(lt.tolist()) <= set(nl.tolist())
        assert {x for a, b, _ in rows for x in (a, b)} <= set(nl.tolist())
        lows = np.concatenate([nl[1:], [0.0]])
        for T, low, L in zip(nl, lows, nq):
            mid = 0.5 * (T + low)
            want = lo_.liquidity_at(lt, lq, mid)
            for a, b, d in rows:
                if a < mid < b:
                    want = want + F(d)
            assert L == want, (T, L, want)


def test_batch_form_equals_row_by_row():
    rng = np.random.default_rng(2)
    failed = 0
    for _ in range(400):
        _, lt, lq = random_ladder(rng)
        rows = random_rows(rng, lt, int(rng.integers(1, 15)))
        if rng.random() < 0.2:  # a burn larger than anything minted
            a, b, _ = rows[int(rng.integers(0, len(rows)))]
            rows.insert(int(rng.integers(0, len(rows) + 1)), (a, b, -1e4))
        off = np.array([0, len(lt)])
        got = batch(lt, lq, rows)
        n_off, nl, nq, bad = lo_.replay(off, lt, lq, np.zeros(len(rows), dtype=np.int64),
                                        *map(np.array, zip(*rows)))
        assert got[2] == bad
        if bad is not None:
            failed += 1
            assert nl is lt and nq is lq
            # the rows before the failing one are fine on their own
            assert lo_.replay(off, lt, lq, np.zeros(bad, dtype=np.int64),
                              *(np.array(c)[:bad] for c in zip(*rows)))[3] is None
        else:
            assert np.array_equal(got[0], nl) and np.array_equal(got[1], nq)
            assert n_off[-1] == len(nl)
    assert failed > 20


def test_burn_of_a_mint_never_fails():
    """The header's guarantee: rounding is monotonic, so a tick raised by x from L >= 0 (with only
    mints in between) holds at least x."""
    rng = np.random.default_rng(3)
    for _ in range(2000):
        L = F(rng.uniform(0, 1e3)) * F(10.0) ** rng.integers(-20, 20)
        x = F(rng.uniform(0, 1e3)) * F(10.0) ** rng.integers(-20, 20)
        y = L + x
        for _ in range(int(rng.integers(0, 3))):
            y = y + F(rng.uniform(0, 1e3)) * F(10.0) ** rng.integers(-20, 20)
        assert y - x >= 0.0


def test_insert_boundary_rules():
    lt, lq = np.array([30.0, 20, 10, 5]), np.array([1.0, 2.0, 1.5, 0.0])
    a, b = lo_.insert_boundary(lt, lq, 20.0)
    assert np.array_equal(a, lt) and np.array_equal(b, lq)
    a, b = lo_.insert_boundary(lt, lq, 15.0)   # inside tick 2 (10, 20]: both parts keep 2.0
    assert a.tolist() == [30, 20, 15, 10, 5] and b.tolist() == [1, 2, 2, 1.5, 0]
    a, b = lo_.insert_boundary(lt, lq, 40.0)   # above T₁: a new first tick with 0
    assert a.tolist() == [40, 30, 20, 10, 5] and b.tolist() == [0, 1, 2, 1.5, 0]
    a, b = lo_.insert_boundary(lt, lq, 1.0)    # below T₄: splits the last tick
    assert a.tolist() == [30, 20, 10, 5, 1] and b.tolist() == [1, 2, 1.5, 0, 0]
    a, b, ok = lo_.apply_row(lt, lq, 12.0, 35.0, 3.0)
    assert ok and a.tolist() == [35, 30, 20, 12, 10, 5] and b.tolist() == [3, 4, 5, 2, 1.5, 0]
    _, _, ok = lo_.apply_row(lt, lq, 10.0, 20.0, -2.5)
    assert not ok


class LiquidityPools:
    """DevicePools stand-in: the UniV3 ladders on the host, changed by liquidity_oracle.replay."""

    def __init__(self, n_tokens, device=0):
        self.n_tokens = n_tokens
        self.off, self.lt, self.lq = np.zeros(1, dtype=np.int64), np.zeros(0), np.zeros(0)
        self.calls = []

    def add_product(self, R, gamma, Ai):
        pass

    def add_geomean(self, R, gamma, Ai, w):
        pass

    def add_univ3(self, cp, gamma, Ai, off, lt, lq):
        self.off, self.lt, self.lq = np.array(off), np.array(lt, float), np.array(lq, float)

    def finalize(self):
        pass

    def modify_univ3_liquidity(self, pools, lo, hi, dL):
        self.calls.append(np.array(pools))
        off, lt, lq, bad = lo_.replay(self.off, self.lt, self.lq, pools, lo, hi, dL)
        if bad is not None:
            raise RuntimeError(f"row {bad}")
        self.off, self.lt, self.lq = off, lt, lq

    def univ3_ticks(self, first=0, count=None, ladders=True):
        count = len(self.off) - 1 - first if count is None else count
        s = slice(self.off[first], self.off[first + count])
        return self.off[first:first + count + 1] - self.off[first], self.lt[s].copy(), self.lq[s].copy()

    def close(self):
        pass


def market(cr, seed=5, n=6):
    rng = np.random.default_rng(seed)
    pools = []
    for k in range(18):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 1:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        else:
            cp, lt, lq = random_ladder(rng)
            pools.append(cr.UniV3(cp, lt, lq, 0.997, [a, b]))
    return pools


def test_router_modify_liquidity_map_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=LiquidityPools)
    uni = [i for i, c in enumerate(pools) if isinstance(c, cr.UniV3)]
    before = {i: (pools[i].lower_ticks.copy(), pools[i].liquidity.copy()) for i in uni}
    rng = np.random.default_rng(6)
    ids = rng.choice(uni, size=30)
    rows = []
    for i in ids:
        lt = pools[i].lower_ticks
        a, b = sorted(rng.choice(np.concatenate([lt, lt * 1.3, [lt[-1] * 0.5]]), size=2, replace=False))
        rows.append((a, b, float(rng.uniform(1, 10))))
    lo, hi, dL = map(np.array, zip(*rows))
    r.modify_liquidity(ids, lo, hi, dL)
    assert np.array_equal(r._pools.calls[-1], [uni.index(i) for i in ids])
    for i in uni:  # the host objects equal a row-by-row replay on each pool
        lt, lq = before[i]
        mine = np.flatnonzero(ids == i)
        for j in mine:
            lt, lq, ok = lo_.apply_row(lt, lq, lo[j], hi[j], dL[j])
            assert ok
        c = pools[i]
        assert np.array_equal(c.lower_ticks, lt) and np.array_equal(c.liquidity, lq)
        assert c.current_tick == int(np.sum(c.lower_ticks >= c.current_price))
        assert (len(mine) > 0) == (not np.array_equal(c.liquidity, before[i][1]) or len(lt) != len(before[i][0]))


def test_router_modify_liquidity_argument_checks(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=LiquidityPools)
    with pytest.raises(TypeError):
        r.modify_liquidity([1], [1.0], [2.0], [1.0])        # r.cfmms[1] is a ProductTwoCoin
    with pytest.raises(IndexError):
        r.modify_liquidity([18], [1.0], [2.0], [1.0])
    with pytest.raises(IndexError):
        r.modify_liquidity([-1], [1.0], [2.0], [1.0])
    with pytest.raises(ValueError):
        r.modify_liquidity([0, 2], [1.0], [2.0, 3.0], [1.0, 1.0])
    assert r._pools.calls == []
    r.modify_liquidity([], [], [], [])                       # nothing to do
    r._world = 2  # a multi-GPU Router
    with pytest.raises(NotImplementedError):
        r.modify_liquidity([0], [1.0], [2.0], [1.0])
    with pytest.raises(ValueError):
        cr.DevicePools.modify_univ3_liquidity(None, [0, 1], [1.0, 1.0], [2.0, 2.0], [1.0])
