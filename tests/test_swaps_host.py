"""Router.quote_swaps / Router.execute_swaps and the host swap oracle, without a GPU.

The Router drives a stand-in for DevicePools whose swaps are the host restatements in
swap_oracle.py: the list-to-type mapping, the order of the results and the refresh of the host
pool objects are checked against it.  The restatements themselves are checked against 50-digit
mpmath, and the UniV3 price rule against the tick the walk ends in."""
import mpmath as mp
import numpy as np
import pytest

import swap_oracle as so

EPS = np.finfo(np.float64).eps


class SwapPools:
    """DevicePools stand-in: per-type host state, swaps by swap_oracle (GeometricMean in the
    expm1/log1p form of the device)."""

    def __init__(self, n_tokens, device=0):
        self.n_tokens = n_tokens
        self.R = {0: np.zeros((0, 2)), 1: np.zeros((0, 2))}
        self.g = {0: np.zeros(0), 1: np.zeros(0), 2: np.zeros(0)}
        self.w = np.zeros((0, 2))
        self.cp, self.ticks = np.zeros(0), []

    def add_product(self, R, gamma, Ai):
        self.R[0], self.g[0] = np.array(R, float).reshape(-1, 2), np.array(gamma, float)

    def add_geomean(self, R, gamma, Ai, w):
        self.R[1], self.g[1], self.w = np.array(R, float).reshape(-1, 2), np.array(gamma, float), np.array(w, float)

    def add_univ3(self, cp, gamma, Ai, off, lt, lq):
        self.cp, self.g[2] = np.array(cp, float), np.array(gamma, float)
        self.ticks = [(lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]]) for i in range(len(cp))]

    def finalize(self):
        pass

    def _one(self, t, i, x):
        if t == 0:
            return np.array(so.product_forward(self.R[0][i], self.g[0][i], x)), None
        if t == 1:
            R, w, d = self.R[1][i], self.w[i], self.g[1][i] * x
            out = np.zeros(2)
            for a in (0, 1):
                if x[a] > 0:
                    o = 1 - a
                    out[o] = min(max(R[o] * -np.expm1(-(w[a] / w[o]) * np.log1p(d[a] / R[a])), 0.0), R[o])
            return out, None
        lam, q = so.univ3_swap(self.cp[i], *self.ticks[i], self.g[2][i], x)
        return (np.array([0.0, lam]) if x[0] > 0 else np.array([lam, 0.0]) if x[1] > 0 else np.zeros(2)), q

    def quote_swaps(self, t, pools, T):
        return np.array([self._one(t, i, x)[0] for i, x in zip(pools, T)]).reshape(-1, 2)

    def execute_swaps(self, t, pools, T):
        out = []
        for i, x in zip(pools, T):
            lam, q = self._one(t, i, x)
            if t == 2:
                self.cp[i] = q
            elif x.max() > 0:
                self.R[t][i] = (self.R[t][i] + self.g[t][i] * x) - lam
            out.append(lam)
        return np.array(out).reshape(-1, 2)

    def pool_state(self, t, first=0, count=None):
        s = self.cp if t == 2 else self.R[t]
        count = len(s) - first if count is None else count
        return s[first:first + count].copy(), np.ones(count, bool)

    def close(self):
        pass


def market(cr, seed=4, n=6):
    rng = np.random.default_rng(seed)
    pools = []
    for k in range(15):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 1:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        elif k % 3 == 2:
            pools.append(cr.GeometricMeanTwoCoin(100 + 900 * rng.random(2), [0.3, 0.7], 0.997, [a, b]))
        else:
            cp = float(np.exp(rng.uniform(-1, 1)))
            lt = cp * 1.5 * np.cumprod([1.0, 0.8, 0.7, 0.6])
            pools.append(cr.UniV3(cp, lt, [50.0, 0.0, 80.0, 20.0], 0.997, [a, b]))
    return pools


def test_router_swaps_map_and_refresh(cr):
    n = 6
    pools = market(cr, n=n)
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=SwapPools)
    ref = SwapPools(n)  # the same pools, addressed by type directly
    r2 = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=lambda *a: ref)
    rng = np.random.default_rng(1)
    ids = rng.integers(0, len(pools), size=40)
    T = np.zeros((40, 2))
    T[np.arange(40), rng.integers(0, 2, size=40)] = rng.uniform(0.1, 30, size=40)
    T[::9] = 0.0
    q = r.quote_swaps(ids, T)
    for j, i in enumerate(ids):  # caller's order, each row on the current state
        t = [0, 1, 2][[cr.ProductTwoCoin, cr.GeometricMeanTwoCoin, cr.UniV3].index(type(pools[i]))]
        k = r2._type_lists[t].index(i)
        assert np.array_equal(q[j], ref.quote_swaps(t, [k], T[j:j + 1])[0])
    before = [c.R.copy() if hasattr(c, "R") else c.current_price for c in pools]
    got = r.execute_swaps(ids, T)
    assert np.array_equal(got[0], q[0])
    for j, i in enumerate(ids):  # replayed one row at a time, in order
        t = [0, 1, 2][[cr.ProductTwoCoin, cr.GeometricMeanTwoCoin, cr.UniV3].index(type(pools[i]))]
        assert np.array_equal(got[j], ref.execute_swaps(t, [r2._type_lists[t].index(i)], T[j:j + 1])[0])
    touched = set(ids[T[:, 0] + T[:, 1] > 0].tolist())
    for i, c in enumerate(pools):
        if isinstance(c, cr.UniV3):
            k = r2._type_lists[2].index(i)
            assert c.current_price == ref.cp[k]
            assert c.current_tick == int(np.sum(c.lower_ticks >= c.current_price))
            assert (c.current_price != before[i]) == (i in touched)
        else:
            t = 0 if isinstance(c, cr.ProductTwoCoin) else 1
            assert np.array_equal(c.R, ref.R[t][r2._type_lists[t].index(i)])
            assert (not np.array_equal(c.R, before[i])) == (i in touched)


def test_router_swap_argument_checks(cr):
    n = 6
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), market(cr, n=n), n, _pools_factory=SwapPools)
    with pytest.raises(ValueError):
        r.quote_swaps([0, 1], [[1.0, 0.0]])
    with pytest.raises(ValueError):
        r.execute_swaps([0], [1.0, 0.0])
    with pytest.raises(IndexError):
        r.quote_swaps([15], [[1.0, 0.0]])
    with pytest.raises(IndexError):
        r.execute_swaps([-1], [[1.0, 0.0]])
    assert r.quote_swaps([], np.zeros((0, 2))).shape == (0, 2)
    r._world = 2  # a multi-GPU Router
    with pytest.raises(NotImplementedError):
        r.execute_swaps([0], [[1.0, 0.0]])
    with pytest.raises(ValueError):
        cr.DevicePools._swap_args([0, 1], np.zeros((3, 2)))


def _mp_univ3(price, lt, lq, gamma, tender):
    """forward_trade at 50 digits: the same walk, exact-ish arithmetic."""
    with mp.workdps(50):
        n = len(lt)
        lt = [mp.mpf(float(x)) for x in lt]
        lq = [mp.mpf(float(x)) for x in lq]
        price = mp.mpf(float(price))
        tok1 = tender[0] > 0
        d = mp.mpf(float(np.float64(gamma) * np.float64(tender[0] if tok1 else tender[1])))
        cur = sum(1 for x in lt if x >= price)
        lam = mp.mpf(0)
        for idx in (range(cur, n + 1) if tok1 else range(cur, 0, -1)):
            k, pplus = lq[idx - 1], lt[idx - 1]
            pminus = lt[idx] if idx < n else mp.mpf(0)
            a, b = mp.sqrt(k / pplus), mp.sqrt(k * pminus)
            p = pplus if idx > cur else (pminus if idx < cur else price)
            R1, R2 = mp.sqrt(k / p) - a, mp.sqrt(k * p) - b
            if not tok1:
                a, b, R1, R2 = b, a, R2, R1
            mx = k / b - (R1 + a) if b > 0 else (mp.inf if a > 0 else mp.mpf(0))
            if mx > d:
                return lam + min(R2, (R2 + b) - k / (R1 + a + d))
            lam += R2
            d -= mx
        return lam


def test_oracle_against_mpmath():
    rng = np.random.default_rng(3)
    for _ in range(300):
        R = np.exp(rng.uniform(-5, 8, size=2))
        g = rng.choice([1.0, 0.997])
        x = R[0] * 10.0 ** rng.uniform(-10, 5)
        lam = so.product_forward(R, g, [x, 0.0])[1]
        with mp.workdps(50):
            d = mp.mpf(float(np.float64(g) * np.float64(x)))
            truth = mp.mpf(R[1]) - mp.mpf(R[0]) * mp.mpf(R[1]) / (mp.mpf(R[0]) + d)
        assert abs(mp.mpf(lam) - truth) <= 4 * EPS * R[1]
    lt, lq = [30.0, 20, 10, 5], [1.0, 2.0, 1.5, 0.0]
    for x in np.geomspace(1e-6, 1e6, 60):
        for T in ([x, 0.0], [0.0, x]):
            lam = so.univ3_swap(15.0, lt, lq, 0.997, T)[0]
            truth = _mp_univ3(15.0, lt, lq, 0.997, T)
            assert abs(mp.mpf(lam) - truth) <= 64 * EPS * (abs(truth) + 1), (T, lam, truth)
    # the GeometricMean truth: a tender that doubles R₁ leaves R₂/2 at w = (1/2, 1/2), and doubling R₂
    # leaves R₁/√2 at w = (1/2, 1/4)
    a, b = so.geomean_truth([2.0, 3.0], [0.5, 0.5], 1.0, [2.0, 0.0])
    assert a == 0.0 and abs(b - 1.5) < mp.mpf(10) ** -45
    with mp.workdps(50):
        a, b = so.geomean_truth([3.0, 2.0], [0.5, 0.25], 1.0, [0.0, 2.0])
        assert b == 0.0 and abs(a - (3 - 3 / mp.sqrt(2))) < mp.mpf(10) ** -45


def test_univ3_price_stays_in_ending_tick():
    rng = np.random.default_rng(9)
    ended = exhausted = 0
    for _ in range(400):
        t = int(rng.integers(1, 9))
        cp = float(np.exp(rng.uniform(-1, 1)))
        lt = cp * 1.7 * np.cumprod(np.concatenate([[1.0], rng.uniform(0.5, 0.9, size=t - 1)]))
        lq = rng.uniform(0, 50, size=t)
        lq[rng.random(t) < 0.25] = 0.0
        T = [0.0, 0.0]
        T[int(rng.integers(0, 2))] = float(10.0 ** rng.uniform(-4, 3))
        lam, q, idx = so.univ3_swap(cp, lt, lq, 0.997, T, end_tick=True)
        if idx:
            ended += 1
            lo = lt[idx] if idx < t else 0.0
            assert lo <= q <= lt[idx - 1] and lq[idx - 1] > 0
            cur = so.current_tick(lt, q)
            assert cur in (idx, idx + 1) or (q == lt[idx - 1] and cur >= idx)
        elif q != cp:
            exhausted += 1
            assert q in lt or q == 0.0
        if T[0] > 0:
            assert q <= cp * (1 + 4 * EPS)
        else:
            assert q >= cp * (1 - 4 * EPS)
        assert 0.0 <= q <= lt[0]
    assert ended > 100 and exhausted > 10
