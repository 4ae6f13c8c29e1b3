"""update_reserves(r) on pool sets that hold UniV3 pools, without a GPU: the Router drives an
oracle-backed stand-in for DevicePools that also implements apply_trades / update_univ3.  The
host UniV3 objects must follow the post-trade price rule of cfmm_apply_trades
(include/cfmm_b200.h) bit for bit, and the next route must start from the moved prices."""
import warnings

import numpy as np
import pytest

from test_host_logic import OraclePools


def moved_price(q, g, t1, va, vb):
    """The rule of include/cfmm_b200.h, written out independently of router.py."""
    with np.errstate(all="ignore"):
        q, g, t1 = np.float64(q), np.float64(g), np.float64(t1)
        p = np.float64(va) / np.float64(vb)
        if g * q <= p <= q / g:
            return float(q)
        target = p / g if p < g * q else g * p
        if np.isnan(target) or target <= 0.0:
            return float(q)
        return float(min(target, t1))


class OraclePoolsWithState(OraclePools):
    """Adds the device-side state updates: R + γΔ − Λ for the two-coin parts, the moved price
    for the UniV3 parts (at the ν of the last materialising sweep)."""

    def sweep(self, v, materialize=False):
        out = super().sweep(v, materialize)
        if materialize:
            self._v_mat = np.array(v, dtype=np.float64)
        return out

    def apply_trades(self):
        D, L = self._trades
        k = 0
        for part in self.parts:
            m = len(part[2])
            if part[0] in ("p", "g"):
                part[1][:] = part[1] + part[2][:, None] * D[k:k + m] - L[k:k + m]
            else:
                cp, g, Ai, off, lt = part[1], part[2], part[3], part[4], part[5]
                for i in range(m):
                    cp[i] = moved_price(cp[i], g[i], lt[off[i]], self._v_mat[Ai[i, 0] - 1], self._v_mat[Ai[i, 1] - 1])
            k += m

    def update_univ3(self, first, current_price=None, liquidity=None, count=None):
        part = [p for p in self.parts if p[0] == "u"][0]
        if current_price is not None:
            part[1][first:first + len(current_price)] = current_price
        if liquidity is not None:
            off = part[4]
            part[6][off[first]:off[first] + len(liquidity)] = liquidity


def mixed_pools(cr, n=8, seed=5):
    rng = np.random.default_rng(seed)
    pools = []
    for k in range(24):
        Ai = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 0:
            cp = float(np.exp(rng.uniform(-1, 1)))
            t = int(rng.integers(1, 7))
            lt = cp * 1.5 * np.cumprod(np.concatenate([[1.0], rng.uniform(0.5, 0.9, size=t - 1)]))
            lq = 100 * rng.uniform(0, 2, size=t)
            lq[rng.random(t) < 0.2] = 0.0
            pools.append(cr.UniV3(cp, lt, lq, 0.997, Ai))
        elif k % 3 == 1:
            pools.append(cr.ProductTwoCoin(1000 * rng.random(2) + 1, 0.997, Ai))
        else:
            w1 = rng.uniform(0.2, 0.8)
            pools.append(cr.GeometricMeanTwoCoin(1000 * rng.random(2) + 1, [w1, 1 - w1], 0.997, Ai))
    return pools


def test_update_reserves_moves_univ3_objects(cr):
    pools = mixed_pools(cr)
    n = 8
    r = cr.Router(cr.LinearNonnegative(np.linspace(0.5, 1.5, n)), pools, n, _pools_factory=OraclePoolsWithState)
    cr.route(r)
    uni = [c for c in pools if isinstance(c, cr.UniV3)]
    before = [(c.current_price, c.lower_ticks[0]) for c in uni]
    expect = [moved_price(q, c.gamma, t1, r.v[c.Ai[0] - 1], r.v[c.Ai[1] - 1]) for (q, t1), c in zip(before, uni)]
    traded = [bool(np.any(D != 0)) for D, c in zip(r.Δs, pools) if isinstance(c, cr.UniV3)]
    assert any(traded)
    with warnings.catch_warnings():
        warnings.simplefilter("error")  # no warning: UniV3 pools are updated like the others
        cr.update_reserves(r)
    for c, q in zip(uni, expect):
        assert c.current_price == q                                    # bit for bit
        assert c.current_tick == int(np.sum(c.lower_ticks >= q)) >= 1
    moved = [c.current_price != q for c, (q, _) in zip(uni, before)]
    assert all(mv for mv, tr in zip(moved, traded) if tr)  # every pool whose walk traded has moved
    # the next route starts from the moved state: the stand-in's device state equals a context
    # built afresh from the host objects
    v = r.v * np.linspace(0.9, 1.1, n)
    cr.find_arb(r, v)
    fresh = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=OraclePoolsWithState)
    cr.find_arb(fresh, v)
    assert np.array_equal(r.Δs, fresh.Δs) and np.array_equal(r.Λs, fresh.Λs)


def test_update_reserves_uses_the_materialising_nu(cr):
    """find_arb!(r, v) materialises at v without touching r.v: the UniV3 prices move by v."""
    c = cr.UniV3(1.0, [2.0, 1.5, 0.8, 0.4], [10.0, 20.0, 15.0, 0.0], 0.997, [1, 2])
    r = cr.Router(cr.LinearNonnegative(np.ones(2)), [c], 2, _pools_factory=OraclePoolsWithState)
    v = np.array([0.5, 1.0])  # p = 0.5 < γq: upper walk to p/γ
    cr.find_arb(r, v)
    cr.update_reserves(r)
    assert c.current_price == float(np.float64(0.5) / np.float64(0.997)) and c.current_tick == 3
    # ν far above the top tick: the lower walk drains tick 1 and the price stops at T₁
    cr.find_arb(r, np.array([100.0, 1.0]))
    cr.update_reserves(r)
    assert c.current_price == 2.0 and c.current_tick == 1


@pytest.mark.parametrize("va,vb", [(1.0, 1.0), (0.2, 1.0), (3.0, 1.0), (1e6, 1.0), (np.nan, 1.0), (0.0, 1.0),
                                   (1.0, 0.0), (1.0, np.inf), (-1.0, 1.0)])
def test_moved_price_table(cr, va, vb):
    """Every row of the table, through router.univ3_moved_price, against the independent form."""
    from cfmmrouter_b200 import router
    c = cr.UniV3(1.0, [2.0, 1.5, 0.8, 0.4], [10.0, 20.0, 15.0, 0.0], 0.997, [1, 2])
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        q = router.univ3_moved_price(c, np.array([va, vb]))
    assert q == moved_price(1.0, 0.997, 2.0, va, vb)
    assert 0.0 < q <= 2.0


def test_sync_reserves_pushes_univ3_state(cr):
    pools = mixed_pools(cr, seed=9)
    n = 8
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=OraclePoolsWithState)
    for c in pools:
        if isinstance(c, cr.UniV3):
            c.current_price = float(c.lower_ticks[-1])  # a tie with the last tick
            c.liquidity = c.liquidity[::-1].copy()
    r.sync_reserves()
    v = np.linspace(0.7, 1.3, n)
    cr.find_arb(r, v)
    fresh = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n, _pools_factory=OraclePoolsWithState)
    cr.find_arb(fresh, v)
    assert np.array_equal(r.Δs, fresh.Δs) and np.array_equal(r.Λs, fresh.Λs)
