"""Router.add_cfmms and Router.set_active without a GPU: the Router drives an oracle-backed
stand-in for DevicePools that also appends pools and retires them.  The list-to-library order map
must follow the appends, retired pools must trade nothing, and update_reserves(r) must leave
retired pools (including UniV3 pools the price rule would move) as they are."""
import numpy as np
import pytest

from test_univ3_host_update import OraclePoolsWithState, moved_price


class OraclePoolsWithMembership(OraclePoolsWithState):
    """Appends are adds (the parts are swept in call order, the library's global order); a retired
    pool trades zero and does not move in apply_trades."""

    def __init__(self, n_tokens, device=0):
        super().__init__(n_tokens, device)
        self.retired = {0: np.zeros(0, bool), 1: np.zeros(0, bool), 2: np.zeros(0, bool)}

    def _grow(self, t, m):
        self.retired[t] = np.concatenate([self.retired[t], np.zeros(m, bool)])

    def add_product(self, R, gamma, Ai):
        super().add_product(R, gamma, Ai)
        self._grow(0, len(gamma))

    def add_geomean(self, R, gamma, Ai, w):
        super().add_geomean(R, gamma, Ai, w)
        self._grow(1, len(gamma))

    def add_univ3(self, cp, gamma, Ai, off, lt, lq):
        super().add_univ3(cp, gamma, Ai, off, lt, lq)
        self._grow(2, len(cp))

    append_product, append_geomean, append_univ3 = add_product, add_geomean, add_univ3

    def set_active(self, t, first, active):
        self.retired[t][first:first + len(active)] = ~np.asarray(active, bool)

    def _mask(self):
        """Retired flags in global (call) order."""
        seen = {0: 0, 1: 0, 2: 0}
        out = []
        for part in self.parts:
            t = "pgu".index(part[0])
            m = len(part[2])
            out.append(self.retired[t][seen[t]:seen[t] + m])
            seen[t] += m
        return np.concatenate(out) if out else np.zeros(0, bool)

    def sweep(self, v, materialize=False):
        super().sweep(v, materialize)
        D, L = self._trades
        off = self._mask()
        D[off] = 0.0
        L[off] = 0.0
        A = np.concatenate([part[3] for part in self.parts])
        acc, G = self.o.fold(A, D, L, v, self.n_tokens)
        return G, acc

    def apply_trades(self):
        keep = [part[1].copy() for part in self.parts if part[0] == "u"]
        super().apply_trades()
        k = 0
        for part in self.parts:
            if part[0] == "u":
                m = len(part[1])
                ret = self.retired[2][k:k + m]
                part[1][ret] = keep.pop(0)[ret]
                k += m


def market(cr, seed=3, n=6):
    rng = np.random.default_rng(seed)
    pools = []
    for k in range(12):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 0:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        elif k % 3 == 1:
            pools.append(cr.GeometricMeanTwoCoin(100 + 900 * rng.random(2), [0.3, 0.7], 0.997, [a, b]))
        else:
            cp = 0.5 + rng.random()
            pools.append(cr.UniV3(cp, cp * np.array([2.0, 1.5, 0.8, 0.4]), [50.0, 80.0, 60.0, 0.0], 0.997, [a, b]))
    return pools


def test_add_cfmms_matches_a_router_built_with_every_pool(cr):
    pools = market(cr)
    n = 6
    obj = cr.LinearNonnegative(np.ones(n))
    r = cr.Router(obj, pools[:5], n, _pools_factory=OraclePoolsWithMembership)
    r.add_cfmms(pools[5:9])
    r.add_cfmms([])
    r.add_cfmms(pools[9:])
    assert len(r.cfmms) == 12 and r.Δs.shape == (12, 2) and r.Λs.shape == (12, 2)
    assert sorted(r._order.tolist()) == list(range(12))
    f = cr.Router(obj, pools, n, _pools_factory=OraclePoolsWithMembership)
    v = np.exp(np.random.default_rng(1).uniform(-1, 1, size=n))
    cr.find_arb(r, v)
    cr.find_arb(f, v)
    assert np.array_equal(r.Δs, f.Δs) and np.array_equal(r.Λs, f.Λs)
    assert np.any(r.Δs[5:] != 0.0)


def test_set_active_zeroes_trades_and_update_reserves_skips_retired(cr):
    pools = market(cr, seed=4)
    n = 6
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools[:8], n, _pools_factory=OraclePoolsWithMembership)
    r.add_cfmms(pools[8:])
    off = [0, 2, 4, 10]  # product, UniV3, geomean, appended geomean
    r.set_active(off, False)
    assert r._retired.tolist() == [i in off for i in range(12)]
    v = np.array([0.3, 3.0, 0.5, 2.0, 0.2, 4.0])  # far from every pool's band: every active pool trades
    cr.find_arb(r, v)
    assert not r.Δs[off].any() and not r.Λs[off].any()
    before = [(c.R.copy() if hasattr(c, "R") else None, getattr(c, "current_price", None)) for c in r.cfmms]
    u = r.cfmms[2]
    assert moved_price(u.current_price, u.gamma, u.lower_ticks[0], v[u.Ai[0] - 1], v[u.Ai[1] - 1]) != u.current_price
    cr.update_reserves(r)
    for i in off:
        c = r.cfmms[i]
        if isinstance(c, cr.UniV3):
            assert c.current_price == before[i][1]
        else:
            assert np.array_equal(c.R, before[i][0])
    moved = [i for i in range(12) if i not in off and isinstance(r.cfmms[i], cr.UniV3)]
    assert any(r.cfmms[i].current_price != before[i][1] for i in moved)
    # restore: the pool trades again
    r.set_active([2], True)
    assert not r._retired[2]
    cr.find_arb(r, v)
    assert r.Δs[2].any() or r.Λs[2].any()
    with pytest.raises(IndexError):
        r.set_active([12], False)


def test_membership_changes_are_single_gpu(cr):
    r = cr.Router(cr.LinearNonnegative(np.ones(2)), [cr.ProductTwoCoin([1, 2], 1, [1, 2])], 2,
                  _pools_factory=OraclePoolsWithMembership)
    r._world = 2  # as a Router with a process group of two ranks
    with pytest.raises(NotImplementedError):
        r.add_cfmms([cr.ProductTwoCoin([1, 2], 1, [1, 2])])
    with pytest.raises(NotImplementedError):
        r.set_active([0], False)
