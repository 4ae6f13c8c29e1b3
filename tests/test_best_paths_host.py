"""cfmm_find_order_paths (include/cfmm_b200.h) on the host (best_path_oracle.py), no GPU.

The mirror states the DP as the header does.  On small random graphs it must agree with a
brute-force enumeration of every walk of at most H hops through B: for ProductTwoCoin, whose quotes
are monotone, the amount is the same number; for all three types the found path is worth what the DP
says, and no walk beats it by more than rounding.  Ties resolve by hops, token and pool position; a
gaining cycle that would reuse a pool gives CFMM_PATH_REPEATS_POOL.  The Python layers reject bad
arguments before they reach the library."""
import types

import numpy as np
import pytest

import best_path_oracle as bo
import hub_oracle as ho
import swap_order_oracle as oo
from test_order_hubs_host import random_market

R0 = np.array([1000.0, 1000.0])


def product_market(rng, n, n_pairs, retire=0.1):
    """ProductTwoCoin pools (a, b, pool, active) on n tokens, 1-2 per pair, prices around ν."""
    nu = np.exp(rng.uniform(-1, 1, size=n + 1))
    pairs = {tuple(sorted(rng.choice(np.arange(1, n + 1), size=2, replace=False).tolist())) for _ in range(n_pairs)}
    pools = []
    for a, b in sorted(pairs):
        for _ in range(int(rng.integers(1, 3))):
            Ai = (a, b) if rng.random() < 0.5 else (b, a)
            R = 10.0 ** rng.uniform(1, 3) / nu[list(Ai)] * np.exp(rng.uniform(-0.2, 0.2, size=2))
            pools.append((Ai[0], Ai[1], oo.ProductPool(R, rng.choice([0.997, 0.999, 1.0])), bool(rng.random() >= retire)))
    return pools


def rows_for(rng, n, q):
    tin = rng.integers(1, n + 1, size=q)
    tout = np.array([rng.choice([x for x in range(1, n + 1) if x != a]) for a in tin])
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    amount = 10.0 ** rng.uniform(-1, 1.5, size=q)
    amount[::7] = 0.0
    return tin.astype(np.int64), tout.astype(np.int64), kind, amount


@pytest.mark.parametrize("seed", range(4))
def test_mirror_equals_brute_force_on_product_pools(seed):
    rng = np.random.default_rng(3000 + seed)
    n = 7
    pools = product_market(rng, n, 12)
    tin, tout, kind, amount = rows_for(rng, n, 14)
    filled = 0
    for H in (1, 2, 3, 4):
        allowed = rng.random(n) < 0.8
        off, hp, ht, x, lam, value, status, dp = bo.find(pools, n, tin, tout, kind, amount, H, allowed)
        for r in range(len(tin)):
            if amount[r] == 0.0:
                assert status[r] == bo.FILLED and off[r + 1] == off[r] and value[r] == 0.0
                continue
            best, _ = bo.brute(pools, n, int(tin[r]), int(tout[r]), int(kind[r]), float(amount[r]), H, allowed)
            if best is None:
                assert status[r] == bo.UNREACHABLE and off[r + 1] == off[r], r
                continue
            assert status[r] in (bo.FILLED, bo.REPEATS_POOL), r
            assert dp[r] == best, (r, H, dp[r], best)
            if status[r] == bo.FILLED:
                filled += 1
                assert value[r] == dp[r] and 1 <= off[r + 1] - off[r] <= H
                assert ht[off[r + 1] - 1] == tout[r]
    assert filled > 10


@pytest.mark.parametrize("seed", range(2))
def test_mirror_against_brute_force_on_all_types(synth, seed):
    """GeometricMeanTwoCoin and UniV3 quotes are not monotone to the last ulp, so a walk the DP drops
    can beat the DP's by rounding; never by more."""
    rng = np.random.default_rng(4000 + seed)
    n = 6
    pools = random_market(rng, synth, n, 10)
    tin, tout, kind, amount = rows_for(rng, n, 12)
    allowed = np.ones(n, dtype=bool)
    for H in (1, 2, 3):
        off, hp, ht, x, lam, value, status, dp = bo.find(pools, n, tin, tout, kind, amount, H, allowed)
        for r in np.flatnonzero((status == bo.FILLED) & (amount > 0)):
            assert value[r] == dp[r]
            best, _ = bo.brute(pools, n, int(tin[r]), int(tout[r]), int(kind[r]), float(amount[r]), H, allowed)
            if kind[r] == bo.EXACT_IN:
                assert dp[r] <= best and dp[r] >= best * (1 - 1e-12), (r, dp[r], best)
            else:
                assert dp[r] >= best and dp[r] <= best * (1 + 1e-12), (r, dp[r], best)


def test_one_hop_is_the_best_direct_pool():
    rng = np.random.default_rng(5)
    pools = product_market(rng, 5, 8, retire=0.0)
    pairs = ho.pair_lists(pools)
    tin, tout, kind, amount = rows_for(rng, 5, 20)
    off, hp, _, _, _, value, status, _ = bo.find(pools, 5, tin, tout, kind, amount, 1, np.ones(5, bool))
    for r in range(len(tin)):
        if amount[r] == 0.0:
            continue
        ks = pairs.get((min(tin[r], tout[r]), max(tin[r], tout[r])), [])
        if kind[r] == 0:
            want = ho.best_f(pools, ks, int(tin[r]), float(amount[r]))
            assert value[r] == want if want > 0 else status[r] == bo.UNREACHABLE
        else:
            want = ho.best_exact_out(pools, ks, int(tin[r]), float(amount[r]))
            assert value[r] == want if want < bo.INF else status[r] == bo.UNREACHABLE


def test_ties_rank_by_hops_token_and_position():
    """Identical pools tie on the amount: the earlier one in the pair's list wins.  Two identical
    intermediate tokens tie on the amount and the hops: the smaller token wins."""
    P = lambda a, b: (a, b, oo.ProductPool(R0.copy(), 0.997), True)
    pools = [P(1, 4), P(4, 2), P(1, 3), P(3, 2), P(3, 2)]  # tokens 3 and 4 are the same route
    for kind, amount in ((0, 5.0), (1, 5.0)):
        off, hp, ht, *_ , status, _ = bo.find(pools, 4, [1], [2], [kind], [amount], 2, np.ones(4, bool))
        assert status[0] == bo.FILLED and hp.tolist() == [2, 3] and ht.tolist() == [3, 2]
    # the second {3, 2} pool first in the pair's list: it is the one taken
    pairs = {(1, 4): [0], (2, 4): [1], (1, 3): [2], (2, 3): [4, 3]}
    off, hp, *_ = bo.find(pools, 4, [1], [2], [0], [5.0], 2, np.ones(4, bool), pairs=pairs)
    assert hp.tolist() == [2, 4]


def test_gaining_cycle_reusing_a_pool():
    """2 → 3 pays two 3 per 2, 3 → 4 and 4 → 2 one for one: the cycle 2 → 3 → 4 → 2 gains.  i = 5 is
    reached only from 3, so with six hops the best walk is 1 → 2 → 3 → 4 → 2 → 3 → 5 and uses the
    {2, 3} pool twice; with three hops it is 1 → 2 → 3 → 5."""
    big = lambda a, b, ra, rb: (a, b, oo.ProductPool(np.array([ra, rb]), 0.997), True)
    pools = [big(1, 2, 1e6, 1e6), big(2, 3, 1e6, 2e6), big(3, 4, 1e6, 1e6), big(4, 2, 1e6, 1e6),
             big(3, 5, 1e6, 1e6)]
    allowed = np.ones(5, bool)
    for kind in (0, 1):
        off, hp, ht, x, lam, value, status, dp = bo.find(pools, 5, [1], [5], [kind], [10.0], 3, allowed)
        assert status[0] == bo.FILLED and hp.tolist() == [0, 1, 4]
        three = dp[0]
        off, hp, *_, status, dp = bo.find(pools, 5, [1], [5], [kind], [10.0], 6, allowed)
        assert status[0] == bo.REPEATS_POOL and off.tolist() == [0, 0]
        assert (dp[0] > three) if kind == 0 else (dp[0] < three)
        best, walk = bo.brute(pools, 5, 1, 5, kind, 10.0, 6, allowed)
        assert best == dp[0] and list(walk) == [0, 1, 2, 3, 1, 4]
    # without token 4 the cycle is gone and the short walk is the best at any length
    allowed[3] = False
    off, hp, *_, status, _ = bo.find(pools, 5, [1], [5], [0], [10.0], 6, allowed)
    assert status[0] == bo.FILLED and hp.tolist() == [0, 1, 4]


def _stub_pools(n_tokens=5):
    def fail(*a):
        raise AssertionError("the library must not be called")
    return types.SimpleNamespace(n_tokens=n_tokens, _ctx=None, _chk=fail,
                                 _lib=types.SimpleNamespace(cfmm_find_order_paths=fail))


def test_python_argument_checks(cr):
    stub = _stub_pools()
    ok = np.ones(5, bool)
    with pytest.raises(ValueError, match="one entry per row"):
        cr.DevicePools.find_order_paths(stub, [1, 2], [2], [0, 0], [1.0, 1.0], 3, ok)
    with pytest.raises(ValueError, match="allowed must have 5 entries"):
        cr.DevicePools.find_order_paths(stub, [1], [2], [0], [1.0], 3, [1, 1, 1])
    router = types.SimpleNamespace(_world=1, _pools=stub, _split_args=None)
    router._split_args = lambda *a: cr.Router._split_args(router, *a)
    for bad in (0, 9):
        with pytest.raises(ValueError, match="max_hops must be 1..8"):
            cr.Router._find(router, [1], [2], [0], [1.0], ok, bad, None, "find_paths")
    with pytest.raises(ValueError, match="allowed .* is required"):
        cr.Router._find(router, [1], [2], [0], [1.0], None, 3, None, "find_paths")
    with pytest.raises(ValueError, match="limits must have 1 entries"):
        cr.Router._find(router, [1], [2], [0], [1.0], ok, 3, [1.0, 2.0], "execute_best_paths")
    router._world = 2
    with pytest.raises(NotImplementedError, match="drives one GPU"):
        cr.Router._find(router, [1], [2], [0], [1.0], ok, 3, None, "find_paths")
