"""cfmm_quote_token_values (include/cfmm_b200.h) on the host (token_value_oracle.py), no GPU.

The mirror states the DP as the header does, over every reached token at every level.  On small
ProductTwoCoin markets, whose quotes are monotone, it must give every token the best amount over a
brute-force enumeration of every walk of at most H hops.  The vectorised numpy restatement, which
relaxes only the tokens that changed at the level before (as the device does), must give the same
values and levels bit for bit."""
import numpy as np
import pytest

import swap_order_oracle as oo
import token_value_oracle as tv
from test_best_paths_host import product_market


def arrays(pools):
    R = np.array([p[2].R for p in pools], dtype=np.float64).reshape(-1, 2)
    g = np.array([p[2].g for p in pools], dtype=np.float64)
    Ai = np.array([(p[0], p[1]) for p in pools], dtype=np.int64).reshape(-1, 2)
    act = np.array([p[3] for p in pools], dtype=bool)
    return R, g, Ai, act


@pytest.mark.parametrize("seed", range(4))
def test_dp_equals_brute_force_on_product_pools(seed):
    rng = np.random.default_rng(7000 + seed)
    n = 7
    pools = product_market(rng, n, 13)
    lists, quote = tv.pool_lists(pools), tv.pool_quote(pools)
    reached = 0
    for H in (1, 2, 3, 4):
        for mask in (None, rng.random(n) < 0.75):
            for kind in (tv.EXACT_IN, tv.EXACT_OUT):
                root = int(rng.integers(1, n + 1))
                amount = 10.0 ** rng.uniform(-1, 1.5)
                res = tv.dp(root, kind, amount, lists, n, mask, H, quote)
                best = tv.brute(pools, n, root, kind, amount, H, mask)
                assert np.array_equal(res.value, best), (H, kind, res.value, best)
                assert res.value[root - 1] == amount and res.hops[root - 1] == 0
                assert res.status[root - 1] == tv.FILLED
                for t in range(1, n + 1):
                    if t == root:
                        continue
                    if res.lvl[t - 1] < 0:
                        assert res.status[t - 1] == tv.UNREACHABLE and res.hops[t - 1] == 0
                        assert res.value[t - 1] == (np.inf if kind else 0.0)
                        continue
                    reached += 1
                    assert mask is None or mask[t - 1]
                    walk = res.walk(t)
                    assert len(walk) == res.hops[t - 1] == res.lvl[t - 1] <= H
                    # the walk priced hop by hop is the value
                    v = amount
                    for a, b, k in (reversed(walk) if kind else walk):
                        pool = pools[k]
                        v = float(oo.exact_out(pool[2], v, a == pool[0])[0]) if kind else float(pool[2].f(v, a == pool[0]))
                    assert v == res.value[t - 1]
                    assert (walk[0][0], walk[-1][1]) == ((t, root) if kind else (root, t))
    assert reached > 40


@pytest.mark.parametrize("seed", range(3))
def test_vectorised_product_dp_equals_the_scalar_dp(seed):
    """The scalar DP relaxes every reached token; the numpy one only the previous level's changed
    tokens.  Same values, same levels, bit for bit."""
    rng = np.random.default_rng(7100 + seed)
    n = 12
    pools = product_market(rng, n, 30)
    R, g, Ai, act = arrays(pools)
    lists, quote = tv.pool_lists(pools), tv.pool_quote(pools)
    for H in (1, 3, 5, 8):
        for mask in (None, rng.random(n) < 0.7):
            root = int(rng.integers(1, n + 1))
            amount = 10.0 ** rng.uniform(-1, 1.5)
            res = tv.dp(root, tv.EXACT_IN, amount, lists, n, mask, H, quote)
            val, lvl, front = tv.product(R, g, Ai, act, n, root, amount, H, mask)
            assert np.array_equal(val, res.value) and np.array_equal(lvl, res.lvl)
            assert np.array_equal(front, [len(p) for p in res.pred])


def test_ties_rank_by_neighbour_then_pool():
    """Two identical pools of one pair: the earlier one wins; two neighbours giving the same amount:
    the smaller token wins."""
    R = np.array([100.0, 100.0])
    pools = [(1, 2, oo.ProductPool(R, 0.997), True), (2, 1, oo.ProductPool(R, 0.997), True),
             (1, 3, oo.ProductPool(R, 0.997), True), (1, 4, oo.ProductPool(R, 0.997), True),
             (3, 5, oo.ProductPool(R, 0.997), True), (4, 5, oo.ProductPool(R, 0.997), True)]
    res = tv.dp(1, tv.EXACT_IN, 1.0, tv.pool_lists(pools), 5, None, 2, tv.pool_quote(pools))
    assert res.walk(2) == [(1, 2, 0)]
    assert res.walk(5) == [(1, 3, 2), (3, 5, 4)]
    res = tv.dp(1, tv.EXACT_OUT, 1.0, tv.pool_lists(pools), 5, None, 2, tv.pool_quote(pools))
    assert res.walk(2) == [(2, 1, 0)]
    assert res.walk(5) == [(5, 3, 4), (3, 1, 2)]


def test_gaining_cycle_through_one_pool_twice_is_reported():
    """A mispriced pair gains on a round trip through two pools; a walk that needs the cheap pool
    twice is CFMM_PATH_REPEATS_POOL and keeps the DP's amount."""
    pools = [(1, 2, oo.ProductPool(np.array([100.0, 100.0]), 1.0), True),
             (1, 2, oo.ProductPool(np.array([100.0, 130.0]), 1.0), True)]
    res = tv.dp(1, tv.EXACT_IN, 1.0, tv.pool_lists(pools), 2, None, 8, tv.pool_quote(pools))
    assert res.hops[1] == 1 and res.status[1] == tv.FILLED  # the root is never a destination
    pools += [(2, 3, oo.ProductPool(np.array([100.0, 100.0]), 1.0), True),
              (2, 3, oo.ProductPool(np.array([130.0, 100.0]), 1.0), True)]
    res = tv.dp(1, tv.EXACT_IN, 1.0, tv.pool_lists(pools), 3, None, 8, tv.pool_quote(pools))
    assert res.status[1] == tv.REPEATS_POOL and res.hops[1] > 1
    steps = [k for _, _, k in res.walk(2)]
    assert len(set(steps)) < len(steps)
