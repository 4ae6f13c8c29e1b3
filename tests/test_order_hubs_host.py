"""cfmm_choose_order_hubs (include/cfmm_b200.h) on the host (hub_oracle.py), no GPU.

The mirror restates the kernel: candidates from the token adjacency, a warp of 32 lanes that each
keep their best max_hubs hubs, a warp-wide merge of the heads.  On random graphs of ProductTwoCoin,
GeometricMeanTwoCoin and UniV3 pools, with retired pools and allowed masks, it must agree with the
definition (every token tried, ranked with sorted()) for both kinds and every max_hubs 0..7.  The
Python layers reject bad arguments before they reach the library."""
import types

import numpy as np
import pytest

import hub_oracle as ho
import swap_order_oracle as oo


def random_market(rng, synth, n, n_pairs, hubs=(), retire=0.1):
    """Pools (a, b, pool, active) on n tokens: n_pairs random pairs with 1-3 pools each, plus every
    hub of `hubs` paired with most tokens (so rows see many candidates, more than a warp on large n)."""
    pairs = {tuple(sorted(rng.choice(np.arange(1, n + 1), size=2, replace=False).tolist())) for _ in range(n_pairs)}
    pairs |= {tuple(sorted((h, x))) for h in hubs for x in range(1, n + 1) if x != h and rng.random() < 0.8}
    cp, gu, _, off, lt, lq = synth.univ3_pools(4 * len(pairs) + 4, n, seed=int(rng.integers(1 << 30)), ragged=True)
    pools, u = [], 0
    nu = np.exp(rng.uniform(-2, 2, size=n + 1))
    for a, b in sorted(pairs):
        for _ in range(int(rng.integers(1, 4))):
            Ai = (a, b) if rng.random() < 0.5 else (b, a)
            depth = 10.0 ** rng.uniform(1, 4)
            R = depth / nu[list(Ai)] * np.exp(rng.uniform(-0.1, 0.1, size=2))
            kind = rng.integers(0, 3)
            if kind == 0:
                p = oo.ProductPool(R, rng.choice([0.997, 0.9995, 1.0]))
            elif kind == 1:
                p = oo.GeoMeanPool(R, 0.997, rng.uniform(0.3, 0.7, size=2))
            else:
                sl = slice(off[u], off[u + 1])
                target = nu[Ai[0]] / nu[Ai[1]] * np.exp(rng.uniform(-0.05, 0.05))
                p = oo.Univ3Pool(target, lt[sl] * target / cp[u], lq[sl] * depth / 100.0, gu[u])
                u += 1
            pools.append((Ai[0], Ai[1], p, bool(rng.random() >= retire)))
    return pools


def random_rows(rng, n, q, pools):
    tin = rng.integers(1, n + 1, size=q)
    tout = np.array([rng.choice([x for x in range(1, n + 1) if x != a]) for a in tin])
    kind = rng.integers(0, 2, size=q).astype(np.uint8)
    scale = np.median([p[2].f(1.0, True) for p in pools[:20]]) if pools else 1.0
    amount = 10.0 ** rng.uniform(-3, 3, size=q) * max(scale, 1e-6)
    amount[::11] = 0.0
    return tin.astype(np.int64), tout.astype(np.int64), kind, amount


def same(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y)), (x, y)


@pytest.mark.parametrize("seed", range(4))
def test_mirror_equals_definition(synth, seed):
    rng = np.random.default_rng(1000 + seed)
    n = 16
    pools = random_market(rng, synth, n, 40, hubs=(1, 2, 3))
    tin, tout, kind, amount = random_rows(rng, n, 24, pools)
    for max_hubs in range(8):
        got = ho.choose(pools, n, tin, tout, kind, amount, max_hubs)
        same(got, ho.brute(pools, n, tin, tout, kind, amount, max_hubs))
        off, hubs, score, n_elig = got
        assert off[0] == 0 and np.all(np.diff(off) == np.minimum(n_elig, max_hubs))
        assert np.all(n_elig[amount == 0.0] == 0)
    allowed = rng.random(n) < 0.6
    same(ho.choose(pools, n, tin, tout, kind, amount, 7, allowed),
         ho.brute(pools, n, tin, tout, kind, amount, 7, allowed))


def test_wide_rows_and_ties(synth):
    """Rows between two hubs of degree > 32 spread their candidates over every lane; duplicated pools
    make equal scores, which rank by token."""
    rng = np.random.default_rng(7)
    n = 80
    pools = [p for p in random_market(rng, synth, n, 30, hubs=(1, 2), retire=0.0) if not 60 < max(p[:2])]
    # tokens 61..70 get identical pools to hubs 1 and 2 and nothing else, so their scores tie
    R = np.array([1000.0, 1000.0])
    pools += [(x, h, oo.ProductPool(R, 0.997), True) for x in range(61, 71) for h in (1, 2)]
    tin = np.array([1, 2, 1, 2], dtype=np.int64)
    tout = np.array([2, 1, 2, 1], dtype=np.int64)
    kind = np.array([0, 0, 1, 1], dtype=np.uint8)
    amount = np.array([5.0, 5.0, 1.0, 1.0])
    for max_hubs in (1, 3, 7):
        got = ho.choose(pools, n, tin, tout, kind, amount, max_hubs)
        same(got, ho.brute(pools, n, tin, tout, kind, amount, max_hubs))
        assert np.all(got[3] > 32)


def test_retired_pools_and_masks(synth):
    """A pair whose pools are all retired stays in the adjacency but gives no route; a masked hub is
    never chosen."""
    R = np.array([1000.0, 1000.0])
    pools = [(1, 3, oo.ProductPool(R, 0.997), True), (3, 2, oo.ProductPool(R, 0.997), True),
             (1, 4, oo.ProductPool(R, 0.997), True), (4, 2, oo.ProductPool(R, 0.997), False),
             (1, 5, oo.ProductPool(R * 2, 0.997), True), (5, 2, oo.ProductPool(R * 2, 0.997), True)]
    args = (np.array([1, 1]), np.array([2, 2]), np.array([0, 1], np.uint8), np.array([10.0, 10.0]))
    off, hubs, score, n_elig = ho.choose(pools, 5, *args, 7)
    assert off.tolist() == [0, 2, 4] and n_elig.tolist() == [2, 2]
    assert hubs.tolist() == [5, 3, 5, 3]  # the deeper route first, for both kinds
    assert score[0] > score[1] and score[2] < score[3]
    allowed = np.array([1, 1, 1, 1, 0], dtype=bool)
    off, hubs, _, n_elig = ho.choose(pools, 5, *args, 7, allowed)
    assert hubs.tolist() == [3, 3] and n_elig.tolist() == [1, 1]
    same(ho.choose(pools, 5, *args, 7, allowed), ho.brute(pools, 5, *args, 7, allowed))


def test_exact_out_beyond_depth_is_not_eligible():
    R = np.array([1000.0, 1000.0])
    pools = [(1, 3, oo.ProductPool(R, 0.997), True), (3, 2, oo.ProductPool(R, 0.997), True)]
    off, hubs, score, n_elig = ho.choose(pools, 3, [1, 1], [2, 2], [1, 1], [999.0, 1000.0], 7)
    assert off.tolist() == [0, 0, 0] and n_elig.tolist() == [0, 0]  # the first hop cannot pay c_h
    off, hubs, score, n_elig = ho.choose(pools, 3, [1], [2], [1], [100.0], 7)
    c = oo.exact_out(pools[1][2], 100.0, False)[0]
    assert hubs.tolist() == [3] and score[0] == oo.exact_out(pools[0][2], c, True)[0]


def _stub_pools(cr, n_tokens=5):
    def fail(*a):
        raise AssertionError("the library must not be called")
    return types.SimpleNamespace(n_tokens=n_tokens, _ctx=None, _chk=fail,
                                 _lib=types.SimpleNamespace(cfmm_choose_order_hubs=fail))


def test_python_argument_checks(cr):
    stub = _stub_pools(cr)
    with pytest.raises(ValueError, match="one entry per row"):
        cr.DevicePools.choose_order_hubs(stub, [1, 2], [2], [0, 0], [1.0, 1.0])
    with pytest.raises(ValueError, match="allowed must have 5 entries"):
        cr.DevicePools.choose_order_hubs(stub, [1], [2], [0], [1.0], 7, allowed=[1, 1, 1])
    router = types.SimpleNamespace(_world=1, _pools=stub, _split_args=None)
    router._split_args = lambda *a: cr.Router._split_args(router, *a)
    for bad in (-1, 8):
        with pytest.raises(ValueError, match="max_hubs must be 0..7"):
            cr.Router._choose(router, [1], [2], [0], [1.0], bad, None, "choose_hubs")
    with pytest.raises(ValueError, match="one entry per row"):
        cr.Router._choose(router, [1], [2, 3], [0], [1.0], 3, None, "choose_hubs")
    router._world = 2
    with pytest.raises(NotImplementedError, match="drives one GPU"):
        cr.Router._choose(router, [1], [2], [0], [1.0], 3, None, "choose_hubs")
