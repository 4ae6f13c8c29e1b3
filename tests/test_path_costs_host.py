"""cfmm_find_order_paths_net / cfmm_quote_token_values_net (include/cfmm_b200.h) on the host
(path_cost_oracle.py), no GPU.

On small ProductTwoCoin markets without gaining cycles (every pool's marginal price agrees with one
price vector, fees > 0), the selection over the existing DP at L = 1 … H must give every row and every
token the best net over a brute-force enumeration of every walk of at most H hops with distinct pools:
the header's argument that the selection is exact.  The selected hops never grow with the hop cost;
κ = +inf keeps the largest filled L; the numpy form equals the scalar one; and the Python packing of
hop_cost rejects what the library would."""
import itertools

import numpy as np
import pytest

import best_path_oracle as bo
import hub_oracle as ho
import path_cost_oracle as pc
import swap_order_oracle as oo
import token_value_oracle as tv
from test_token_values_host import arrays

INF = float("inf")


def consistent_market(rng, n, n_pairs):
    """ProductTwoCoin pools (a, b, pool, active) whose marginal prices all agree with one price vector."""
    nu = np.exp(rng.uniform(-1, 1, size=n + 1))
    pairs = {tuple(sorted(rng.choice(np.arange(1, n + 1), size=2, replace=False).tolist())) for _ in range(n_pairs)}
    pools = []
    for a, b in sorted(pairs):
        for _ in range(int(rng.integers(1, 3))):
            Ai = (a, b) if rng.random() < 0.5 else (b, a)
            R = 10.0 ** rng.uniform(1, 3) / nu[list(Ai)]
            pools.append((Ai[0], Ai[1], oo.ProductPool(R, rng.choice([0.997, 0.999])), bool(rng.random() >= 0.1)))
    return pools


def walk_amount(pools, toks, ks, kind, amount):
    """The amount a walk carries (exact-in received, exact-out paid), or None when it carries none."""
    out = kind == bo.EXACT_OUT
    v = amount
    for h in (range(len(ks) - 1, -1, -1) if out else range(len(ks))):
        pool, a = pools[ks[h]], toks[h]
        v = float(oo.exact_out(pool[2], v, a == pool[0])[0]) if out else float(pool[2].f(v, a == pool[0]))
        if not (v < INF if out else v > 0.0):
            return None
    return v


def brute_net(pools, n, j, i, kind, amount, H, allowed, kappa):
    """The best net over every walk j → … → i of at most H hops through allowed tokens (j and i only
    at its ends), one active pool per hop, no pool twice."""
    pairs = ho.pair_lists(pools)
    mids = [t for t in range(1, n + 1) if (allowed is None or allowed[t - 1]) and t not in (j, i)]
    out, best = kind == bo.EXACT_OUT, None
    for L in range(1, H + 1):
        for mid in itertools.product(mids, repeat=L - 1):
            toks = [j, *mid, i]
            choices = [[k for k in pairs.get((min(a, b), max(a, b)), []) if pools[k][3]] for a, b in zip(toks, toks[1:])]
            for ks in itertools.product(*choices):
                if len(set(ks)) < len(ks):
                    continue
                v = walk_amount(pools, toks, ks, kind, amount)
                if v is None:
                    continue
                x = pc.net(v, L, kappa, out)
                if best is None or (x < best if out else x > best):
                    best = x
    return best


@pytest.mark.parametrize("seed", range(3))
def test_best_paths_selection_is_the_best_net_over_every_walk(seed):
    rng = np.random.default_rng(9100 + seed)
    n = 6
    pools = consistent_market(rng, n, 11)
    lists, quote = bo.pool_lists(pools), bo.pool_quote(pools)
    shorter = 0
    for H in (2, 3, 4):
        allowed = rng.random(n) < 0.85
        rows = []
        for _ in range(8):
            j, i = (int(x) for x in rng.choice(np.arange(1, n + 1), size=2, replace=False))
            rows.append((j, i, int(rng.integers(0, 2)), float(10.0 ** rng.uniform(-1, 1.5))))
        for scale in (0.0, 1e-4, 1e-2, 0.3):
            kappa = [scale * a for _, _, _, a in rows]
            for r, (walk, st, amt, x, L) in enumerate(pc.paths(rows, lists, n, allowed, H, quote, kappa)):
                j, i, kind, a = rows[r]
                best = brute_net(pools, n, j, i, kind, a, H, allowed, kappa[r])
                if best is None:
                    assert st == bo.UNREACHABLE
                    continue
                assert st == bo.FILLED and x == best, (H, r, x, best)
                assert x == pc.net(amt, len(walk), kappa[r], kind == bo.EXACT_OUT)
                shorter += len(walk) < H and scale > 0
    assert shorter > 0


@pytest.mark.parametrize("seed", range(3))
def test_token_values_selection_is_the_best_net_over_every_walk(seed):
    rng = np.random.default_rng(9200 + seed)
    n = 6
    pools = consistent_market(rng, n, 11)
    lists, quote = tv.pool_lists(pools), tv.pool_quote(pools)
    checked = 0
    for H in (2, 3, 4):
        mask = rng.random(n) < 0.85
        for kind in (tv.EXACT_IN, tv.EXACT_OUT):
            root = int(rng.integers(1, n + 1))
            mask[root - 1] = True
            amount = float(10.0 ** rng.uniform(-1, 1.5))
            kappa = amount * 10.0 ** rng.uniform(-5, -0.5, size=n)
            _, value, hops, status, net, sel, walk = pc.values(root, kind, amount, lists, n, mask, H, quote, kappa)
            assert value[root - 1] == amount and net[root - 1] == amount and hops[root - 1] == 0
            for t in range(1, n + 1):
                if t == root:
                    continue
                if not mask[t - 1]:  # only allowed tokens are reached
                    assert status[t - 1] == tv.UNREACHABLE
                    continue
                j, i = (t, root) if kind else (root, t)
                best = brute_net(pools, n, j, i, kind, amount, H, mask, kappa[t - 1])
                if best is None:
                    assert status[t - 1] == tv.UNREACHABLE
                    continue
                assert status[t - 1] == tv.FILLED and net[t - 1] == best, (H, t, net[t - 1], best)
                assert len(walk(t)) == hops[t - 1] <= sel[t - 1]
                checked += 1
    assert checked > 15


@pytest.mark.parametrize("seed", range(2))
def test_hops_never_grow_with_the_cost(seed):
    rng = np.random.default_rng(9300 + seed)
    n = 8
    pools = consistent_market(rng, n, 20)
    lists, quote = bo.pool_lists(pools), bo.pool_quote(pools)
    rows = []
    for _ in range(10):
        j, i = (int(x) for x in rng.choice(np.arange(1, n + 1), size=2, replace=False))
        rows.append((j, i, int(rng.integers(0, 2)), float(10.0 ** rng.uniform(-1, 1.5))))
    prev = None
    for scale in (0.0, 1e-6, 1e-4, 1e-3, 1e-2, 1e-1, 1.0):
        got = pc.paths(rows, lists, n, np.ones(n, bool), 5, quote, [scale * a for *_, a in rows])
        hops = [len(w) for w, *_ in got]
        if prev is not None:
            assert all(a <= b for a, b in zip(hops, prev)), (scale, hops, prev)
        prev = hops
    tl, tq = tv.pool_lists(pools), tv.pool_quote(pools)
    for kind in (0, 1):
        prev = None
        for scale in (0.0, 1e-5, 1e-3, 1e-1):
            hops = pc.values(2, kind, 5.0, tl, n, None, 5, tq, np.full(n, 5.0 * scale))[2]
            if prev is not None:
                assert np.all(hops <= prev)
            prev = hops


def test_infinite_cost_keeps_the_largest_filled_level():
    rng = np.random.default_rng(9400)
    n = 7
    pools = consistent_market(rng, n, 16)
    lists, quote = tv.pool_lists(pools), tv.pool_quote(pools)
    for kind in (0, 1):
        kappa = np.full(n, INF)
        kappa[::2] = 0.0
        per_L, value, hops, status, net, sel, _ = pc.values(3, kind, 2.0, lists, n, None, 4, quote, kappa)
        last = per_L[-1]
        for t in range(1, n + 1):
            if t == 3 or not np.isinf(kappa[t - 1]):
                continue
            filled = [L for L in range(1, 5) if per_L[L - 1].status[t - 1] == tv.FILLED]
            if not filled:
                assert net[t - 1] == last.value[t - 1] and status[t - 1] == last.status[t - 1]
                continue
            assert sel[t - 1] == max(filled) and net[t - 1] == (INF if kind else -INF)
            assert value[t - 1] == per_L[max(filled) - 1].value[t - 1]
    # a row: the largest filled L, with net ∓inf
    rows = [(1, 5, 0, 3.0), (5, 1, 1, 3.0)]
    got = pc.paths(rows, bo.pool_lists(pools), n, np.ones(n, bool), 4, bo.pool_quote(pools), [INF, INF])
    per_L = [bo.dp(rows, bo.pool_lists(pools), n, np.ones(n, bool), L, bo.pool_quote(pools)) for L in range(1, 5)]
    for r, (walk, st, amt, x, L) in enumerate(got):
        filled = [L for L in range(1, 5) if per_L[L - 1][r][1] == bo.FILLED]
        assert L == (max(filled) if filled else 4)
        if filled:
            assert x == (INF if rows[r][2] else -INF)


@pytest.mark.parametrize("seed", range(2))
def test_vectorised_selection_equals_the_scalar_one(seed):
    rng = np.random.default_rng(9500 + seed)
    n = 12
    pools = consistent_market(rng, n, 30)
    R, g, Ai, act = arrays(pools)
    lists, quote = tv.pool_lists(pools), tv.pool_quote(pools)
    for H in (1, 3, 6):
        root = int(rng.integers(1, n + 1))
        amount = float(10.0 ** rng.uniform(-1, 1.5))
        kappa = amount * 10.0 ** rng.uniform(-6, -1, size=n)
        kappa[0] = INF
        _, value, hops, status, net, _, _ = pc.values(root, 0, amount, lists, n, None, H, quote, kappa)
        v2, h2, n2 = pc.product(R, g, Ai, act, n, root, amount, H, kappa)
        assert np.all(status[value > 0] == tv.FILLED)
        assert np.array_equal(value, v2) and np.array_equal(hops, h2) and np.array_equal(net, n2)


def test_hop_cost_packing():
    from cfmmrouter_b200.router import pack_hop_cost
    assert np.array_equal(pack_hop_cost(2.5, 4, None, "f"), [2.5] * 4)
    assert np.array_equal(pack_hop_cost(2.5, 4, [1, 3], "f"), [2.5, 2.5])
    per_token = np.array([1.0, 2.0, INF, 0.0])
    assert np.array_equal(pack_hop_cost(per_token, 4, None, "f"), per_token)
    assert np.array_equal(pack_hop_cost(per_token, 4, np.array([3, 1, 4]), "f"), [INF, 1.0, 0.0])
    for bad, msg in ((np.nan, "NaN or negative"), (-1.0, "NaN or negative"), ([1.0, 2.0], "one per token"),
                     ([1.0, -0.5, 0.0, 0.0], "NaN or negative"), ([1.0, np.nan, 0.0, 0.0], "NaN or negative")):
        with pytest.raises(ValueError) as e:
            pack_hop_cost(bad, 4, None, "find_paths")
        assert msg in str(e.value) and "find_paths" in str(e.value)
    assert pack_hop_cost([1, 2, 3, 4], 4, None, "f").dtype == np.float64
