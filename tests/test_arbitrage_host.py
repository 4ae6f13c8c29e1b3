"""The arbitrage rows and scan of include/cfmm_b200.h on the host (arbitrage_oracle.py), no GPU.

An arbitrage row (base p, other x, hubs y) is route! with BasketLiquidation(p, 0) over the pools of
{x, p}, {x, y} and {y, p}: checked against scipy route() on exactly those pools, and on the
quick-start pools of the README.  On small random graphs every pair cycle and triangle through the
base tokens that is worth min_profit on its own must be covered by a scan row, and every scan row
passes the 50-digit certificate at δ = 0 (arbitrage_certificate.py)."""
import numpy as np
import pytest

import arbitrage_certificate as ac
import arbitrage_oracle as ao
import order_certificate as oc
import split_oracle as so
from test_routed_orders_host import hub_market
from test_split_orders_host import SplitPools, random_pair_pools


def basket_route(cr, spec, base, n):
    """Ψ of route() with BasketLiquidation(base, 0) over ProductTwoCoin pools spec = [(Ai, R)], γ 0.997."""
    cs = [cr.ProductTwoCoin(R, 0.997, Ai) for Ai, R in spec]
    r = cr.Router(cr.BasketLiquidation(base, [0.0] * n), cs, n, _pools_factory=SplitPools)
    cr.route(r, pgtol=1e-10, factr=1e1)
    return cs, cr.netflows(r)


@pytest.mark.parametrize("nh", [0, 1, 3], ids=["pair", "triangle", "three-hubs"])
def test_rows_match_route_on_the_row_pools(cr, nh):
    rng = np.random.default_rng(30 + nh)
    for trial in range(3):
        hubs = [3, 4, 5][:nh]
        spec = hub_market(rng, hubs, direct=2)
        n = 2 + nh
        cs, psi = basket_route(cr, spec, 1, n)
        mirror = [so.Product(c.R, c.gamma, c.Ai) for c in cs]
        of = lambda a, b: [mirror[k] for k, c in enumerate(cs) if set(c.Ai) == {a, b}]
        row = ao.arb_row(of(2, 1), [(h, of(2, h), of(h, 1)) for h in hubs], 1, 2)
        assert row["status"] == ao.FILLED and row["profit"] > 0.0
        scale = max(psi[0], 1e-3)
        assert abs(row["profit"] - psi[0]) <= 1e-5 * scale, (trial, row["profit"], psi[0])
        assert np.all(psi[1:] >= -1e-4 * scale), psi  # L-BFGS-B leaves a small constraint residual
        assert row["surplus_in"] >= 0.0 and all(x >= 0.0 for x in row["hub_surplus"])
        of_k = lambda a, b: [k for k, c in enumerate(cs) if set(c.Ai) == {a, b}]
        keys = of_k(2, 1) + [k for h in hubs for k in of_k(2, h) + of_k(h, 1)]  # the legs' list order
        for pos, k in enumerate(keys):  # the legs keep the invariant, to rounding relative to R₀R₁
            D, L, R = row["D"][pos], row["L"][pos], cs[k].R
            n = R + cs[k].gamma * D - L
            assert np.all(D >= 0.0) and np.all(L >= 0.0) and n[0] * n[1] >= R[0] * R[1] * (1 - 1e-12)


def test_readme_quick_start_pools(cr):
    """Two ProductTwoCoin pools on {1, 2}, γ = 1: route() with LinearNonnegative([1, 1]) leaves Ψ₂ ≈ 171.40;
    the arbitrage row with base 2 and other 1 finds the same cycle."""
    spec = [([1, 2], [1e6, 1e6]), ([1, 2], [1e3, 2e3])]
    cs = [cr.ProductTwoCoin(R, 1.0, Ai) for Ai, R in spec]
    r = cr.Router(cr.LinearNonnegative([1.0, 1.0]), cs, 2, _pools_factory=SplitPools)
    cr.route(r, pgtol=1e-10, factr=1e1)
    psi = cr.netflows(r)
    assert abs(psi[1] - 171.40) < 0.01 and abs(psi[0]) < 1e-3
    row = ao.arb_row([so.Product(c.R, c.gamma, c.Ai) for c in cs], [], 2, 1)
    assert row["status"] == ao.FILLED
    assert abs(row["profit"] - psi[1]) <= 1e-5 * psi[1], (row["profit"], psi[1])
    # the rates screen it: r(2 → 1) · r(1 → 2) = 1 · 2
    by = {(1, 2): [so.Product(c.R, c.gamma, c.Ai) for c in cs]}
    found, rows = ao.scan(by, lambda a, b: by[(min(a, b), max(a, b))], [2], [1.0], 7)
    assert found == 1 and rows[0]["other"] == 1 and rows[0]["profit"] == row["profit"]


def random_graph(rng, n, n_pairs, types):
    pairs = sorted({tuple(sorted(rng.choice(np.arange(1, n + 1), size=2, replace=False).tolist()))
                    for _ in range(n_pairs)})
    by = {}
    for a, b in pairs:
        by[(a, b)] = random_pair_pools(rng, int(rng.integers(1, 4)), types, a=a, b=b)
        for p in by[(a, b)]:
            if rng.random() < 0.1:
                p.active = False
    return by


def cert_pool(p):
    if isinstance(p, so.GeoMean):
        return oc.geomean(p.R, p.g, p.w, p.Ai, p.active)
    if isinstance(p, so.Product):
        return oc.product(p.R, p.g, p.Ai, p.active)
    return oc.univ3(p.price, p.lt, p.lq, p.g, p.Ai, p.active)


@pytest.mark.parametrize("types", [(0,), (2,), (0, 1, 2)], ids=["product", "univ3", "mixed"])
def test_scan_covers_every_cycle_and_is_certified(types):
    rng = np.random.default_rng(50 + len(types) + types[0])
    for trial in range(2):
        by = random_graph(rng, 7, 14, types)
        pairs = lambda a, b: by.get((min(a, b), max(a, b)), [])
        base, mins = [1, 2], [1e-3, 1e-3]
        found, rows = ao.scan(by, pairs, base, mins, 7)
        assert found == len(rows)
        covered = set()
        for r in rows:
            covered.add((r["base"], r["other"]))
            covered |= {(r["base"], r["other"], y) for y in r["hubs"]}
        nbr = {}
        for a, b in by:
            nbr.setdefault(a, set()).add(b)
            nbr.setdefault(b, set()).add(a)
        checked = 0
        alone = lambda p, x: ao.arb_row(pairs(x, p), [], p, x)
        worth = lambda row, m: row["status"] == ao.FILLED and row["profit"] >= m * (1 + 1e-9)
        for bi, p in enumerate(base):
            for x in sorted(nbr.get(p, ())):
                if worth(alone(p, x), mins[bi]):
                    assert (p, x) in covered, (trial, p, x)
                    checked += 1
                for y in sorted(nbr[p] & nbr[x]):
                    row = ao.arb_row(pairs(x, p), [(y, pairs(x, y), pairs(y, p))], p, x)
                    if not worth(row, mins[bi]):
                        continue
                    # the triangle itself, or the pair cycles on {x, p} and {y, p} the row's pools also
                    # hold, when the triangle adds less than min_profit to them
                    pairs_alone = alone(p, x)["profit"] + alone(p, y)["profit"]
                    assert (p, x, y) in covered or (p, y, x) in covered or (
                        ((p, x) in covered or (p, y) in covered) and row["profit"] - pairs_alone < mins[bi]), \
                        (trial, p, x, y, row["profit"])
                    checked += 1
        assert checked >= 1
        # every row: its profit, and the 50-digit bound at δ = 0
        for r in rows:
            p, x, hs = r["base"], r["other"], r["hubs"]
            row = ao.arb_row(pairs(x, p), [(y, pairs(x, y), pairs(y, p)) for y in hs], p, x)
            assert row["profit"] == r["profit"] and row["profit"] >= mins[base.index(p)]
            cp = lambda a, b: [cert_pool(q) for q in pairs(a, b)]
            crow = oc.Row(cp(x, p), [(y, cp(x, y), cp(y, p)) for y in hs], x, p)
            c = ac.certify_arbitrage(crow, row)
            assert c["gap"] is not None and c["gap"] <= c["allowance"]


def test_screen_and_order():
    """Rates are the best boundary per direction (retired pools and NaNs ignored, 0 without an active
    pool); hubs are kept in (score desc, y asc) order up to max_hubs; rows sort by (base, profit desc, x)."""
    rng = np.random.default_rng(4)
    by = random_graph(rng, 6, 12, (0,))
    r = ao.rates(by)
    for (a, b), pools in by.items():
        act = [p for p in pools if p.active]
        assert r[(a, b)] == max([p.boundary(b, a) for p in act], default=0.0)
        assert r[(b, a)] == max([p.boundary(a, b) for p in act], default=0.0)
    for mh in (0, 1, 2, 7):
        cands = ao.candidates(by, [1, 3], mh)
        assert [(b, x) for b, _, x, _ in cands] == sorted((b, x) for b, _, x, _ in cands)
        assert all(len(h) <= mh for *_, h in cands)
    pairs = lambda a, b: by.get((min(a, b), max(a, b)), [])
    found, rows = ao.scan(by, pairs, [1, 3], [1e-6, 1e-6], 7)
    key = [([1, 3].index(x["base"]), -x["profit"], x["other"]) for x in rows]
    assert key == sorted(key)
    for cap in (0, 1, found):
        assert ao.scan(by, pairs, [1, 3], [1e-6, 1e-6], 7, cap) == (found, rows[:cap])


def test_replay_limits_and_reverts():
    """Execute in batch order: a row re-solves on the state the earlier rows left, so a repeated row
    finds the cycle closed; a min_profit above the profit reverts and changes nothing."""
    rng = np.random.default_rng(8)
    spec = hub_market(rng, [3], direct=2)
    pools = [so.Product(R, 0.997, Ai) for Ai, R in spec]
    of = lambda a, b: [p for p in pools if set(p.Ai) == {a, b}]
    pairs = lambda a, b: of(a, b)
    q = ao.quote_arbitrage(pairs, [1], [2], [0, 1], [3])[0]
    assert q["profit"] > 0.0
    before = [p.R.copy() for p in pools]
    rows = ao.replay_arbitrage(pairs, [1], [2], [0, 1], [3], [q["profit"] * 2])
    assert rows[0]["status"] == ao.LIMIT and rows[0]["profit"] == 0.0
    assert all(np.array_equal(p.R, b) for p, b in zip(pools, before))
    rows = ao.replay_arbitrage(pairs, [1, 1], [2, 2], [0, 1, 2], [3, 3], [q["profit"], 0.0])
    assert rows[0]["status"] == ao.FILLED and rows[0]["profit"] == q["profit"]
    assert abs(rows[1]["profit"]) <= 1e-9 * q["profit"]
    assert any(not np.array_equal(p.R, b) for p, b in zip(pools, before))
