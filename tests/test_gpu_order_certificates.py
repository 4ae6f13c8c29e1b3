"""cfmm_quote/execute_split_orders and cfmm_quote/execute_routed_orders (include/cfmm_b200.h)
certified on the device by the 50-digit duality bound of order_certificate.py.

  * Deep pairs: pairs holding 1, 31, 32, 33, 64, 65 and 200 pools of every type, both token
    orientations, fees {1, 0.9995, 0.997}, reserves from 1e-3 to 1e9, some pools mispriced beyond
    their fees (so the optimum trades some pools in reverse), GeometricMean weights down to
    (0.05, 0.95), UniV3 ladders with zero-liquidity gaps and empty last ticks; a main set laid out
    with orient_by_degree = 1, appended pools and retired pools.  Pairs deeper than a warp take the
    kernels' lane loops past their first iteration.
  * Full hub sets: seven hubs (the whole CTA), one hub with 20 pools on {j, h} and 25 on {h, i},
    hubs with pools on one side only, a hub far better than the direct pools, a useless hub, and rows
    with no direct pool.
  * Amounts from 1e-9 of the depth to 0.99 of it, both kinds, and exact-out amounts just below and
    just above the depth.
  * Executes: a batch with several rows on one deep pair, certified row by row on the state each
    row saw, and equal bit for bit to the same rows run one call at a time."""
import numpy as np
import pytest

import order_certificate as oc
from test_gpu_parity import make_pools
from test_gpu_paths import APPEND, same_state
from test_gpu_split_orders import expected_pairs

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
DEEP = {(1, 2): 1, (1, 3): 31, (2, 3): 32, (1, 4): 33, (2, 4): 64, (3, 4): 65, (5, 6): 200}
J, I, J2 = 1, 2, 10                      # hub rows: j = 1 (direct pools) or 10 (none), i = 2
HUBS = (3, 4, 5, 6, 7, 8, 9)


def ladder(rng, price, depth):
    """A UniV3 ladder around price: 3-8 ticks, some with zero liquidity, the last one often empty."""
    n = int(rng.integers(3, 9))
    top = price * rng.uniform(1.1, 2.0)
    lt = top * np.cumprod(np.concatenate([[1.0], rng.uniform(0.55, 0.9, size=n - 1)]))
    if lt[-1] >= price:
        lt = np.concatenate([lt, [price * 0.7]])
        n += 1
    lq = depth ** 2 / price * rng.uniform(0.2, 2.0, size=n)
    lq[rng.random(n) < 0.2] = 0.0
    cur = int(np.sum(lt >= price))
    lq[cur - 1] = max(lq[cur - 1], depth ** 2 / price * 0.5)  # the current tick trades
    if rng.random() < 0.5:
        lq[-1] = 0.0
    return lt, lq


class PoolSet:
    """Pools given as (type, Ai, state) specs, split into a main set (orient_by_degree = 1) and
    appended pools per type, some retired; the attributes test_gpu_split_orders' helpers read.
    keep_pairs: retire no pair's last active pool (a retire then never changes which pairs are active).
    build: make the device context now (else p is None until fresh())."""

    def __init__(self, cr, n, specs, seed, tail=0.2, retire=0.06, keep_pairs=False, build=True):
        rng = np.random.default_rng(seed)
        self._cr, self.n = cr, n
        by = {t: [s for s in specs if s[0] == t] for t in (P, G, U)}
        self.Ai, self.g, self.main, self.tail, self.mm, self.mt, self.m = {}, {}, {}, {}, {}, {}, {}
        self.w = np.array([s[2]["w"] for s in by[G]]).reshape(-1, 2)
        for t in (P, G, U):
            ss = by[t]
            m = len(ss)
            A = np.array([s[1] for s in ss], dtype=np.int64).reshape(-1, 2)
            g = np.array([s[2]["g"] for s in ss])
            self.Ai[t], self.g[t], self.m[t] = A, g, m
            k = m - int(round(m * tail))
            self.mm[t], self.mt[t] = k, m - k
            if t == U:
                cp = np.array([s[2]["price"] for s in ss])
                off = np.concatenate([[0], np.cumsum([len(s[2]["lt"]) for s in ss])]).astype(np.int64)
                lt = np.concatenate([s[2]["lt"] for s in ss]) if m else np.zeros(0)
                lq = np.concatenate([s[2]["lq"] for s in ss]) if m else np.zeros(0)
                o1 = off[k]
                self.main[t] = (cp[:k], g[:k], A[:k], off[:k + 1], lt[:o1], lq[:o1])
                self.tail[t] = (cp[k:], g[k:], A[k:], off[k:] - o1, lt[o1:], lq[o1:])
            else:
                R = np.array([s[2]["R"] for s in ss]).reshape(-1, 2)
                data = (R, g, A) + ((self.w,) if t == G else ())
                self.main[t] = tuple(x[:k] for x in data)
                self.tail[t] = tuple(x[k:] for x in data)
        self.retired = {(t, int(i)) for t in (P, G, U) for i in range(self.m[t]) if rng.random() < retire}
        if keep_pairs:
            by_pair = {}
            for k in self.keys():
                by_pair.setdefault(frozenset(int(x) for x in self.Ai[k[0]][k[1]]), []).append(k)
            self.retired -= {ks[0] for ks in by_pair.values() if all(k in self.retired for k in ks)}
        self.p = self.fresh() if build else None

    def fresh(self):
        kw = {("product", "geomean", "univ3")[t]: self.main[t] for t in (P, G, U) if self.mm[t]}
        p = make_pools(self._cr, self.n, pre={"orient_by_degree": 1}, **kw)
        for t in (P, G, U):
            if self.mt[t]:
                getattr(p, APPEND[t])(*self.tail[t])
            if self.m[t]:
                act = np.ones(self.m[t], bool)
                act[[i for (s, i) in self.retired if s == t]] = False
                p.set_active(t, 0, act)
        return p

    def state(self, p):
        return [p.pool_state(t)[0].copy() for t in (P, G, U) if self.m[t]] + \
            (list(p.univ3_ticks()) if self.m[U] else [])

    def keys(self):
        return [(t, i) for t in (P, G, U) for i in range(self.mm[t])] + \
            [(t, self.mm[t] + i) for t in (P, G, U) for i in range(self.mt[t])]

    def cert_pools(self, p):
        """order_certificate pools at p's current state, keyed (type, index)."""
        out = {}
        for t in (P, G, U):
            if not self.m[t]:
                continue
            st = p.pool_state(t)[0]
            if t == U:
                off, lt, lq = p.univ3_ticks()
            for i in range(self.m[t]):
                act = (t, i) not in self.retired
                Ai = self.Ai[t][i]
                if t == P:
                    out[(t, i)] = oc.product(st[i], self.g[t][i], Ai, act)
                elif t == G:
                    out[(t, i)] = oc.geomean(st[i], self.g[t][i], self.w[i], Ai, act)
                else:
                    out[(t, i)] = oc.univ3(st[i], lt[off[i]:off[i + 1]], lq[off[i]:off[i + 1]], self.g[t][i], Ai, act)
        return out

    def row(self, objs, j, i, hubs=()):
        ks = self.keys()
        lst = lambda a, b: [objs[k] for k in expected_pairs(self, ks, a, b)]
        return oc.Row(lst(j, i), [(h, lst(j, h), lst(h, i)) for h in hubs], j, i)


def pool_spec(rng, t, a, b, nu, depth=None, misprice=None, fees=(1.0, 0.9995, 0.997)):
    Ai = [a, b] if rng.random() < 0.5 else [b, a]
    depth = 10.0 ** rng.uniform(-3, 9) if depth is None else depth
    mis = np.exp(rng.choice([-1, 1]) * rng.uniform(0.004, 0.05)) if misprice is None else misprice
    g = float(rng.choice(fees))
    if t == U:
        price = nu[Ai[0]] / nu[Ai[1]] * mis
        lt, lq = ladder(rng, price, depth / nu[Ai[1]])
        return (t, Ai, dict(g=g, price=price, lt=lt, lq=lq))
    R = np.array([depth / nu[Ai[0]], depth / nu[Ai[1]]])
    R[0] *= mis
    if t == G:
        w = [0.05, 0.95] if rng.random() < 0.3 else list(rng.uniform(0.2, 0.8, size=2))
        if rng.random() < 0.5:
            w = w[::-1]
        R = np.array([depth * w[0] / nu[Ai[0]], depth * w[1] / nu[Ai[1]]])  # spot price ν at weights w
        R[0] *= mis
        return (t, Ai, dict(g=g, R=R, w=w))
    return (t, Ai, dict(g=g, R=R))


@pytest.fixture(scope="module")
def deep(cr):
    rng = np.random.default_rng(71)
    nu = {t: float(np.exp(rng.uniform(-1, 1))) for t in range(1, 9)}
    specs = []
    for (a, b), cnt in DEEP.items():
        for k in range(cnt):
            t = (P, G, U)[k % 3] if cnt > 1 else P
            specs.append(pool_spec(rng, t, a, b, nu, misprice=None if rng.random() < 0.4 else
                                   float(np.exp(rng.uniform(-0.001, 0.001)))))
    specs[0] = pool_spec(rng, U, 1, 2, nu, depth=50.0)  # the single pool of {1, 2}: a UniV3 ladder
    ds = PoolSet(cr, 8, specs, seed=72)
    ds.retired -= {(U, 0)}
    ds.p.set_active(U, 0, [True])
    yield ds
    ds.p.close()


def deep_rows(rng, ds, objs, per_pair=6):
    tin, tout, kind, amount = [], [], [], []
    for (a, b) in DEEP:
        for k in range(per_pair):
            j, i = (a, b) if k % 2 else (b, a)
            kd = (k // 2) % 2
            row = ds.row(objs, j, i)
            if kd == oc.EXACT_OUT:
                d = float(row.reach_out())
            else:
                d = sum(float(p.R[p.Ai.index(j)]) if p.kind != "univ3" else 1.0 for p in row.direct if p.active)
            f = 10.0 ** rng.uniform(-9, np.log10(0.99))
            tin.append(j), tout.append(i), kind.append(kd), amount.append(d * f)
    return (np.array(tin, np.int64), np.array(tout, np.int64), np.array(kind, np.uint8), np.array(amount))


def geomean_overflow(row, out):
    """The reference's GeometricMeanTwoCoin closed form (geom_arb_δ) overflows to an infinite tender
    where γ·m·η·R₁·R₂^η exceeds DBL_MAX, though the optimum of the trading set is finite; the kernels
    keep parity with it, so such a row reports paid = inf.  True when every non-finite leg is such a
    pool's."""
    bad = [n for n in range(len(row.pools)) if not np.all(np.isfinite(out["D"][n]))]
    if not bad:
        return False
    s = float(out["price"])
    for n in bad:
        p = row.pools[n]
        assert p.kind == "geomean", n
        a = int(np.flatnonzero(~np.isfinite(out["D"][n]))[0])
        m = (1.0 / s) if p.Ai[a] == row.j else s  # ν_out / ν_in of that direction
        eta = p.w[a] / p.w[1 - a]
        with np.errstate(over="ignore"):
            base = p.g * m * eta * p.R[1 - a] * p.R[a] ** eta
        assert not np.isfinite(base), n
    return True


def certify_all(ds, objs, dev, tin, tout, kind, amount, hub_off=None, hubs=None, nested_rows=(), limit=None,
                overflow=None):
    routed = hub_off is not None
    paid, got, price, st = dev[:4]
    o, D, L = dev[6] if routed else dev[4]
    seen = {}
    for r in range(len(tin)):
        hr = [int(h) for h in hubs[hub_off[r]:hub_off[r + 1]]] if routed else []
        row = ds.row(objs, int(tin[r]), int(tout[r]), hr)
        g = slice(int(hub_off[r]), int(hub_off[r + 1])) if routed else slice(0, 0)
        out = dict(paid=paid[r], received=got[r], price=price[r], status=st[r],
                   hub_price=dev[4][g] if routed else [], hub_surplus=dev[5][g] if routed else [],
                   D=D[o[r]:o[r + 1]], L=L[o[r]:o[r + 1]])
        if overflow is not None and geomean_overflow(row, out):
            overflow.append(r)
            continue
        c = oc.certify_row(row, kind[r], amount[r], out, nested=r in nested_rows,
                           limit=None if limit is None else limit[r])
        if c["gap"] is not None and len(c["kinds"]) == 1:
            k = next(iter(c["kinds"]))
            seen[k] = max(seen.get(k, -np.inf), c["gap"] / c["allowance"])
    return seen


def test_deep_pairs_quote(deep):
    rng = np.random.default_rng(3)
    objs = deep.cert_pools(deep.p)
    tin, tout, kind, amount = deep_rows(rng, deep, objs)
    dev = deep.p.quote_split_orders(tin, tout, kind, amount, legs=True)
    assert np.sum(dev[3] == oc.FILLED) >= len(tin) - 4
    seen = certify_all(deep, objs, dev, tin, tout, kind, amount)
    print("largest gap / allowance per type:", seen)
    # the same rows as routed orders without hubs: the same certificate holds
    none = np.zeros(len(tin) + 1, np.int64)
    dev2 = deep.p.quote_routed_orders(tin, tout, kind, amount, none, [], legs=True)
    assert all(np.array_equal(x, y) for x, y in zip(dev[:4], dev2[:4]))


def test_depth_edges(deep):
    """Exact-out just below and just above the depth of the pair; exact-in past a capped ladder."""
    objs = deep.cert_pools(deep.p)
    tin, tout, kind, amount = [], [], [], []
    for (a, b) in [(1, 2), (1, 3), (2, 4), (5, 6)]:
        for j, i in ((a, b), (b, a)):
            y = float(deep.row(objs, j, i).reach_out())
            for f in (1 - 1e-11, 1 - 1e-9, 1 + 1e-9):
                tin.append(j), tout.append(i), kind.append(1), amount.append(y * f)
    for j, i in ((1, 2), (2, 1)):
        x = float(deep.row(objs, j, i).reach_in())
        if np.isfinite(x):
            for f in (0.5, 1 - 1e-9, 1 + 1e-9):
                tin.append(j), tout.append(i), kind.append(0), amount.append(x * f)
    tin, tout, kind, amount = (np.array(tin, np.int64), np.array(tout, np.int64), np.array(kind, np.uint8),
                               np.array(amount))
    dev = deep.p.quote_split_orders(tin, tout, kind, amount, legs=True)
    assert oc.UNREACHABLE in dev[3].tolist() and oc.FILLED in dev[3].tolist()
    over = []
    certify_all(deep, objs, dev, tin, tout, kind, amount, overflow=over)
    assert all(dev[0][r] == np.inf and dev[3][r] == oc.FILLED for r in over)
    assert len(over) < len(tin) // 2


def test_deep_pairs_execute_batch(deep):
    """Several rows per deep pair in one batch: each filled row certified on the state it saw, and the
    batch equal bit for bit to the rows one call at a time."""
    rng = np.random.default_rng(5)
    objs = deep.cert_pools(deep.p)
    tin, tout, kind, amount = deep_rows(rng, deep, objs, per_pair=4)
    sel = [r for r in range(len(tin)) if {int(tin[r]), int(tout[r])} in ({1, 3}, {2, 4}, {3, 4}, {5, 6})]
    tin, tout, kind, amount = tin[sel], tout[sel], kind[sel], amount[sel] * 0.1
    batch = deep.fresh()
    out = batch.execute_split_orders(tin, tout, kind, amount, legs=True)
    one = deep.fresh()
    filled = 0
    for r in range(len(tin)):
        objs = deep.cert_pools(one)
        x = one.execute_split_orders(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], legs=True)
        assert [v[0] for v in x[:4]] == [out[k][r] for k in range(4)], r
        o = out[4][0]
        assert np.array_equal(x[4][1], out[4][1][o[r]:o[r + 1]]) and np.array_equal(x[4][2], out[4][2][o[r]:o[r + 1]])
        certify_all(deep, objs, x, tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1])
        filled += int(x[3][0] == oc.FILLED)
    assert filled >= len(tin) - 2
    assert same_state(deep.state(batch), deep.state(one))
    batch.close()
    one.close()


# ---- full hub sets ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hubset(cr):
    rng = np.random.default_rng(81)
    nu = {t: float(np.exp(rng.uniform(-1, 1))) for t in range(1, 11)}
    specs = []
    add = lambda cnt, a, b, **kw: specs.extend(pool_spec(rng, (P, G, U)[int(rng.integers(0, 3))], a, b, nu, **kw)
                                               for _ in range(cnt))
    add(4, J, I, depth=200.0)
    add(20, J, 3, depth=100.0)              # hub 3: {j, h} 20 pools, {h, i} 25: list b starts mid-lane
    add(25, 3, I, depth=100.0)
    add(3, J2, 3, depth=100.0)
    add(2, J, 4, depth=300.0)               # hub 4: {j, h} only
    add(2, 5, I, depth=300.0)               # hub 5: {h, i} only
    # hub 6 far better than the direct pools (h cheap on {j, h}, dear on {h, i}); hub 7 useless
    for h, f, d in ((6, 1.1, 5000.0), (7, 1 / 1.3, 10.0)):
        for a, b, cnt, v in ((J, h, 3, nu[h] / f), (h, I, 3, nu[h] * f), (J2, h, 2, nu[h] / f)):
            specs.extend(pool_spec(rng, (P, G, U)[k % 3], a, b, {**nu, h: v}, depth=d, misprice=1.0)
                         for k in range(cnt))
    for h in (8, 9):
        add(int(rng.integers(1, 3)), J, h, depth=150.0)
        add(int(rng.integers(1, 3)), h, I, depth=150.0)
        add(1, J2, h, depth=150.0)
    hs = PoolSet(cr, 10, specs, seed=82, retire=0.04)
    yield hs
    hs.p.close()


def hub_rows(rng, hs, objs, q):
    tin = np.where(np.arange(q) % 3 == 2, J2, J).astype(np.int64)
    tout = np.full(q, I, np.int64)
    per = [list(HUBS) if r % 4 != 3 else list(rng.permutation(HUBS)[:int(rng.integers(1, 7))]) for r in range(q)]
    hub_off = np.concatenate([[0], np.cumsum([len(h) for h in per])]).astype(np.int64)
    hubs = np.array([h for x in per for h in x], dtype=np.int64)
    kind = (np.arange(q) // 2 % 2).astype(np.uint8)
    amount = np.zeros(q)
    for r in range(q):
        row = hs.row(objs, int(tin[r]), I, per[r])
        y = float(row.reach_out())
        amount[r] = y * 10.0 ** rng.uniform(-9, np.log10(0.99)) if kind[r] else 100.0 * 10.0 ** rng.uniform(-9, 0.5)
    return tin, tout, kind, amount, hub_off, hubs


def test_full_hub_sets_quote(hubset):
    rng = np.random.default_rng(7)
    objs = hubset.cert_pools(hubset.p)
    tin, tout, kind, amount, hub_off, hubs = hub_rows(rng, hubset, objs, 12)
    dev = hubset.p.quote_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    assert np.sum(dev[3] == oc.FILLED) >= 10
    assert max(np.diff(hub_off)) == 7
    # the nested 50-digit re-solves of every t_h on the first rows only (the others fix t_h*)
    seen = certify_all(hubset, objs, dev, tin, tout, kind, amount, hub_off, hubs, nested_rows=(0, 1, 2, 3))
    print("largest gap / allowance per type:", seen)
    # the routes beat the pair alone where there is one
    sp = hubset.p.quote_split_orders(tin, tout, kind, amount)
    for r in np.flatnonzero((dev[3] == oc.FILLED) & (sp[3] == oc.FILLED) & (kind == oc.EXACT_IN)):
        assert dev[1][r] > sp[1][r], r


def test_full_hub_sets_execute(hubset):
    rng = np.random.default_rng(9)
    objs = hubset.cert_pools(hubset.p)
    tin, tout, kind, amount, hub_off, hubs = hub_rows(rng, hubset, objs, 6)
    batch = hubset.fresh()
    out = batch.execute_routed_orders(tin, tout, kind, amount, hub_off, hubs, legs=True)
    one = hubset.fresh()
    for r in range(len(tin)):
        objs = hubset.cert_pools(one)
        h = hubs[hub_off[r]:hub_off[r + 1]]
        x = one.execute_routed_orders(tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], [0, len(h)], h,
                                      legs=True)
        assert [v[0] for v in x[:4]] == [out[k][r] for k in range(4)], r
        o = out[6][0]
        assert np.array_equal(x[6][1], out[6][1][o[r]:o[r + 1]]) and np.array_equal(x[6][2], out[6][2][o[r]:o[r + 1]])
        certify_all(hubset, objs, x, tin[r:r + 1], tout[r:r + 1], kind[r:r + 1], amount[r:r + 1], [0, len(h)], h)
    assert same_state(hubset.state(batch), hubset.state(one))
    batch.close()
    one.close()
