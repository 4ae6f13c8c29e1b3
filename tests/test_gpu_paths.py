"""cfmm_quote_paths / cfmm_execute_paths (include/cfmm_b200.h) on the device.

One context holds all three pool types, each with a main set and appended pools (a tail), some
pools retired; the ProductTwoCoin main set is laid out with orient_by_degree, so some of its pools
are stored with their tokens exchanged.  Paths are random walks of 1-8 hops on the token graph.
Quotes are checked bit for bit against cfmm_quote_swaps / cfmm_quote_swaps_exact_out composed hop by
hop on the same context, and against the host mirror (path_oracle.py) for ProductTwoCoin and UniV3
hops.  Executes are checked against a fresh context that replays path by path with the existing
entry points (quote, decide, one cfmm_execute_swaps per hop), and against the mirror."""
import numpy as np
import pytest

import path_oracle as po
import swap_order_oracle as oo
from swap_oracle import current_tick
from test_gpu_parity import check_psi, make_pools
from test_gpu_swap_orders import univ3_host_pools
from test_gpu_swaps import product_set

pytestmark = pytest.mark.gpu

P, G, U = 0, 1, 2
APPEND = ("append_product", "append_geomean", "append_univ3")


class Mixed:
    """All three types on one context (main + tail each, some retired) and the host's copy of them."""

    def __init__(self, cr, synth, seed=11, m=(1500, 1200, 1000), mt=(300, 250, 200), n=48):
        self._cr, self.n, self.mm, self.mt = cr, n, m, mt
        R, g, A = product_set(m[P] + mt[P], n, seed=seed, wide=False)
        Rg, gg, Ag, wg = synth.geomean_pools(m[G] + mt[G], n, seed=seed + 1)
        cu = synth.univ3_pools(m[U], n, seed=seed + 2, ragged=True)
        cut = synth.univ3_pools(mt[U], n, seed=seed + 3, ragged=True)
        self.main = {P: (R[:m[P]], g[:m[P]], A[:m[P]]), G: (Rg[:m[G]], gg[:m[G]], Ag[:m[G]], wg[:m[G]]), U: cu}
        self.tail = {P: (R[m[P]:], g[m[P]:], A[m[P]:]), G: (Rg[m[G]:], gg[m[G]:], Ag[m[G]:], wg[m[G]:]), U: cut}
        self.Ai = {P: A, G: Ag, U: np.concatenate([cu[2], cut[2]])}
        self.g = {P: g, G: gg, U: np.concatenate([cu[1], cut[1]])}
        self.w = wg
        self.m = {t: m[t] + mt[t] for t in (P, G, U)}
        self.retired = {(t, i) for t in (P, G, U) for i in list(range(40, 55)) + [m[t] + 5, m[t] + 6]}
        self.p = self.fresh()
        self.by_token = {}
        for t in (P, G, U):
            for i, (a, b) in enumerate(self.Ai[t]):
                self.by_token.setdefault(int(a), []).append((t, i))
                self.by_token.setdefault(int(b), []).append((t, i))

    def fresh(self):
        p = make_pools(self._cr, self.n, product=self.main[P], geomean=self.main[G], univ3=self.main[U],
                       pre={"orient_by_degree": 1})
        for t in (P, G, U):
            getattr(p, APPEND[t])(*self.tail[t])
            act = np.ones(self.m[t], bool)
            act[[i for (s, i) in self.retired if s == t]] = False
            p.set_active(t, 0, act)
        return p

    def host_pools(self, p=None):
        """The mirror's pool objects at the device's state, keyed (type, index)."""
        p = p or self.p
        out = {}
        st, _ = p.pool_state(P)
        for i in range(self.m[P]):
            out[(P, i)] = oo.ProductPool(st[i], self.g[P][i])
        st, _ = p.pool_state(G)
        for i in range(self.m[G]):
            out[(G, i)] = oo.GeoMeanPool(st[i], self.g[G][i], self.w[i])
        for i, h in enumerate(univ3_host_pools(p, self.g[U])):
            out[(U, i)] = h
        return out

    def state(self, p):
        return [p.pool_state(t)[0].copy() for t in (P, G, U)] + list(p.univ3_ticks())


def same_state(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


class Batch:
    """A CSR batch of paths: hop keys, sides, kinds, amounts."""

    def __init__(self, mx, paths, starts, kind, amount):
        self.paths, self.starts = paths, np.asarray(starts, np.int64)
        self.off = np.concatenate([[0], np.cumsum([len(x) for x in paths])]).astype(np.int64)
        self.keys = [k for x in paths for k in x]
        self.ht = np.array([k[0] for k in self.keys], np.int32)
        self.hp = np.array([k[1] for k in self.keys], np.int64)
        self.tok1 = np.zeros(len(self.keys), bool)
        for j, x in enumerate(paths):
            sides = po.hop_sides([mx.Ai[t][i] for t, i in x], starts[j])
            assert sides is not None
            self.tok1[self.off[j]:self.off[j + 1]] = sides
        self.kind = np.asarray(kind, np.uint8)
        self.amount = np.asarray(amount, float)
        self.q = len(paths)

    def args(self):
        return self.off, self.ht, self.hp, self.starts, self.kind, self.amount

    def sub(self, mx, js):
        return Batch(mx, [self.paths[j] for j in js], self.starts[js], self.kind[js], self.amount[js])


def walks(mx, rng, q, max_hops=8, types=(P, G, U)):
    paths, starts = [], []
    while len(paths) < q:
        t0 = int(rng.choice(sorted(mx.by_token)))
        t, path = t0, []
        for _ in range(int(rng.integers(1, max_hops + 1))):
            nxt = [k for k in mx.by_token.get(t, []) if k[0] in types and k not in path]
            if not nxt:
                break
            k = nxt[int(rng.integers(0, len(nxt)))]
            path.append(k)
            a, b = (int(v) for v in mx.Ai[k[0]][k[1]])
            t = b if t == a else a
        if path:
            paths.append(path)
            starts.append(t0)
    return paths, starts


def random_batch(mx, rng, q, types=(P, G, U), max_hops=8):
    paths, starts = walks(mx, rng, q, max_hops, types)
    kind = rng.integers(0, 2, size=q)
    amount = np.where(kind == 0, 10.0 ** rng.uniform(-3, 1.5, size=q), 10.0 ** rng.uniform(-4, 0.5, size=q))
    amount[::23] = 0.0
    return Batch(mx, paths, starts, kind, amount)


# ---- composing the existing entry points hop by hop -------------------------------------------
def quote_rows(p, ht, hp, tok1, v, exact_out):
    """Per row, cfmm_quote_swaps (f of the tender v) or cfmm_quote_swaps_exact_out (x* for the want v)."""
    res = np.zeros(len(v))
    for t in (P, G, U):
        m = ht == t
        if not m.any():
            continue
        rows = np.zeros((m.sum(), 2))
        t1 = tok1[m]
        if exact_out:
            rows[t1, 1], rows[~t1, 0] = v[m][t1], v[m][~t1]
            out = p.quote_swaps_exact_out(t, hp[m], rows)
            res[m] = np.where(t1, out[:, 0], out[:, 1])
        else:
            rows[t1, 0], rows[~t1, 1] = v[m][t1], v[m][~t1]
            out = p.quote_swaps(t, hp[m], rows)
            res[m] = np.where(t1, out[:, 1], out[:, 0])
    return res


def compose(p, b, retired):
    """cfmm_quote_paths composed from the single-pool quotes, hop by hop."""
    x, lam = np.zeros(len(b.keys)), np.zeros(len(b.keys))
    st = np.zeros(b.q, np.uint8)
    nh = np.diff(b.off)
    for j in range(b.q):
        if any(k in retired for k in b.paths[j]):
            st[j] = po.RETIRED
    cur = b.amount.copy()
    for d in range(8):
        js = np.flatnonzero((nh > d) & (st == 0))
        if not len(js):
            break
        fwd = b.kind[js] == 0
        h = np.where(fwd, b.off[js] + d, b.off[js + 1] - 1 - d)
        xs = cur[js].copy()
        out = js[~fwd]
        if len(out):
            hh = h[~fwd]
            xo = quote_rows(p, b.ht[hh], b.hp[hh], b.tok1[hh], cur[out], True)
            xs[~fwd] = xo
            st[out[np.isinf(xo)]] = po.UNREACHABLE
        ok = np.isfinite(xs)
        hk = h[ok]
        lk = quote_rows(p, b.ht[hk], b.hp[hk], b.tok1[hk], xs[ok], False)
        x[hk], lam[hk] = xs[ok], lk
        jk = js[ok]
        cur[jk] = np.where(b.kind[jk] == 0, np.where(lk > 0, lk, 0.0), xs[ok])
    for j in np.flatnonzero(st != 0):
        x[b.off[j]:b.off[j + 1]] = lam[b.off[j]:b.off[j + 1]] = 0.0
    return x, lam, st


def replay_with_swaps(p, b, limit, retired):
    """cfmm_execute_paths by the existing entry points: per path, quote, decide, then one
    cfmm_execute_swaps per hop."""
    x, lam = np.zeros(len(b.keys)), np.zeros(len(b.keys))
    st = np.zeros(b.q, np.uint8)
    for j in range(b.q):
        one = _one(b, j)
        xj, lj, sj = compose(p, one, retired)
        s = sj[0]
        if s == 0:
            lim = limit[j] if limit is not None else (np.inf if b.kind[j] else 0.0)
            if (b.kind[j] == 0 and lj[-1] < lim) or (b.kind[j] == 1 and xj[0] > lim):
                s = po.LIMIT
        st[j] = s
        if s != 0:
            continue
        for h in range(len(xj)):
            if xj[h] > 0:
                t, i = one.keys[h]
                row = [[xj[h], 0.0]] if one.tok1[h] else [[0.0, xj[h]]]
                r = p.execute_swaps(t, [i], row)[0]
                lj[h] = r[1] if one.tok1[h] else r[0]
        x[b.off[j]:b.off[j + 1]], lam[b.off[j]:b.off[j + 1]] = xj, lj
    return x, lam, st


def _one(b, j):
    o = Batch.__new__(Batch)
    s = slice(b.off[j], b.off[j + 1])
    o.paths, o.starts = [b.paths[j]], b.starts[j:j + 1]
    o.off = np.array([0, b.off[j + 1] - b.off[j]], np.int64)
    o.keys, o.ht, o.hp, o.tok1 = b.keys[s], b.ht[s], b.hp[s], b.tok1[s]
    o.kind, o.amount, o.q = b.kind[j:j + 1], b.amount[j:j + 1], 1
    return o


def no_geomean(b):
    return [j for j in range(b.q) if all(k[0] != G for k in b.paths[j])]


def limits_for(b, x, lam, rng):
    """Limits around each path's own quote, so that some fill and some revert."""
    f = 10.0 ** rng.uniform(-0.02, 0.02, size=b.q)
    paid, got = x[b.off[:-1]], lam[b.off[1:] - 1]
    lim = np.where(b.kind == 1, np.where(paid > 0, paid * f, 1.0), np.maximum(got, 0.0) * f)
    lim[::13] = np.where(b.kind[::13] == 1, np.inf, 0.0)
    return lim


@pytest.fixture(scope="module")
def mixed(cr, synth):
    mx = Mixed(cr, synth)
    yield mx
    mx.p.close()


# ---- 1. quotes -------------------------------------------------------------------------------
def test_quotes(mixed):
    mx, p = mixed, mixed.p
    assert p.pool_set_info(P)["tail"] > 0
    rng = np.random.default_rng(1)
    b = random_batch(mx, rng, 3000)
    assert set(np.diff(b.off)) == set(range(1, 9))
    s0 = mx.state(p)
    x, lam, st = p.quote_paths(*b.args())
    assert same_state(s0, mx.state(p))
    counts = np.bincount(st, minlength=4)
    assert counts[0] > 1000 and counts[2] > 20 and counts[3] > 20, counts
    x2, lam2, st2 = compose(p, b, mx.retired)
    assert np.array_equal(st, st2), np.flatnonzero(st != st2)[:5]
    assert np.array_equal(x, x2) and np.array_equal(lam, lam2)
    # exact-out: every hop receives at least what the next one needs
    for j in np.flatnonzero((st == 0) & (b.kind == 1))[:300]:
        s = slice(b.off[j], b.off[j + 1])
        need = np.concatenate([x[s][1:], [b.amount[j]]])
        assert np.all(lam[s] >= need)
    # the mirror, bit for bit, on the paths without GeometricMean hops
    js = no_geomean(b)
    sb = b.sub(mx, js)
    hx, hl, hs = po.quote_paths(mx.host_pools(), sb.off, sb.keys, sb.tok1, sb.kind, sb.amount, mx.retired)
    xs, ls, ss = p.quote_paths(*sb.args())
    assert np.array_equal(ss, hs) and np.array_equal(xs, hx) and np.array_equal(ls, hl)


# ---- 2. one-hop paths are order rows ---------------------------------------------------------
def test_one_hop_paths_are_order_rows(cr, synth):
    mx = Mixed(cr, synth, seed=21)
    a, b = mx.p, mx.fresh()
    rng = np.random.default_rng(2)
    for t in (P, G, U):
        q = 1500
        idx = rng.integers(0, mx.m[t], size=q)
        idx[: q // 2] = rng.integers(0, 60, size=q // 2)  # repeats, retired pools among them
        tok1 = rng.integers(0, 2, size=q).astype(bool)
        starts = np.where(tok1, mx.Ai[t][idx, 0], mx.Ai[t][idx, 1])
        kind = rng.integers(0, 2, size=q).astype(np.uint8)
        amount = 10.0 ** rng.uniform(-4, 1, size=q)
        bt = Batch(mx, [[(t, int(i))] for i in idx], starts, kind, amount)
        x0, l0, _ = a.quote_paths(*bt.args())
        lim = limits_for(bt, x0, l0, rng)
        x, lam, st = a.execute_paths(*bt.args(), lim)
        rows = np.zeros((q, 2))
        side = np.where(tok1, 0, 1)  # the tendered side
        rows[np.arange(q), np.where(kind == 0, side, 1 - side)] = amount
        paid, rec, st2 = b.execute_swap_orders(t, idx, kind, rows, lim)
        assert np.array_equal(st, st2) and {0, 1, 3} <= set(st.tolist())
        assert np.array_equal(x, paid[np.arange(q), side]) and np.array_equal(lam, rec[np.arange(q), 1 - side])
        assert same_state(mx.state(a), mx.state(b))
    a.close()
    b.close()


# ---- 3. execute --------------------------------------------------------------------------------
def test_execute_against_swaps_and_mirror(cr, synth):
    mx = Mixed(cr, synth, seed=31)
    a, b = mx.p, mx.fresh()
    rng = np.random.default_rng(3)
    bt = random_batch(mx, rng, 600)
    x0, l0, _ = a.quote_paths(*bt.args())
    lim = limits_for(bt, x0, l0, rng)
    x, lam, st = a.execute_paths(*bt.args(), lim)
    counts = np.bincount(st, minlength=4)
    assert counts[0] > 100 and counts[1] > 30 and counts[3] > 5, counts
    x2, l2, s2 = replay_with_swaps(b, bt, lim, mx.retired)
    assert np.array_equal(st, s2), np.flatnonzero(st != s2)[:5]
    assert np.array_equal(x, x2) and np.array_equal(lam, l2)
    assert same_state(mx.state(a), mx.state(b))
    b.close()
    # the mirror, on a batch without GeometricMean hops
    hp = mx.host_pools()
    bt = random_batch(mx, rng, 600, types=(P, U))
    x0, l0, _ = a.quote_paths(*bt.args())
    lim = limits_for(bt, x0, l0, rng)
    x, lam, st = a.execute_paths(*bt.args(), lim)
    hx, hl, hs = po.replay_paths(hp, bt.off, bt.keys, bt.tok1, bt.kind, bt.amount, lim, mx.retired)
    assert np.array_equal(st, hs) and np.array_equal(x, hx) and np.array_equal(lam, hl)
    st_p, _ = a.pool_state(P)
    st_u, _ = a.pool_state(U)
    live = [k for k in hp if k not in mx.retired]
    assert all((st_p[i] == hp[(t, i)].R).all() for t, i in live if t == P)
    assert all(st_u[i] == hp[(t, i)].price for t, i in live if t == U)
    a.close()


# ---- 4. scheduling ----------------------------------------------------------------------------
def hub_batch(mx, rng, hub, q):
    """q two-hop paths through the pool hub, alternating its direction, each continuing into a
    different ProductTwoCoin or UniV3 pool (one-hop paths where none is left)."""
    a, b = (int(v) for v in mx.Ai[hub[0]][hub[1]])
    paths, starts = [], []
    for j in range(q):
        t0, t1 = (a, b) if j % 2 == 0 else (b, a)
        nxt = [k for k in mx.by_token[t1] if k != hub and k[0] != G and k not in mx.retired]
        paths.append([hub, nxt[int(rng.integers(0, len(nxt)))]] if j % 3 else [hub])
        starts.append(t0)
    kind = rng.integers(0, 2, size=q)
    amount = np.where(kind == 0, 10.0 ** rng.uniform(-1, 1.5, size=q), 10.0 ** rng.uniform(-2, 0.5, size=q))
    return Batch(mx, paths, starts, kind, amount)


def test_scheduling(cr, synth):
    mx = Mixed(cr, synth, seed=41)
    p = mx.p
    rng = np.random.default_rng(4)
    # the hub: a UniV3 pool with many ticks, crossed 2000 times in one call (2000 levels)
    off = p.univ3_ticks(ladders=False)[0]
    hub = (U, int(np.argmax(np.diff(off)[:100] * np.array([(U, i) not in mx.retired for i in range(100)]))))
    assert np.diff(off)[hub[1]] >= 8
    hp = mx.host_pools()
    bt = hub_batch(mx, rng, hub, 2000)
    l0 = p.launch_count
    x, lam, st = p.execute_paths(*bt.args())
    assert p.launch_count - l0 >= 2000
    hx, hl, hs = po.replay_paths(hp, bt.off, bt.keys, bt.tok1, bt.kind, bt.amount, None, mx.retired)
    assert np.array_equal(st, hs) and np.array_equal(x, hx) and np.array_equal(lam, hl)
    assert (st == 0).sum() > 1000
    # the hub's walks crossed tick boundaries: its current tick changed between levels of the call
    h2 = mx.host_pools()
    ticks = []
    for j in range(200):
        one = _one(bt, j)
        po.replay_paths(h2, one.off, one.keys, one.tok1, one.kind, one.amount)
        ticks.append(current_tick(h2[hub].lt, h2[hub].price))
    assert np.count_nonzero(np.diff(ticks)) >= 10
    state, _ = p.pool_state(U)
    assert state[hub[1]] == hp[hub].price
    # wide independent levels: every pool at most once in the batch (one level)
    used, paths, starts = set(), [], []
    for path, s in zip(*walks(mx, rng, 4000, 4, (P, U))):
        if not used & set(path):
            used |= set(path)
            paths.append(path)
            starts.append(s)
    assert len(paths) > 300
    wide = Batch(mx, paths, starts, rng.integers(0, 2, size=len(paths)), 10.0 ** rng.uniform(-3, 0.5, size=len(paths)))
    hp = mx.host_pools()
    l0 = p.launch_count
    x, lam, st = p.execute_paths(*wide.args())
    assert p.launch_count - l0 < 30
    hx, hl, hs = po.replay_paths(hp, wide.off, wide.keys, wide.tok1, wide.kind, wide.amount, None, mx.retired)
    assert np.array_equal(st, hs) and np.array_equal(x, hx) and np.array_equal(lam, hl)
    # mixes: hub paths interleaved with random walks, against the replay on a fresh context
    mix_paths = hub_batch(mx, rng, (P, int(rng.integers(60, 200))), 150)
    rb = random_batch(mx, rng, 300)
    order = rng.permutation(450)
    allp = mix_paths.paths + rb.paths
    mb = Batch(mx, [allp[k] for k in order], np.concatenate([mix_paths.starts, rb.starts])[order],
               np.concatenate([mix_paths.kind, rb.kind])[order], np.concatenate([mix_paths.amount, rb.amount])[order])
    a, b2 = mx.fresh(), mx.fresh()
    x, lam, st = a.execute_paths(*mb.args())
    x2, l2, s2 = replay_with_swaps(b2, mb, None, mx.retired)
    assert np.array_equal(st, s2) and np.array_equal(x, x2) and np.array_equal(lam, l2)
    assert same_state(mx.state(a), mx.state(b2))
    a.close()
    b2.close()
    p.close()


# ---- 5. atomicity ------------------------------------------------------------------------------
def test_limits_and_atomic_revert(cr, synth):
    mx = Mixed(cr, synth, seed=51)
    p = mx.p
    rng = np.random.default_rng(5)
    # a 3-hop path crossing all three types, avoiding retired pools, that fills both ways
    while True:
        paths, starts = walks(mx, rng, 1, 3)
        if len(paths[0]) == 3 and len({k[0] for k in paths[0]}) == 3 and not mx.retired & set(paths[0]):
            both = Batch(mx, paths * 2, starts * 2, [0, 1], [0.5, 0.05])
            if not p.quote_paths(*both.args())[2].any():
                break
    for kind, amt in ((0, 0.5), (1, 0.05)):
        bt = Batch(mx, paths * 3, starts * 3, [kind] * 3, [amt] * 3)
        x, lam, st = p.quote_paths(*bt.args())
        assert st.tolist() == [0, 0, 0]
        v = x[0] if kind == 1 else lam[2]
        beyond = np.nextafter(v, 0.0 if kind == 1 else np.inf)
        s0 = mx.state(p)
        _, _, st = p.execute_paths(*bt.sub(mx, [0]).args(), [beyond])
        assert st.tolist() == [po.LIMIT]
        assert same_state(s0, mx.state(p))  # every hop reverted
        # in one batch: the reverting path leaves the state to the next, which fills at its exact limit
        x2, lam2, st = p.execute_paths(*bt.sub(mx, [0, 1]).args(), [beyond, v])
        assert st.tolist() == [po.LIMIT, po.FILLED]
        assert not x2[:3].any() and np.array_equal(x2[3:], x[:3]) and np.array_equal(lam2[3:], lam[:3])
        assert not same_state(s0, mx.state(p))
    p.close()


# ---- 6. rejections ----------------------------------------------------------------------------
def test_rejections_change_nothing(cr, synth):
    mx = Mixed(cr, synth, seed=61, m=(300, 300, 300), mt=(50, 50, 50), n=20)
    p = mx.p
    rng = np.random.default_rng(6)
    good = random_batch(mx, rng, 20, max_hops=4)
    s0 = mx.state(p)

    def args(**kw):
        d = dict(zip(("off", "ht", "hp", "tok", "kind", "amount"), [np.array(a, copy=True) for a in good.args()]))
        d["limit"] = None
        d.update(kw)
        return d

    def rejected(d, code=-1):
        for fn in ("quote_paths", "execute_paths"):
            a = (d["off"], d["ht"], d["hp"], d["tok"], d["kind"], d["amount"])
            with pytest.raises(cr.CFMMError) as e:
                getattr(p, fn)(*a) if fn == "quote_paths" else p.execute_paths(*a, d["limit"])
            assert e.value.code == code, (fn, e.value)
        assert same_state(s0, mx.state(p))
        return e.value.message

    base = args()
    H = int(base["off"][-1])
    off = base["off"].copy(); off[0] = 1; off[-1] += 1
    rejected(args(off=off, ht=np.zeros(H + 1, np.int32), hp=np.zeros(H + 1)))        # hop_off[0] != 0
    off = base["off"].copy(); off[3] = off[2]
    rejected(args(off=off))                                                           # an empty path
    off = np.array([0, 9]); rejected(args(off=off, ht=np.zeros(9, np.int32), hp=np.arange(9), tok=[1], kind=[0],
                                          amount=[1.0]))                              # 9 hops
    ht = base["ht"].copy(); ht[4] = 3; rejected(args(ht=ht))                         # bad type
    hp = base["hp"].copy(); hp[2] = 10 ** 6; rejected(args(hp=hp))                   # pool out of range
    rejected(args(off=np.array([0, 2]), ht=np.array([P, P], np.int32), hp=np.array([3, 3]), tok=[1], kind=[0],
                  amount=[1.0]))                                                      # same pool twice
    tok = base["tok"].copy(); tok[1] = mx.n + 1; rejected(args(tok=tok))              # token out of range
    kind = base["kind"].copy(); kind[5] = 2; rejected(args(kind=kind))
    for v in (np.nan, np.inf, -1.0):
        amount = base["amount"].copy(); amount[3] = v; rejected(args(amount=amount))
    for v, k in ((np.nan, 1), (-1.0, 1), (np.inf, 0)):
        kind = base["kind"].copy(); kind[0] = k
        lim = np.ones(good.q); lim[0] = v
        with pytest.raises(cr.CFMMError) as e:
            p.execute_paths(base["off"], base["ht"], base["hp"], base["tok"], kind, base["amount"], lim)
        assert e.value.code == -1
    # the device finds a token mismatch on the last hop of the last path
    j = good.q - 1
    last = int(base["off"][-1]) - 1
    t_in = mx.Ai[good.ht[last]][good.hp[last]]
    bad = next(k for k in range(mx.m[P]) if (P, k) not in good.paths[j]
               and not set(mx.Ai[P][k].tolist()) & set(t_in.tolist()))
    ht, hp = base["ht"].copy(), base["hp"].copy()
    ht[last], hp[last] = P, bad
    msg = rejected(args(ht=ht, hp=hp))
    assert f"path {j} hop {len(good.paths[j]) - 1}" in msg, msg
    # an exact-out path with an infinite limit is fine; q == 0 does nothing
    one = good.sub(mx, [0])
    p.execute_paths(one.off, one.ht, one.hp, one.starts, [1], [0.0], [np.inf])
    x, lam, st = p.execute_paths([0], [], [], [], [], [])
    assert x.shape == (0,) and st.shape == (0,)
    p.close()
    q = cr.DevicePools(mx.n)
    q.add_product(*mx.main[P])
    with pytest.raises(cr.CFMMError) as e:
        q.quote_paths([0, 1], [P], [0], [int(mx.Ai[P][0, 0])], [0], [1.0])
    assert e.value.code == -3
    with pytest.raises(cr.CFMMError) as e:
        q.execute_paths([0, 1], [P], [0], [int(mx.Ai[P][0, 0])], [0], [1.0])
    assert e.value.code == -3
    q.close()


# ---- 7. interaction with the rest --------------------------------------------------------------
def test_sweeps_after_paths(cr, oracle, synth):
    m = 20000
    R, g, A, v = synth.disjoint_product(m, seed=81, adversarial=False)
    n = 2 * m
    p = make_pools(cr, n, product=(R, g, A))
    for _ in range(3):  # the second call captures the sweep graph, the third replays it
        p.sweep(v)
    rng = np.random.default_rng(82)
    q = 6000
    pools = rng.integers(0, m, size=q)
    tok1 = rng.integers(0, 2, size=q).astype(bool)
    starts = np.where(tok1, A[pools, 0], A[pools, 1])
    amount = R[pools, np.where(tok1, 0, 1)] * 10.0 ** rng.uniform(-4, -0.5, size=q)
    off = np.arange(q + 1)
    _, _, st = p.execute_paths(off, np.zeros(q, np.int32), pools, starts, np.zeros(q, np.uint8), amount)
    assert (st == 0).all()
    state, _ = p.pool_state(P)
    assert not np.array_equal(state, R)
    psi, acc = p.sweep(v)  # the captured graph sees the new state
    f = make_pools(cr, n, product=(state, g, A))
    psi_f, acc_f = f.sweep(v)
    assert np.array_equal(psi, psi_f) and abs(acc - acc_f) <= 1e-12 * abs(acc_f)
    D, L = oracle.sweep_product(state, g, A, v)
    check_psi(oracle, A, D, L, v, n, psi, acc, R=state, g=g)
    f.close()
    p.close()


def rebuilt(cr, mx, p):
    """A context built afresh from p's read-back state, with the same pools retired."""
    st = {t: p.pool_state(t)[0] for t in (P, G, U)}
    off, lt, lq = p.univ3_ticks()
    q = make_pools(cr, mx.n, product=(st[P], mx.g[P], mx.Ai[P]), geomean=(st[G], mx.g[G], mx.Ai[G], mx.w),
                   univ3=(st[U], mx.g[U], mx.Ai[U], off, lt, lq))
    for t in (P, G, U):
        act = np.ones(mx.m[t], bool)
        act[[i for (s, i) in mx.retired if s == t]] = False
        q.set_active(t, 0, act)
    return q


def test_materialise_apply_compact_liquidity_after_paths(cr, synth):
    mx = Mixed(cr, synth, seed=71)
    p = mx.p
    rng = np.random.default_rng(7)
    v = synth.dual_prices(mx.n, "wide")
    p.sweep(v, materialize=True)
    bt = random_batch(mx, rng, 800)
    p.execute_paths(*bt.args())
    f = rebuilt(cr, mx, p)
    p.sweep(v, materialize=True)
    f.sweep(v, materialize=True)
    (D, L), (Df, Lf) = p.trades(), f.trades()
    # p holds the main sets first, then the appended pools; f holds every pool of a type together
    perm = np.concatenate([np.concatenate([np.arange(mx.mm[t]) + sum(mx.mm[:t]),
                                           np.arange(mx.mt[t]) + sum(mx.mm) + sum(mx.mt[:t])]) for t in (P, G, U)])
    D, L = D[perm], L[perm]
    mP, mG = mx.m[P], mx.m[P] + mx.m[G]
    assert np.array_equal(D[:mP], Df[:mP]) and np.array_equal(L[:mP], Lf[:mP])
    assert np.array_equal(D[mG:], Df[mG:]) and np.array_equal(L[mG:], Lf[mG:])
    assert np.allclose(D[mP:mG], Df[mP:mG], rtol=1e-9, atol=1e-12)
    p.apply_trades()
    f.apply_trades()
    for t in (P, U):
        assert np.array_equal(p.pool_state(t)[0], f.pool_state(t)[0])
    f.close()
    # paths after apply, then compact: the same state quotes the same paths
    bt = random_batch(mx, rng, 500)
    p.execute_paths(*bt.args())
    bt = random_batch(mx, rng, 500)
    before = p.quote_paths(*bt.args())
    p.compact()
    assert p.pool_set_info(U)["tail"] == 0
    after = p.quote_paths(*bt.args())
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    # liquidity changes, then paths against the mirror (the ladders read back)
    rows = rng.integers(0, mx.m[U], size=300)
    price, _ = p.pool_state(U)
    p.modify_univ3_liquidity(rows, price[rows] * rng.uniform(0.5, 0.99, size=300),
                             price[rows] * rng.uniform(1.01, 1.5, size=300), rng.uniform(1, 20, size=300))
    hp = mx.host_pools()
    bt = random_batch(mx, rng, 600, types=(P, U))
    x, lam, st = p.execute_paths(*bt.args())
    hx, hl, hs = po.replay_paths(hp, bt.off, bt.keys, bt.tok1, bt.kind, bt.amount, None, mx.retired)
    assert np.array_equal(st, hs) and np.array_equal(x, hx) and np.array_equal(lam, hl)
    # pools appended after all this take paths too
    Rn, gn, An = product_set(50, mx.n, seed=77, wide=False)
    p.append_product(Rn, gn, An)
    i0 = mx.m[P]
    x, lam, st = p.quote_paths([0, 1], [P], [i0], [int(An[0, 0])], [0], [1.0])
    assert st[0] == 0 and lam[0] == oo.ProductPool(Rn[0], gn[0]).f(1.0, True)
    p.close()


# ---- 8. the Router -----------------------------------------------------------------------------
def test_router_paths_device(cr):
    rng = np.random.default_rng(95)
    n = 8
    pools = []
    for k in range(30):
        a, b = rng.choice(np.arange(1, n + 1), size=2, replace=False)
        if k % 3 == 0:
            pools.append(cr.ProductTwoCoin(100 + 900 * rng.random(2), 0.997, [a, b]))
        elif k % 3 == 1:
            pools.append(cr.GeometricMeanTwoCoin(100 + 900 * rng.random(2), [0.3, 0.7], 0.997, [a, b]))
        else:
            c = float(np.exp(rng.uniform(-1, 1)))
            pools.append(cr.UniV3(c, c * 1.5 * np.cumprod([1.0, 0.8, 0.7, 0.6]), [100.0, 50.0, 0.0, 80.0], 0.997, [a, b]))
    r = cr.Router(cr.LinearNonnegative(np.ones(n)), pools, n)
    paths, starts = [], []
    for _ in range(40):
        t = int(rng.integers(1, n + 1))
        s, path = t, []
        for _ in range(int(rng.integers(1, 5))):
            nxt = [i for i, c in enumerate(pools) if t in (int(c.Ai[0]), int(c.Ai[1])) and i not in path]
            if not nxt:
                break
            i = int(rng.choice(nxt))
            path.append(i)
            t = int(pools[i].Ai[1]) if t == int(pools[i].Ai[0]) else int(pools[i].Ai[0])
        if path:
            paths.append(path)
            starts.append(s)
    q = len(paths)
    kinds = rng.integers(0, 2, size=q)
    amounts = 10.0 ** rng.uniform(-1, 1, size=q)
    paid, got, st, ht, hr = r.quote_paths(paths, starts, kinds, amounts)
    assert (st == 0).sum() > q // 2
    paid2, got2, st2, _, _ = r.execute_paths(paths[:1], starts[:1], kinds[:1], amounts[:1])
    assert paid2[0] == paid[0] and got2[0] == got[0] and st2[0] == st[0]
    paid, got, st, ht, hr = r.execute_paths(paths, starts, kinds, amounts)
    for i, c in enumerate(pools):
        t = (P, G, U)[i % 3]
        k = r._type_lists[t].index(i)
        state = r._pools.pool_state(t, k, 1)[0]
        if t == U:
            assert c.current_price == state[0]
        else:
            assert np.array_equal(c.R, state[0])
    r._pools.close()
