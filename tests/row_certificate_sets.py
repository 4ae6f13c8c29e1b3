"""Pool sets and row shapes that take the per-row order solver (subgraph_kernels.cuh, basket_kernels.cuh,
price_arb_kernels.cuh) to its widest and deepest rows, for test_gpu_row_certificates and
test_row_certificates_host.  No GPU code: a set builds its device context only when asked.

  * Wide: WIDE_N tokens.  Rows run between i and j over up to 256 B tokens, each joined to i, to j and
    to its neighbours.  Light rows (i = 1, j = 2) have one pool per pair, so a row's pool count is set
    exactly by how many B tokens it takes and how many of them are neighbours; deep rows (i = 3,
    j = 4) have two pools per pair and 38 more on {b, 3} for three of the b, so i holds more than 256
    of the row's pools, some b hold 33 to 64, and the row's padded pool count reaches 2048.  Every pool
    is priced at one reference ν with its misprice inside its fee, so the rows converge.
  * Deep/extreme: test_gpu_order_certificates' DEEP pairs (1, 31, 32, 33, 64, 65 and 200 pools), linked
    into one chain of eight tokens, over pool_spec's full ranges (reserves 1e-3 to 1e9, fees {1, 0.9995,
    0.997}, GeometricMean weights down to (0.05, 0.95), UniV3 ladders with zero-liquidity ticks and
    empty last ticks, pools mispriced beyond their fees), so rows also arbitrage inside T.

Both are built through test_gpu_order_certificates.PoolSet: a main set laid out with orient_by_degree = 1,
appended pools and retired pools (retired only where the pair keeps an active pool, so a retire never
changes a row's token set)."""
import numpy as np

from test_gpu_order_certificates import DEEP, G, P, U, PoolSet, ladder, pool_spec  # noqa: F401

SG_THREADS = 256                     # kSubgraphThreads: a row's CTA
WIDE_N = 600
LIGHT = list(range(11, WIDE_N))      # B tokens of the light rows (i = 1, j = 2)
HEAVY = list(range(11, 11 + 256))    # B tokens of the deep rows (i = 3, j = 4)
HEAVY_EXTRA = {11: 38, 12: 38, 13: 38}  # more pools on {b, 3}
DEEP_N = 8
DEEP_LINKS = {(4, 5): 3, (6, 7): 2, (7, 8): 1}  # joins the DEEP pairs into one chain 1 .. 8

# Price rows (LinearNonnegative: no token's net may fall below 0) gain only from cycles whose pools disagree;
# over pools that all agree within their fees the optimum profit is 0 and m_r = max ν·|pg| / g is 0 / 0.
# So the neighbour pools from token PRICED_FROM on are mispriced 2 % beyond their fees, and the price rows
# take the light shapes from there (PRICE_OFFSET); the other rows stay below it.
PRICED_FROM = 311
PRICE_OFFSET = PRICED_FROM - LIGHT[0]
N_LOC = (32, 33, 256, 257, 258)
POOL_COUNTS = (255, 256, 257, 511, 512, 513)


class RowSet(PoolSet):
    """A PoolSet that retires no pair's last active pool and builds its device context in build(), with
    the pair lists the row oracles take."""

    def __init__(self, cr, n, specs, seed, **kw):
        super().__init__(cr, n, specs, seed, keep_pairs=True, build=False, **kw)
        self.gidx = {k: e for e, k in enumerate(self.keys())}

    def build(self):
        self.p = self.fresh()
        return self

    def pair_of(self, k):
        a, b = (int(x) for x in self.Ai[k[0]][k[1]])
        return (min(a, b), max(a, b))

    def lists(self):
        """{(a, b): [(type, index, active)]} in global insertion order, as cfmm_pair_pools lists them."""
        out = {}
        for k in self.keys():
            out.setdefault(self.pair_of(k), []).append((k[0], k[1], k not in self.retired))
        return out

    def mask(self, tokens):
        m = np.zeros(self.n, bool)
        m[np.asarray(list(tokens), np.int64) - 1] = True
        return m


def calm_spec(rng, a, b, nu, depth, beyond=1.0):
    """A pool of a random type on {a, b} priced at ν, its misprice inside its fee (none without one),
    times `beyond`."""
    g = float(rng.choice([1.0, 0.9995, 0.997]))
    mis = float(np.exp(rng.uniform(-0.4, 0.4) * (1.0 - g))) * beyond
    return pool_spec(rng, (P, G, U)[int(rng.integers(0, 3))], a, b, nu, depth=depth, misprice=mis, fees=(g,))


def wide_set(cr, seed=91):
    rng = np.random.default_rng(seed)
    nu = {t: float(np.exp(rng.uniform(-1, 1))) for t in range(1, WIDE_N + 1)}
    specs = []
    add = lambda a, b, cnt: specs.extend(calm_spec(rng, a, b, nu, 10.0 ** rng.uniform(2, 4)) for _ in range(cnt))
    add(1, 2, 1)
    for b in LIGHT:
        add(b, 1, 1)
        add(b, 2, 1)
        if b + 1 in LIGHT:
            beyond = float(np.exp(0.02 * (-1) ** b)) if b >= PRICED_FROM else 1.0
            specs.append(calm_spec(rng, b, b + 1, nu, 10.0 ** rng.uniform(2, 4), beyond))
    add(3, 4, 3)
    for b in HEAVY:
        add(b, 3, 2 + HEAVY_EXTRA.get(b, 0))
        add(b, 4, 2)
    ws = RowSet(cr, WIDE_N, specs, seed=seed + 1)
    ws.nu = nu
    return ws


def deep_set(cr, seed=93):
    rng = np.random.default_rng(seed)
    nu = {t: float(np.exp(rng.uniform(-1, 1))) for t in range(1, DEEP_N + 1)}
    specs = []
    for (a, b), cnt in list(DEEP.items()) + list(DEEP_LINKS.items()):
        for k in range(cnt):
            t = (P, G, U)[k % 3] if cnt > 1 else P
            specs.append(pool_spec(rng, t, a, b, nu, misprice=None if rng.random() < 0.4 else
                                   float(np.exp(rng.uniform(-0.001, 0.001)))))
    ds = RowSet(cr, DEEP_N, specs, seed=seed + 1)
    ds.nu = nu
    return ds


# ---- the rows ---------------------------------------------------------------------------------
def light_b(k, adj):
    """k light B tokens with exactly adj neighbour pairs among them: a run of adj + 1, then every other."""
    assert 0 <= adj <= k - 1
    run = LIGHT[:adj + 1]
    rest = LIGHT[adj + 2:adj + 2 + 2 * (k - adj - 1):2]
    out = run + rest
    assert len(out) == k
    return out


def light_for_pools(target, direct=1):
    """Light B tokens whose row (i = 1, j = 2) holds exactly target pools: direct + 2k + adj."""
    for k in range(1, 257):
        adj = target - direct - 2 * k
        if 0 <= adj <= k - 1:
            return light_b(k, adj)
    raise ValueError(target)


def shapes(price=False):
    """{name: (i, j, B)} of the wide set: n_loc 32 .. 258, the pool counts around 256 and 512, and the
    deep row (p2 >= 2048, i holding more than 256 pools, some B tokens 33 to 64).  price: the light
    shapes over the mispriced neighbours (the deep row's pools all agree: no price row fills there)."""
    o = PRICE_OFFSET if price else 0
    shift = lambda B: [t + o for t in B]  # noqa: E731
    out = {f"n_loc={n}": (1, 2, shift(LIGHT[:n - 2])) for n in N_LOC}
    out.update({f"pools={c}": (1, 2, shift(light_for_pools(c))) for c in POOL_COUNTS})
    if not price:
        out["p2>=2048"] = (3, 4, list(HEAVY))
    return out


def deep_rows():
    """{name: (i, j, B)} of the deep/extreme set: multi-token rows across the deep pairs."""
    return {"deep 2<-1 B={3,4}": (2, 1, [3, 4]),
            "deep 1<-4 B={2,3}": (1, 4, [2, 3]),
            "deep 5<-6 B={4,7}": (5, 6, [4, 7]),
            "deep 1<-8 B=all": (1, 8, [2, 3, 4, 5, 6, 7])}


def local_degrees(rs, pools, T):
    """The number of the row's pools holding each token of T."""
    deg = {t: 0 for t in T}
    for k in pools:
        for x in rs.Ai[k[0]][k[1]]:
            deg[int(x)] += 1
    return deg


def p2(n):
    p = 1
    while p < n:
        p <<= 1
    return p
