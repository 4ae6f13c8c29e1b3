"""Synthetic pool sets for the parity tests and bench.py.

Template: the reference's own benchmark generator (benchmark/scaling.jl:13-38)
and its random-market tests (test/arb.jl:60-78):  R = 1000*rand(2),
γ = rand((0.997, 1.0)), Ai = sample(1:n, 2, replace=false),
LinearNonnegative(rand(n)).  Julia's RNG stream is not reproducible outside
Julia, so inputs are drawn from numpy's PCG64 with a fixed seed instead.
"""
from __future__ import annotations

import numpy as np


def token_pairs(rng, m: int, n_tokens: int):
    """m pairs of distinct 1-based token ids, uniform (scaling.jl:22)."""
    a = rng.integers(1, n_tokens + 1, size=m, dtype=np.int64)
    b = rng.integers(1, n_tokens, size=m, dtype=np.int64)
    b = b + (b >= a)  # skip a: uniform over the other n-1 tokens
    return np.stack([a, b], axis=1)


def product_pools(m: int, n_tokens: int, seed: int = 1234):
    """(R [m,2], gamma [m], Ai [m,2] 1-based)."""
    rng = np.random.default_rng(seed)
    R = 1000.0 * rng.random((m, 2))
    R = np.maximum(R, 1e-3)  # rand() can return exactly 0; a pool has reserves
    gamma = rng.choice(np.array([0.997, 1.0]), size=m)
    return R, gamma, token_pairs(rng, m, n_tokens)


def product_pools_skewed(m: int, n_tokens: int, alpha: float = 1.0, seed: int = 1234):
    """Like product_pools, but token popularity follows a Zipf law (rank^-alpha):
    a few hub tokens (the WETH / USDC of a real DEX graph) sit in a large share
    of the pools, on either side.  The reference's own generators are uniform;
    this one exists to exercise hub contention."""
    rng = np.random.default_rng(seed)
    R = np.maximum(1000.0 * rng.random((m, 2)), 1e-3)
    gamma = rng.choice(np.array([0.997, 1.0]), size=m)
    w = 1.0 / np.arange(1, n_tokens + 1) ** alpha
    w /= w.sum()
    a = rng.choice(n_tokens, size=m, p=w) + 1
    b = rng.choice(n_tokens, size=m, p=w) + 1
    clash = a == b
    b[clash] = (a[clash] % n_tokens) + 1
    return R, gamma, np.stack([a, b], axis=1).astype(np.int64)


def geomean_pools(m: int, n_tokens: int, seed: int = 4321):
    """(R, gamma, Ai, w) with w1 ~ U(0.05, 0.95), w2 = 1 - w1 (test/cfmms.jl:101)."""
    rng = np.random.default_rng(seed)
    R = np.maximum(1000.0 * rng.random((m, 2)), 1e-3)
    gamma = rng.choice(np.array([0.997, 1.0]), size=m)
    w1 = rng.uniform(0.05, 0.95, size=m)
    w = np.stack([w1, 1.0 - w1], axis=1)
    return R, gamma, token_pairs(rng, m, n_tokens), w


def univ3_pools(m: int, n_tokens: int, seed: int = 777, ragged: bool = False):
    """Pools shaped like examples/Univ3.jl:11-15 (4 ticks: cp·[2, 4/3, 2/3, 1/3],
    liquidity [1, 2, 1.5, 0]·s); with ragged=True the tick count varies 1..16.
    Returns (current_price, gamma, Ai, tick_off, lower_ticks, liquidity)."""
    rng = np.random.default_rng(seed)
    cp = np.exp(rng.uniform(np.log(0.1), np.log(10.0), size=m))
    s = rng.uniform(1.0, 1000.0, size=m)
    gamma = np.full(m, 0.997)
    Ai = token_pairs(rng, m, n_tokens)
    if not ragged:
        lower = cp[:, None] * np.array([2.0, 4.0 / 3.0, 2.0 / 3.0, 1.0 / 3.0])[None, :]
        liq = s[:, None] * np.array([1.0, 2.0, 1.5, 0.0])[None, :]
        off = np.arange(m + 1, dtype=np.int64) * 4
        return cp, gamma, Ai, off, lower.reshape(-1), liq.reshape(-1)
    T = rng.integers(1, 17, size=m)
    off = np.concatenate([[0], np.cumsum(T)]).astype(np.int64)
    lower = np.empty(off[-1])
    liq = np.empty(off[-1])
    for i in range(m):
        t = int(T[i])
        # strictly decreasing ladder whose first rung is above the current price
        rungs = cp[i] * 2.0 * np.cumprod(np.concatenate([[1.0], rng.uniform(0.5, 0.9, size=t - 1)]))
        lower[off[i]:off[i + 1]] = rungs
        lq = s[i] * rng.uniform(0.0, 2.0, size=t)
        lq[rng.random(t) < 0.15] = 0.0  # some empty ticks (skipped, not terminal)
        liq[off[i]:off[i + 1]] = lq
    return cp, gamma, Ai, off, lower, liq


# ---- token-disjoint pool sets ------------------------------------------------------------
# Pool i holds tokens (2i+1, 2i+2) and no other pool holds either, so Ψ of a gradient-only sweep
# is a per-pool readout: Ψ[2i+1], Ψ[2i+2] are pool i's own Λ−Δ, with no summation order
# involved.  ν is part of each case (every pool has prices of its own), and the first rows of a
# set are adversarial inputs, cycling through their categories so that small sets see them too.

def disjoint_tokens(m: int):
    """Ai[i] = (2i+1, 2i+2): n = 2m tokens, every one in exactly one pool."""
    a = 2 * np.arange(m, dtype=np.int64) + 1
    return np.stack([a, a + 1], axis=1)


def _fill_cyclic(m: int, groups):
    """Row indices for each group of adversarial rows, cycling over the groups so that every
    group gets rows while rows last (the first rows of a small set cover all groups)."""
    sizes = [len(gr) for gr in groups]
    take = [[] for _ in groups]
    row, k = 0, 0
    while row < m and any(k < s for s in sizes):
        for g, s in enumerate(sizes):
            if k < s and row < m:
                take[g].append((row, k))
                row += 1
        k += 1
    return take


def fee_levels(seed: int = 5):
    """256 distinct fees, 1.0 among them: every code of the compact stream's γ dictionary."""
    rng = np.random.default_rng(seed)
    f = np.unique(1.0 - rng.random(400) * 0.05)[::-1]
    f = f[f < 1.0][:255]
    assert len(f) == 255
    return np.concatenate([[1.0], f])


def disjoint_product(m: int, seed: int = 1, adversarial: bool = True):
    """(R, gamma, Ai, v) of a token-disjoint ProductTwoCoin set.  Random rows: all 256 fee codes
    (m >= 512), log2 R2 in U(-25, 40), log2(γP/Q) in U(-40, 40), log2 ν in U(-6, 6).  Adversarial rows:
    γP/Q = 1 ± k·2^-41 (both sides of the economized margin 1 ± 2^-40, both trade directions),
    γP/Q = 2^±80 exactly, a b-side tender of 256·R2·(1 ± δ) (the fixed-point guard), γ = 1."""
    rng = np.random.default_rng(seed)
    fees = fee_levels()
    g = fees[rng.integers(0, len(fees), size=m)]
    if m >= 2 * len(fees):
        g[-len(fees):] = fees                     # every code present (the adversarial rows come first)
    v = np.exp2(rng.uniform(-6, 6, size=2 * m))
    va, vb = v[0::2], v[1::2]                     # views: writes go to v
    R2 = np.exp2(rng.uniform(-25, 40, size=m))
    rho = np.exp2(rng.uniform(-40, 40, size=m))   # target γP/Q; every reserve stays in [2^-100, 2^100]
    R1 = R2 * g * vb / (rho * va)
    R = np.stack([R1, R2], axis=1)
    if adversarial:
        ties = [(k, s) for k in range(-8, 9) for s in (0, 1)]
        wide = [(e, s) for e in (80, 60, 41, -41, -60, -80) for s in (0, 1)]
        guard = [d for d in (0.0, 2.0 ** -40, -2.0 ** -40, 2.0 ** -20, -2.0 ** -20, 2.0 ** -8, -2.0 ** -8)]
        for grp, rows in zip(("ties", "wide", "guard"), _fill_cyclic(m, [ties, wide, guard])):
            for i, k in rows:
                if grp == "ties":
                    kk, side = ties[k]
                    r = 1.0 + kk * 2.0 ** -41       # γP/Q (side 0) or γQ/P (side 1)
                    g[i] = 1.0 if kk % 3 == 0 else g[i]
                    va[i], vb[i] = 1.0, 1.0
                    R[i] = [1.0, r / g[i]] if side == 0 else [r / g[i], 1.0]
                elif grp == "wide":
                    e, side = wide[k]
                    va[i], vb[i] = 1.0, 1.0
                    g[i] = 1.0
                    lo, hi = 2.0 ** (-e / 2), 2.0 ** (e / 2)
                    R[i] = [lo, hi] if side == 0 else [hi, lo]
                else:
                    # token 2 tendered with γ = 1: |Λ2 − Δ2| = R2·(sqrt(Q/P) − 1) = 256·R2·(1 + δ)
                    d = guard[k]
                    g[i], va[i], vb[i] = 1.0, 1.0, 1.0
                    R[i] = [3.0 * (1.0 + 256.0 * (1.0 + d)) ** 2, 3.0]
    return R, g, disjoint_tokens(m), v


def disjoint_geomean(m: int, seed: int = 2, adversarial: bool = True):
    """(R, gamma, Ai, w, v) of a token-disjoint GeometricMeanTwoCoin set.  Random rows: w1/w2 in
    LogU(1/20, 20), uA = ν_a·w2·R1 and uB = ν_b·w1·R2 in 2^U(-28, 28), γ in {0.997, 1}.
    Adversarial rows: w1/w2 at 24 and 1/24 (1 ± δ), uA or uB at the 2^±32 edges (inside and
    outside), |log2(γ uB/uA)| up to 64, ties γ·uB/uA = 1 ± k·2^-31 around the 1 ± 2^-30 margin."""
    rng = np.random.default_rng(seed)
    g = rng.choice(np.array([0.997, 1.0]), size=m)
    eta = np.exp(rng.uniform(np.log(1 / 20), np.log(20), size=m))
    w = np.stack([eta / (1 + eta), 1 / (1 + eta)], axis=1)
    v = np.exp2(rng.uniform(-4, 4, size=2 * m))
    va, vb = v[0::2], v[1::2]
    uA = np.exp2(rng.uniform(-28, 28, size=m))
    uB = np.exp2(rng.uniform(-28, 28, size=m))
    R = np.stack([uA / (va * w[:, 1]), uB / (vb * w[:, 0])], axis=1)
    if adversarial:
        cut = [(c, d) for c in (24.0, 1 / 24) for d in (0.0, 2.0 ** -40, -2.0 ** -40, 2.0 ** -10, -2.0 ** -10)]
        edge = [(x, y) for x in (2.0 ** 32 * (1 - 2.0 ** -53), 2.0 ** 32, 2.0 ** -32, 2.0 ** -32 * (1 - 2.0 ** -53))
                for y in (1.0, 2.0 ** -31, 2.0 ** 31)] + [(2.0 ** -32, 2.0 ** 32 * (1 - 2.0 ** -52)),
                                                         (2.0 ** 32 * (1 - 2.0 ** -52), 2.0 ** -32)]
        ties = [(k, s) for k in range(-4, 5) for s in (0, 1)]
        for grp, rows in zip(("cut", "edge", "ties"), _fill_cyclic(m, [cut, edge, ties])):
            for i, k in rows:
                va[i], vb[i] = 1.0, 1.0
                if grp == "cut":
                    c, d = cut[k]
                    w[i] = [c * (1 + d), 1.0]
                    R[i] = [3.0, 5.0]
                elif grp == "edge":
                    x, y = edge[k]            # uA, uB with ν = 1, w = (1/2, 1/2) scaled to 1
                    g[i] = 1.0
                    w[i] = [1.0, 1.0]
                    R[i] = [x, y] if k % 2 == 0 else [y, x]
                else:
                    kk, side = ties[k]
                    g[i] = 1.0
                    w[i] = [0.5, 0.5]
                    r = 1.0 + kk * 2.0 ** -31
                    R[i] = [7.0, 7.0 * r] if side == 0 else [7.0 * r, 7.0]
    return R, g, disjoint_tokens(m), w, v


def disjoint_univ3(m: int, seed: int = 3, ragged: bool = False, adversarial: bool = True):
    """(current_price, gamma, Ai, tick_off, lower_ticks, liquidity, v) of a token-disjoint UniV3
    set, ladders shaped like univ3_pools.  Adversarial rows: p = ν1/ν2 exactly at γ·cp and at
    cp/γ (the no-trade band edges), p exactly on a tick price, beyond the last tick in both
    directions, single-tick pools, zero liquidity in the current tick, all ticks empty."""
    cp, g, _, off, lower, liq = univ3_pools(m, 2, seed=seed, ragged=ragged)
    rng = np.random.default_rng(seed + 1)
    p = cp * np.exp(rng.uniform(np.log(0.25), np.log(4.0), size=m))
    v = np.ones(2 * m)
    v[0::2] = p
    if not adversarial:
        return cp, g, disjoint_tokens(m), off, lower, liq, v
    cases = ["band_lo", "band_hi", "tick_lo", "tick_hi", "below", "above",
             "single_lo", "single_hi", "empty_cur", "all_empty"]
    # rebuild the ladders of the adversarial rows (single-tick rows change the CSR)
    rows = {i: cases[i % len(cases)] for i in range(min(m, 4 * len(cases)))}
    lad = [(lower[off[i]:off[i + 1]].copy(), liq[off[i]:off[i + 1]].copy()) for i in range(m)]
    for i, case in rows.items():
        lt, lq = lad[i]
        if case.startswith("single"):
            lt, lq = np.array([cp[i] * 1.5]), np.array([10.0 + i])
        if len(lt) < 3 and case in ("tick_lo", "tick_hi", "empty_cur"):
            lt = cp[i] * np.array([2.0, 4.0 / 3.0, 2.0 / 3.0, 1.0 / 3.0])
            lq = (10.0 + i) * np.array([1.0, 2.0, 1.5, 0.0])
        ct = int(np.sum(lt >= cp[i]))       # current tick (1-based): the last rung >= cp
        if case == "empty_cur":
            lq = lq.copy()
            lq[ct - 1] = 0.0
        if case == "all_empty":
            lq = np.zeros_like(lq)
        lad[i] = (lt, lq)
        if case == "band_lo":
            v[2 * i] = g[i] * cp[i]
        elif case == "band_hi":
            v[2 * i] = cp[i] / g[i]
        elif case == "tick_lo":
            v[2 * i] = lt[min(ct, len(lt) - 1)]          # on the rung below the current one
        elif case == "tick_hi":
            v[2 * i] = lt[max(ct - 2, 0)]                # on the rung above
        elif case in ("below", "single_lo"):
            v[2 * i] = lt[-1] * 1e-3
        elif case in ("above", "single_hi"):
            v[2 * i] = lt[0] * 1e3
        else:
            v[2 * i] = cp[i] * (0.3 if i % 2 else 3.0)
    T = np.array([len(lt) for lt, _ in lad], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(T)]).astype(np.int64)
    lower = np.concatenate([lt for lt, _ in lad])
    liq = np.concatenate([lq for _, lq in lad])
    return cp, g, disjoint_tokens(m), off, lower, liq, v


def objective_prices(n_tokens: int, seed: int = 99):
    """c = rand(n) for LinearNonnegative (scaling.jl:31), kept away from 0."""
    rng = np.random.default_rng(seed)
    return rng.uniform(0.05, 1.0, size=n_tokens)


def dual_prices(n_tokens: int, kind: str = "near", seed: int = 7):
    """ν for timing/parity: 'ones' = the benchmark's start (scaling.jl:16);
    'near' = c·(1 + 0.05·U(0,1)), an in-bounds, near-optimal point;
    'wide' = LogU(0.2, 5), every pool far from its no-trade band."""
    rng = np.random.default_rng(seed)
    if kind == "ones":
        return np.ones(n_tokens)
    if kind == "near":
        return objective_prices(n_tokens) * (1.0 + 0.05 * rng.random(n_tokens))
    if kind == "wide":
        return np.exp(rng.uniform(np.log(0.2), np.log(5.0), size=n_tokens))
    raise ValueError(kind)
