"""GPU parity tests: the CUDA path, called through the C ABI (ctypes over
libcfmm_b200.so), against the CPU oracle on the same seeded inputs.

Bars (BASELINE north_star): token-index scatter bit-exact; Δ, Λ, Ψ within 1e-6
relative.  What is actually enforced here is tighter:
  ProductTwoCoin / UniV3 : Δ, Λ BIT-EXACT per pool (both the default fast path
                           and exact=1), because every operation is IEEE
                           correctly rounded on both sides;
  GeometricMeanTwoCoin   : |Δgpu−Δcpu| ≤ 1e-12·max(R)/γ (CUDA pow vs glibc pow
                           differ in the last ulps);
  Ψ, acc                 : ‖Ψgpu−Ψref‖∞ ≤ 1e-6‖Ψref‖∞ AND component-wise
                           ≤ 1e-12·Σ(|Λ|+|Δ|)_j vs an extended-precision
                           pool-order sum (atomics reorder the fp64 adds).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def make_pools(cr, n, product=None, geomean=None, univ3=None, exact=None, pre=None):
    p = cr.DevicePools(n)
    for k, val in (pre or {}).items():  # options that fix the layout (before finalize)
        p.set_option(k, val)
    if product is not None:
        p.add_product(*product)
    if geomean is not None:
        p.add_geomean(*geomean)
    if univ3 is not None:
        p.add_univ3(*univ3)
    p.finalize()
    if exact is not None:
        p.set_option("exact", exact)
    return p


EPS = np.finfo(np.float64).eps


def check_psi(oracle, Ai, D, L, v, n, psi, acc, R=None, g=None, Rq=None):
    """Ψ, acc against an extended-precision pool-order sum of the oracle's
    per-pool trades.  Strict form (R is None): only summation-order noise is
    allowed, 1e-12·Σ(|Λ|+|Δ|)_j per component.  With R, g given (gradient-only
    ProductTwoCoin sweeps in the default economized math) each pool may add up
    to 32 ulp of its reserves: the same order as the rounding of the
    reference's own expression sqrt(γmk) − R.  Rq (the reserves; defaults to R):
    gradient-only sweeps of the TMA kernel accumulate Ψ[b] partials in 64-bit
    fixed point with the quantum 2^(e−54), e = ilogb(S_j·(1+2^-30)) + 1, i.e. at most
    2^-53 S_j, so each of token j's pools may round by up to half of it, 2^-54 S_j.
    The allowance deg_j · S_j · 2^-59 does NOT cover that worst case: it is 32x smaller.
    These tests pass because the 1e-12·Σ(|Λ|+|Δ|)_j term dominates on their pool sets,
    where every token's pools trade a sizeable share of S_j.  A token whose pools trade
    very little next to S_j could exceed it with a correct kernel.  The quantisation
    itself is checked exactly, pool by pool, in test_gpu_pool_readout.py (the integer
    sum is exact and order-independent)."""
    accx, Gx, absG = oracle.fold_compensated(Ai, D, L, v, n)
    ref = Gx.astype(np.float64)
    slack = np.zeros(n)
    if R is not None:
        w = 32 * EPS * (R[:, 0] + R[:, 1]) / g
        np.add.at(slack, Ai[:, 0] - 1, w)
        np.add.at(slack, Ai[:, 1] - 1, w)
    if Rq is None:
        Rq = R
    if Rq is not None:
        S, deg = np.zeros(n), np.zeros(n)
        for side in (0, 1):
            np.add.at(S, Ai[:len(Rq), side] - 1, np.abs(Rq[:, side]))
            np.add.at(deg, Ai[:len(Rq), side] - 1, 1.0)
        slack = slack + deg * S * 2.0 ** -59
    # north_star tolerance: 1e-6 relative (norm-wise); the rounding floor of the sums
    # themselves is added so that a Ψ that is zero up to noise (pools already at their
    # no-arbitrage point) does not turn the relative test into noise / noise
    floor = float(np.max(1e-12 * absG + slack)) if n else 0.0
    assert np.max(np.abs(psi - ref)) <= 1e-6 * max(np.max(np.abs(ref)), 1e-300) + floor
    assert np.all(np.abs(psi - ref) <= 1e-12 * absG + slack + 1e-300)
    scale = float(np.sum(absG * v))
    aslack = float(np.sum(slack * v))
    assert abs(acc - float(accx)) <= 1e-12 * scale + aslack + 1e-300
    # acc == νᵀΨ (router.jl:79-83 vs 98-100)
    assert abs(acc - float(np.dot(v, psi))) <= 1e-11 * scale + 2 * aslack + 1e-300


# ---------------------------------------------------------------------------
# known-answer tests of the reference, through find_arb!(Δ, Λ, cfmm, v)
# ---------------------------------------------------------------------------

def test_reference_kats_product(cr):
    # test/cfmms.jl:70-90
    D, L = np.zeros(2), np.zeros(2)
    pool = cr.ProductTwoCoin([1, 1], 1, [1, 2])
    cr.find_arb(D, L, pool, [1.0, 1.0])
    assert not D.any() and not L.any()
    cr.find_arb(D, L, pool, [2.0, 2.0])
    assert not D.any() and not L.any()
    cr.find_arb(D, L, pool, [2.0, 1.0])
    assert D[0] == 0 and D[1] == 0.41421356237309515
    assert L[0] == 0.2928932188134524 and L[1] == 0
    assert len(cr.ProductTwoCoin([1, 1], .9, [1, 2])) == 2
    with pytest.raises(ValueError):
        cr.ProductTwoCoin([1, 1], .9, [1])


@pytest.mark.parametrize("gamma", [1.0, 0.997])
def test_reference_univ3_scenarios(cr, oracle, gamma):
    # test/cfmms.jl:117-201: the seven price scenarios, bit-exact vs the oracle
    cp, lt, lq = 15.0, [30.0, 20, 10, 5], [1.0, 2.0, 1.5, 0.0]
    pool = cr.UniV3(cp, lt, lq, gamma, [1, 2])
    assert pool.current_tick == 2
    first = [15.0, 1.0] if gamma == 1.0 else [15.0 * (1 + gamma) / 2, 1.0]
    for v in (first, [16.0, 1.0], [14.0, 1.0], [25.0, 1.0], [7.5, 1.0], [4.0, 1.0], [35.0, 1.0]):
        D, L = np.zeros(2), np.zeros(2)
        cr.find_arb(D, L, pool, v)
        Do, Lo = oracle.univ3_arb(cp, lt, lq, gamma, v)
        assert np.array_equal(D, Do) and np.array_equal(L, Lo), (v, D, Do, L, Lo)


def test_golden_vectors(cr):
    import json, os
    with open(os.path.join(os.path.dirname(__file__), "golden", "closed_forms.json")) as f:
        g = json.load(f)
    eps = np.finfo(np.float64).eps
    for case in g["product"]:
        D, L = np.zeros(2), np.zeros(2)
        cr.find_arb(D, L, cr.ProductTwoCoin(case["R"], case["gamma"], [1, 2]), case["v"])
        scale = max(case["R"]) / min(case["gamma"], 1.0)
        assert np.all(np.abs(D - np.array([float(s) for s in case["Delta"]])) <= 8 * eps * scale)
        assert np.all(np.abs(L - np.array([float(s) for s in case["Lambda"]])) <= 8 * eps * scale)
    for case in g["geomean"][:40]:
        D, L = np.zeros(2), np.zeros(2)
        cr.find_arb(D, L, cr.GeometricMeanTwoCoin(case["R"], case["w"], case["gamma"], [1, 2]), case["v"])
        scale = max(case["R"]) / min(case["gamma"], 1.0)
        assert np.all(np.abs(D - np.array([float(s) for s in case["Delta"]])) <= 256 * eps * scale)
        assert np.all(np.abs(L - np.array([float(s) for s in case["Lambda"]])) <= 256 * eps * scale)


# ---------------------------------------------------------------------------
# sweep parity per pool type
# ---------------------------------------------------------------------------

@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("m,n", [(1, 2), (31, 5), (64, 7), (1000, 10), (100_000, 1000), (300_007, 4099)])
@pytest.mark.parametrize("kind", ["near", "wide", "ones"])
def test_product_sweep_parity(cr, oracle, synth, m, n, kind, exact):
    R, g, Ai = synth.product_pools(m, n, seed=m + n)
    v = synth.dual_prices(n, kind)
    p = make_pools(cr, n, product=(R, g, Ai), exact=exact)
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    assert np.array_equal(D, Do), np.argwhere(D != Do)[:5]
    assert np.array_equal(L, Lo), np.argwhere(L != Lo)[:5]
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    # the gradient-only sweep: default economized math (few ulp of the reserves) ...
    psi2, acc2 = p.sweep(v, materialize=False)
    check_psi(oracle, Ai, Do, Lo, v, n, psi2, acc2, R=R, g=g)
    # ... and the reference operation order (only summation-order noise)
    p.set_option("gradient_math", 0)
    psi3, acc3 = p.sweep(v, materialize=False)
    check_psi(oracle, Ai, Do, Lo, v, n, psi3, acc3, Rq=R)
    # ... and with fp64 (CAS) slice partials instead of fixed point: strictly summation noise
    p.set_option("psi_fixed_point", 0)
    psi4, acc4 = p.sweep(v, materialize=False)
    check_psi(oracle, Ai, Do, Lo, v, n, psi4, acc4)
    p.close()


def test_product_ties_and_extremes(cr, oracle):
    """Exact ties (fee-less pool at its own price), the no-trade band edge and
    huge/tiny magnitudes: the fast path must fall back to the full form."""
    R = np.array([[1, 1], [3, 7], [100, 100], [1e-150, 1e-150], [1e150, 1e150], [5, 9], [2, 8], [1e3, 2e3]], dtype=float)
    g = np.array([1, 1, 1, 1, 1, 0.5, 0.997, 0.997])
    Ai = np.array([[1, 2], [1, 2], [2, 1], [1, 2], [2, 1], [1, 2], [3, 4], [4, 3]])
    v = np.array([7.0, 3.0, 8.0 * 0.997, 2.0])
    for exact in (0, 1):
        p = make_pools(cr, 4, product=(R, g, Ai), exact=exact)
        p.sweep(v, materialize=True)
        D, L = p.trades()
        Do, Lo = oracle.sweep_product(R, g, Ai, v)
        assert np.array_equal(D, Do) and np.array_equal(L, Lo)
        p.close()


@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("m,n", [(1, 2), (65, 9), (50_000, 500)])
def test_geomean_sweep_parity(cr, oracle, synth, m, n, exact):
    R, g, Ai, w = synth.geomean_pools(m, n, seed=m)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, geomean=(R, g, Ai, w), exact=exact)
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_geomean(R, g, Ai, w, v, threads=8)
    tol = 1e-12 * (np.max(R, axis=1) / g)[:, None]
    assert np.all(np.abs(D - Do) <= tol) and np.all(np.abs(L - Lo) <= tol)
    assert np.all((D == 0) == (Do == 0)) and np.all((L == 0) == (Lo == 0))
    # 1e-6 relative where the trade is non-negligible
    big = Do > 1e-6 * np.max(R, axis=1)[:, None]
    assert np.all(np.abs(D - Do)[big] <= 1e-6 * Do[big])
    # fold parity against the GPU's own per-pool trades
    check_psi(oracle, Ai, D, L, v, n, psi, acc)
    if exact == 0:
        # gradient-only sweep: economized one-pow form (few ulp of the reserves) ...
        psi2, acc2 = p.sweep(v)
        check_psi(oracle, Ai, D, L, v, n, psi2, acc2, R=R, g=g)
        # ... the same on the first-generation kernel (the default is the TMA kernel) ...
        p.set_option("geomean_tma", 0)
        psi4, acc4 = p.sweep(v)
        check_psi(oracle, Ai, D, L, v, n, psi4, acc4, R=R, g=g)
        p.set_option("geomean_tma", 1)
        # ... and the reference operation order
        p.set_option("gradient_math", 0)
        psi3, acc3 = p.sweep(v)
        check_psi(oracle, Ai, D, L, v, n, psi3, acc3, Rq=R)
    p.close()


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("m,n", [(1, 2), (100, 6), (20_000, 300)])
def test_univ3_sweep_parity(cr, oracle, synth, m, n, ragged):
    cp, g, Ai, off, lt, lq = synth.univ3_pools(m, n, seed=m, ragged=ragged)
    # prices with p/cp ~ LogU(0.25, 4): 0-3 tick crossings in both directions
    rng = np.random.default_rng(3)
    v = np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n))
    p = make_pools(cr, n, univ3=(cp, g, Ai, off, lt, lq))
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_univ3(cp, g, Ai, off, lt, lq, v, threads=8)
    assert np.array_equal(D, Do), np.argwhere(D != Do)[:5]
    assert np.array_equal(L, Lo), np.argwhere(L != Lo)[:5]
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    p.close()


def test_mixed_types_insertion_order(cr, oracle, synth):
    """Trades come back in global insertion order across pool types."""
    n = 40
    Rp, gp, Ap = synth.product_pools(300, n, seed=1)
    Rg, gg, Ag, wg = synth.geomean_pools(200, n, seed=2)
    cp, gu, Au, off, lt, lq = synth.univ3_pools(100, n, seed=3)
    v = synth.dual_prices(n, "wide")
    p = cr.DevicePools(n)
    p.add_product(Rp[:100], gp[:100], Ap[:100])
    p.add_geomean(Rg, gg, Ag, wg)
    p.add_product(Rp[100:], gp[100:], Ap[100:])
    p.add_univ3(cp, gu, Au, off, lt, lq)
    p.finalize()
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    D1, L1 = oracle.sweep_product(Rp, gp, Ap, v)
    D2, L2 = oracle.sweep_geomean(Rg, gg, Ag, wg, v)
    D3, L3 = oracle.sweep_univ3(cp, gu, Au, off, lt, lq, v)
    assert np.array_equal(D[:100], D1[:100]) and np.array_equal(D[300:500], D1[100:])
    assert np.allclose(D[100:300], D2, rtol=1e-12, atol=1e-9)
    assert np.array_equal(D[500:], D3) and np.array_equal(L[500:], L3)
    Ai = np.concatenate([Ap[:100], Ag, Ap[100:], Au])
    check_psi(oracle, Ai, D, L, v, n, psi, acc)
    p.close()


# ---------------------------------------------------------------------------
# second-generation ProductTwoCoin kernel (TMA-staged, guard-free in-range math)
# ---------------------------------------------------------------------------

def test_inrange_math(cr):
    """The guard-free div / sqrt recurrences equal IEEE `/` and sqrt bit for bit
    on operands in the validated range, including adversarial mantissas."""
    import ctypes as C
    rng = np.random.default_rng(12345)
    n = 4_000_000
    expo = rng.integers(-100, 100, size=n)
    a = np.ldexp(1.0 + rng.random(n), expo)
    b = np.ldexp(1.0 + rng.random(n), rng.integers(-100, 100, size=n))
    # mantissas near 1, near 2, all-ones, powers of two, perfect squares
    edge = np.array([1.0, 1.0 + 2**-52, 2.0 - 2**-52, 1.5, 1.0 + 2**-26, 4.0, 9.0, 0.25, 3.0, 7.0, 1e10, 1e-10])
    a[:len(edge) ** 2] = np.repeat(edge, len(edge))
    b[:len(edge) ** 2] = np.tile(edge, len(edge))
    a[1000:2000] = np.ldexp(1.0 + 2.0 ** -rng.integers(1, 53, size=1000), rng.integers(-100, 100, size=1000))
    b[1000:2000] = np.ldexp(2.0 - 2.0 ** -rng.integers(1, 52, size=1000), rng.integers(-100, 100, size=1000))
    p = cr.DevicePools(2)
    bad = C.c_int64(-1)
    rc = p._lib.cfmm_selftest_inrange_math(p._ctx, a.ctypes.data_as(C.POINTER(C.c_double)),
                                           b.ctypes.data_as(C.POINTER(C.c_double)), n, C.byref(bad))
    assert rc == 0 and bad.value == 0, bad.value
    p.close()


@pytest.mark.parametrize("variant,fixed,per_sm,compact", [(-1, 1, 0, 1), (0, 1, 0, 1), (0, 0, 0, 1), (0, 1, 1, 1),
                                                           (0, 1, 0, 0), (0, 0, 0, 0)])
@pytest.mark.parametrize("m,n", [(200_003, 3_001), (300_000, 20_011), (5_000, 7), (96, 2), (97, 1601), (40_000, 1601)])
def test_product_gradient_sweep_variants(cr, oracle, synth, variant, fixed, per_sm, compact, m, n):
    """The b-bucketed TMA kernel with fixed-point and with fp64 slice partials, with the 20-byte
    (γ dictionary, chunk-relative first token) and the 32-byte stream, with two and with one CTA per SM (several buckets at
    n = 20011, one bucket at n = 7, a single chunk, two buckets with CTAs that straddle the
    boundary), and the first-generation kernel (-1)."""
    R, g, Ai = synth.product_pools(m, n, seed=variant + 10)
    p = make_pools(cr, n, product=(R, g, Ai), pre={"tma_variant": variant})
    p.set_option("psi_fixed_point", fixed)
    p.set_option("blocks_per_sm", per_sm)
    p.set_option("compact_stream", compact)
    for kind in ("near", "wide"):
        v = synth.dual_prices(n, kind)
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
        p.set_option("gradient_math", 1)
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
        p.set_option("gradient_math", 0)
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, Rq=R if fixed else None)
    # same layout, first-generation kernel
    p.set_option("use_tma", 0)
    psi, acc = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    # trades in insertion order despite the bucketed, padded device order
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    with pytest.raises(cr.CFMMError):  # the layout is fixed at finalize
        p.set_option("tma_variant", 0)
    p.close()


def test_many_fee_levels_keep_the_wide_stream(cr, oracle, synth):
    """More than 256 distinct fees: no γ dictionary, the 32-byte stream is used; exactly 256 (and a
    fee of 1.0 among them) still go through the dictionary.  Ψ must match the oracle either way, and
    the speed feedback of the CTA ranges (many sweeps on the same pools) must not change results."""
    m, n = 150_000, 2_500
    R, g, Ai = synth.product_pools(m, n, seed=17)
    rng = np.random.default_rng(5)
    for levels in (1000, 256):
        fees = np.concatenate([[1.0], 1.0 - rng.random(levels - 1) * 0.05])
        g2 = fees[rng.integers(0, levels, size=m)]
        g2[:levels] = fees            # every level present
        p = make_pools(cr, n, product=(R, g2, Ai))
        for k in range(12):
            v = synth.dual_prices(n, ["wide", "near"][k % 2], seed=k)
            Do, Lo = oracle.sweep_product(R, g2, Ai, v, threads=8)
            psi, acc = p.sweep(v)
            check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g2)
        p.close()


def test_fixed_point_slice_rules(cr, oracle, synth):
    """The fixed-point slice is used only when every token's pools span <= 2^40 in
    reserve; a pool set that violates the rule silently takes the fp64 slice, and a
    reserve push that repairs it switches back.  Oversized tenders (|flow| > 4 R2) and
    NaN leave the integer path through a global fp64 RED.  Checked through results
    only: Ψ must match the oracle in every state."""
    m, n = 120_000, 2_000
    R, g, Ai = synth.product_pools(m, n, seed=9)
    R[5] = [3.0e-9, 2.0e-9]                    # 2^40 below its tokens' totals (~1e5)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, product=(R, g, Ai))
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    psi, acc = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g, Rq=np.zeros_like(R))  # fp64 slice: no quantisation
    R[5] = [30.0, 20.0]
    p.update_reserves(0, 5, R[5:6])
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    psi, acc = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    # prices 1e6 apart: most pools tender far more than 4x their reserve
    v2 = v.copy()
    v2[::2] *= 1.0e6
    Do, Lo = oracle.sweep_product(R, g, Ai, v2, threads=8)
    psi, acc = p.sweep(v2)
    check_psi(oracle, Ai, Do, Lo, v2, n, psi, acc, R=R * 1e4, g=g)
    p.set_option("gradient_math", 0)
    psi, acc = p.sweep(v2)
    check_psi(oracle, Ai, Do, Lo, v2, n, psi, acc, Rq=R)
    p.close()


@pytest.mark.parametrize("orient", [-1, 1, 0])
def test_skewed_token_graph(cr, oracle, synth, orient):
    """Zipf-distributed tokens (hubs on either side of many pools): per-pool
    trades stay bit-exact and in insertion order whether or not pools are stored
    with their tokens exchanged; Ψ within tolerance; reserves update correctly."""
    m, n = 200_000, 5_000
    R, g, Ai = synth.product_pools_skewed(m, n, alpha=1.0, seed=77)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, product=(R, g, Ai), pre={"orient_by_degree": orient})
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    psi, acc = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    R2 = R.copy()
    R2[1000:90_000] *= 1.25
    p.update_reserves(0, 1000, R2[1000:90_000])
    p.sweep(v, materialize=True)
    D, L = p.trades()
    D2, L2 = oracle.sweep_product(R2, g, Ai, v, threads=8)
    assert np.array_equal(D, D2) and np.array_equal(L, L2)
    p.close()


def test_device_resident_api(cr, oracle, synth):
    """cfmm_sweep_device (caller's buffer) and cfmm_sweep_device_view (zero-copy,
    ping-pong accumulators cleared in-kernel) over many consecutive sweeps."""
    import torch
    n = 7_001
    R, g, Ai = synth.product_pools(150_000, n, seed=31)
    Rg, gg, Ag, wg = synth.geomean_pools(20_000, n, seed=32)
    p = make_pools(cr, n, product=(R, g, Ai), geomean=(Rg, gg, Ag, wg))
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.full((n + 1,), 7.0, dtype=torch.float64, device=dev)  # must be overwritten, not accumulated
    for k, kind in enumerate(["wide", "near", "ones", "wide", "near"]):
        v = synth.dual_prices(n, kind, seed=k)
        d_v = torch.from_numpy(v).to(dev)
        D1, L1 = oracle.sweep_product(R, g, Ai, v, threads=8)
        p.sweep(v, materialize=True)  # geomean reference = the GPU's own per-pool trades
        D, L = p.trades()
        assert np.array_equal(D[:150_000], D1)
        A = np.concatenate([Ai, Ag])
        p.sweep_device(d_v.data_ptr(), out.data_ptr(), False, stream)
        torch.cuda.synchronize()
        h = out.cpu().numpy()
        check_psi(oracle, A, D, L, v, n, h[:n], float(h[n]), R=np.concatenate([R, Rg]), g=np.concatenate([g, gg]))
        ptr = p.sweep_device_view(d_v.data_ptr(), False, stream)
        torch.cuda.synchronize()
        # read the context-owned buffer through torch: wrap the raw pointer
        check = _from_ptr(torch, ptr, n + 1, dev).clone().cpu().numpy()
        check_psi(oracle, A, D, L, v, n, check[:n], float(check[n]), R=np.concatenate([R, Rg]), g=np.concatenate([g, gg]))
    p.close()


def test_flat_pool_file_ingest(cr, oracle, synth, tmp_path):
    """cfmm_add_pool_file == cfmm_add_product / cfmm_add_geomean on the same arrays (insertion
    order across files and direct adds included); a file for another token count is refused."""
    n = 700
    R, g, Ai = synth.product_pools(30_000, n, seed=8)
    Rg, gg, Ag, wg = synth.geomean_pools(5_000, n, seed=9)
    cr.write_pool_file(tmp_path / "a.cfmm", n, R[:20_000], g[:20_000], Ai[:20_000])
    cr.write_pool_file(tmp_path / "g.cfmm", n, Rg, gg, Ag, wg)
    p = cr.DevicePools(n)
    p.add_file(tmp_path / "a.cfmm")
    p.add_file(tmp_path / "g.cfmm")
    p.add_product(R[20_000:], g[20_000:], Ai[20_000:])
    p.finalize()
    q = make_pools(cr, n, product=(R, g, Ai), geomean=(Rg, gg, Ag, wg))
    v = synth.dual_prices(n, "wide")
    p.sweep(v, materialize=True)
    q.sweep(v, materialize=True)
    Dp, Lp = p.trades()
    Dq, Lq = q.trades()
    # p's insertion order: product[:20k], geomean, product[20k:];  q's: product, geomean
    assert np.array_equal(Dp[:20_000], Dq[:20_000]) and np.array_equal(Dp[25_000:], Dq[20_000:30_000])
    assert np.array_equal(Dp[20_000:25_000], Dq[30_000:]) and np.array_equal(Lp[20_000:25_000], Lq[30_000:])
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    assert np.array_equal(Dq[:30_000], Do) and np.array_equal(Lq[:30_000], Lo)
    other = cr.DevicePools(n + 1)
    with pytest.raises(cr.CFMMError):
        other.add_file(tmp_path / "a.cfmm")
    for x in (p, q, other):
        x.close()


def test_sweep_graph_replay(cr, oracle, synth):
    """cfmm_sweep on the same pinned buffers: eager, then captured, then replayed as one
    graph launch; ν changes between calls, options and reserve pushes invalidate the graphs,
    materialising and device-resident sweeps interleave (both parities).  Every result is
    checked against the oracle, and the launch counter keeps counting one kernel per replay."""
    n = 3_001
    R, g, Ai = synth.product_pools(150_000, n, seed=41)
    p = make_pools(cr, n, product=(R, g, Ai))
    rng = np.random.default_rng(0)
    for it in range(14):
        v = synth.dual_prices(n, ["near", "wide"][it % 2], seed=100 + it)
        if it == 6:
            p.set_option("gradient_math", 0)     # bumps the version: graphs are re-captured
        if it == 9:
            p.set_option("gradient_math", 1)
            R = R.copy()
            R[10:5000] *= 1.5
            p.update_reserves(0, 10, R[10:5000])
        if it == 11:
            p.sweep(v, materialize=True)          # flips the accumulator parity only
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
        l0 = p.launch_count
        psi, acc = p.sweep(v)
        assert p.launch_count - l0 in (1, 2)      # one sweep kernel (+ a re-pack after option / reserve changes)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    p.set_option("sweep_graphs", 0)
    psi2, acc2 = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi2, acc2, R=R, g=g)
    p.close()


def _from_ptr(torch, ptr, count, dev):
    """A float64 torch view of `count` elements at a raw device pointer."""
    class _Holder:
        pass
    h = _Holder()
    h.__cuda_array_interface__ = {"shape": (count,), "typestr": "<f8", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device=dev)


def test_update_reserves_bucketed_layout(cr, oracle, synth):
    n = 9_000  # 3 buckets with the default tile shape
    R, g, Ai = synth.product_pools(50_000, n, seed=21)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, product=(R, g, Ai))
    R2 = R.copy()
    R2[777:30_001] *= 0.75
    p.update_reserves(0, 777, R2[777:30_001])
    psi, acc = p.sweep(v)
    Do, Lo = oracle.sweep_product(R2, g, Ai, v, threads=8)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R2, g=g)
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    p.close()


def test_product_fast_kernel_fallbacks(cr, oracle, synth):
    """Inputs outside the validated range (ν or reserves), ties and γ > 1 must
    all give the reference result through the generic path."""
    m, n = 50_000, 500
    R, g, Ai = synth.product_pools(m, n, seed=5)
    v = synth.dual_prices(n, "wide")
    for mutate in ("nu_tiny", "nu_huge", "nu_nan", "R_tiny", "gamma_gt1", "ties"):
        R2, g2, v2 = R.copy(), g.copy(), v.copy()
        if mutate == "nu_tiny":
            v2[7] = 1e-200
        elif mutate == "nu_huge":
            v2[11] = 1e200
        elif mutate == "nu_nan":
            v2[13] = np.nan
        elif mutate == "R_tiny":
            R2[100] = [1e-180, 1e-170]
        elif mutate == "gamma_gt1":
            g2[5] = 1.01
        else:
            # pools exactly at their no-arbitrage price: R1 ν1 == R2 ν2, γ = 1
            g2[:1000] = 1.0
            R2[:1000, 0] = v2[Ai[:1000, 1] - 1] * 8.0
            R2[:1000, 1] = v2[Ai[:1000, 0] - 1] * 8.0
        p = make_pools(cr, n, product=(R2, g2, Ai))
        psi, acc = p.sweep(v2)
        Do, Lo = oracle.sweep_product(R2, g2, Ai, v2, threads=8)
        if mutate == "nu_nan":
            accx, Gx, absG = oracle.fold_compensated(Ai, Do, Lo, v2, n)
            ref = Gx.astype(np.float64)
            assert np.array_equal(np.isnan(psi), np.isnan(ref)) and np.isnan(acc)
            ok = ~np.isnan(ref)
            assert np.all(np.abs(psi[ok] - ref[ok]) <= 1e-12 * absG[ok] + 1e-300)
        else:
            check_psi(oracle, Ai, Do, Lo, v2, n, psi, acc, R=np.minimum(R2, 1e6), g=np.minimum(g2, 1.0))
        # and the materialised trades are bit-exact as always
        p.sweep(v2, materialize=True)
        D, L = p.trades()
        assert np.array_equal(D, Do, equal_nan=True) and np.array_equal(L, Lo, equal_nan=True)
        p.close()


# ---------------------------------------------------------------------------
# edge cases and error behaviour of the boundary
# ---------------------------------------------------------------------------

def test_empty_pool_set(cr):
    p = cr.DevicePools(5)
    p.finalize()
    psi, acc = p.sweep(np.ones(5))
    assert not psi.any() and acc == 0.0
    p.close()


def test_error_codes(cr):
    p = cr.DevicePools(3)
    with pytest.raises(cr.CFMMError) as e:  # BoundsError analogue
        p.add_product([[1, 1]], [1.0], [[1, 4]])
    assert e.value.code == -1 and "outside 1..3" in e.value.message
    with pytest.raises(cr.CFMMError):  # duplicate index
        p.add_product([[1, 1]], [1.0], [[2, 2]])
    with pytest.raises(cr.CFMMError) as e:  # sweep before finalize
        p.sweep(np.ones(3))
    assert e.value.code == -3
    with pytest.raises(cr.CFMMError):  # current price above the first tick
        p.add_univ3([31.0], [1.0], [[1, 2]], [0, 2], [30.0, 20.0], [1.0, 1.0])
    with pytest.raises(cr.CFMMError):  # ticks not decreasing
        p.add_univ3([15.0], [1.0], [[1, 2]], [0, 2], [20.0, 30.0], [1.0, 1.0])
    p.finalize()
    with pytest.raises(cr.CFMMError):
        p.add_product([[1, 1]], [1.0], [[1, 2]])
    with pytest.raises(cr.CFMMError) as e:
        p.trades()
    assert e.value.code == -3
    p.close()


def test_two_contexts_interleaved_on_one_device(cr, oracle, synth):
    """Contexts are independent: per-context kernel set-up (shared-memory opt-in,
    occupancy), ping-pong accumulators and streams.  Two pool sets swept
    alternately must give what each gives alone, bit for bit when repeated."""
    na, nb = 3_001, 977
    A = synth.product_pools(150_007, na, seed=31)
    B = synth.product_pools(90_001, nb, seed=32)
    va, vb = synth.dual_prices(na, "wide", seed=1), synth.dual_prices(nb, "near", seed=2)
    pa = make_pools(cr, na, product=A)
    ra0 = pa.sweep(va)                       # context a fully warmed before b exists
    pb = make_pools(cr, nb, product=B)
    seen_a, seen_b = [], []
    for _ in range(3):
        seen_b.append(pb.sweep(vb))
        seen_a.append(pa.sweep(va))
    for (R, g, Ai), v, n, seen in ((A, va, na, seen_a), (B, vb, nb, seen_b)):
        D, L = oracle.sweep_product(R, g, Ai, v)
        for psi, acc in seen:
            check_psi(oracle, Ai, D, L, v, n, psi, acc, R=R, g=g)
    # materialising sweeps are per-pool bit-exact and do not disturb the other context
    pa.sweep(va, materialize=True)
    pb.sweep(vb, materialize=True)
    for p, (R, g, Ai), v in ((pa, A, va), (pb, B, vb)):
        D, L = oracle.sweep_product(R, g, Ai, v)
        Dg, Lg = p.trades()
        assert np.array_equal(Dg, D) and np.array_equal(Lg, L)
    assert np.all(np.isfinite(ra0[0]))
    pa.close()
    pb.close()


def test_profile_per_launch_times(cr, synth):
    """cfmm_profile_read_times: the individual event-bracketed durations add up to
    cfmm_profile_read's total, one per armed launch of that pool type."""
    n = 500
    p = make_pools(cr, n, product=synth.product_pools(40_000, n, seed=5),
                   geomean=synth.geomean_pools(10_000, n, seed=6))
    v = synth.dual_prices(n, "near")
    p.set_option("profile", 8)          # 4 sweeps x (product kernel + geomean kernel)
    for _ in range(5):                   # the 5th sweep is past the armed window
        p.sweep(v)
    for t in (0, 1):
        total, cnt = p.profile_read(t)
        times = p.profile_times(t)
        assert cnt == 4 and times.shape == (4,) and np.all(times > 0)
        assert abs(float(times.astype(np.float64).sum()) - total) <= 1e-6 * total
    assert p.profile_times(2).shape == (0,)
    p.set_option("profile", 0)
    p.close()


def test_comm_attach_twice_is_refused(cr):
    """Exchange epochs restart at attach, so a second attach over used receive
    areas is an error (detach + export + attach is the way to re-join)."""
    import ctypes as C
    from cfmmrouter_b200 import _lib
    p = cr.DevicePools(4)
    p.add_product([[10.0, 20.0]], [0.997], [[1, 3]])
    p.finalize()
    buf = (C.c_ubyte * _lib.COMM_HANDLE_BYTES)()
    p._chk(p._lib.cfmm_comm_export(p._ctx, buf))
    p._chk(p._lib.cfmm_comm_attach(p._ctx, 1, 0, bytes(buf)))      # world of one: no exchange
    psi, acc = p.sweep(np.array([1.0, 1.0, 3.0, 1.0]))
    assert np.isfinite(acc) and psi[1] == 0.0 and psi[3] == 0.0
    with pytest.raises(cr.CFMMError) as e:
        p._chk(p._lib.cfmm_comm_attach(p._ctx, 1, 0, bytes(buf)))
    assert e.value.code == -5 and "already attached" in e.value.message
    p._chk(p._lib.cfmm_comm_detach(p._ctx))
    p._chk(p._lib.cfmm_comm_export(p._ctx, buf))
    p._chk(p._lib.cfmm_comm_attach(p._ctx, 1, 0, bytes(buf)))
    p.close()


def test_update_reserves(cr, oracle, synth):
    n = 20
    R, g, Ai = synth.product_pools(1000, n, seed=11)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, product=(R, g, Ai))
    R2 = R.copy()
    R2[100:400] *= 1.5
    p.update_reserves(0, 100, R2[100:400])
    p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_product(R2, g, Ai, v)
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    p.close()


def test_apply_trades_on_device(cr, oracle, synth):
    """cfmm_apply_trades: R <- R + γΔ − Λ on the device, bit-identical to the same
    numpy expression; the next sweep sees the new reserves (both kernels)."""
    n = 6_000
    R, g, Ai = synth.product_pools(80_000, n, seed=41)
    Rg, gg, Ag, wg = synth.geomean_pools(20_000, n, seed=42)
    v = synth.dual_prices(n, "wide")
    p = make_pools(cr, n, product=(R, g, Ai), geomean=(Rg, gg, Ag, wg))
    with pytest.raises(cr.CFMMError):
        p.apply_trades()  # nothing materialised yet
    p.sweep(v, materialize=True)
    D, L = p.trades()
    p.apply_trades()
    R2 = R + g[:, None] * D[:80_000] - L[:80_000]
    Rg2 = Rg + gg[:, None] * D[80_000:] - L[80_000:]
    v2 = synth.dual_prices(n, "near")
    p.sweep(v2, materialize=True)
    Dn, Ln = p.trades()
    Do, Lo = oracle.sweep_product(R2, g, Ai, v2, threads=8)
    assert np.array_equal(Dn[:80_000], Do) and np.array_equal(Ln[:80_000], Lo)
    Dg, Lg = oracle.sweep_geomean(Rg2, gg, Ag, wg, v2, threads=8)
    tol = 1e-12 * (np.max(Rg2, axis=1) / gg)[:, None]
    assert np.all(np.abs(Dn[80_000:] - Dg) <= tol) and np.all(np.abs(Ln[80_000:] - Lg) <= tol)
    psi, acc = p.sweep(v2)
    check_psi(oracle, np.concatenate([Ai, Ag]), Dn, Ln, v2, n, psi, acc,
              R=np.concatenate([R2, Rg2]), g=np.concatenate([g, gg]))
    # after trading to the no-arbitrage point at v, the pools do not trade at v again
    # (fee-less pools would be exactly at their no-trade boundary; with fees: inside the band)
    p2 = make_pools(cr, n, product=(R[g < 1], g[g < 1], Ai[g < 1]))
    p2.sweep(v, materialize=True)
    p2.apply_trades()
    p2.sweep(v, materialize=True)
    D3, L3 = p2.trades()
    assert np.all(D3 <= 1e-9 * R[g < 1]) and np.all(L3 <= 1e-9 * R[g < 1])
    p.close()
    p2.close()


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_operation_sequences(cr, oracle, synth, seed):
    """State-machine fuzz: random sequences of gradient-only / materialising
    sweeps at changing ν, reserve pushes, on-device trade application and option
    toggles; after every step Ψ, acc (and trades, when materialised) are checked
    against the oracle run on a host mirror of the pool state."""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(40, 9000))
    mp_, mg_ = int(rng.integers(1, 60_000)), int(rng.integers(0, 8_000))
    R, g, Ai = synth.product_pools(mp_, n, seed=100 + seed)
    Rg, gg, Ag, wg = synth.geomean_pools(max(mg_, 1), n, seed=200 + seed)
    if mg_ == 0:
        Rg, gg, Ag, wg = Rg[:0], gg[:0], Ag[:0], wg[:0]
    p = cr.DevicePools(n)
    p.set_option("tma_variant", int(rng.choice([0, 0, 0, -1])))
    p.add_product(R, g, Ai)
    if mg_:
        p.add_geomean(Rg, gg, Ag, wg)
    p.finalize()
    R, Rg = R.copy(), Rg.copy()
    A = np.concatenate([Ai, Ag])
    last_mat = None

    def reference(v):
        D1, L1 = oracle.sweep_product(R, g, Ai, v, threads=8)
        if mg_:
            D2, L2 = oracle.sweep_geomean(Rg, gg, Ag, wg, v, threads=8)
            return np.concatenate([D1, D2]), np.concatenate([L1, L2])
        return D1, L1

    for step in range(14):
        op = rng.choice(["grad", "grad", "mat", "push", "apply", "toggle"])
        v = synth.dual_prices(n, str(rng.choice(["near", "wide", "ones"])), seed=int(rng.integers(1 << 30)))
        if op == "grad":
            psi, acc = p.sweep(v)
            Do, Lo = reference(v)
            check_psi(oracle, A, Do, Lo, v, n, psi, acc, R=np.concatenate([R, Rg]) * 64, g=np.concatenate([g, gg]))
        elif op == "mat":
            psi, acc = p.sweep(v, materialize=True)
            D, L = p.trades()
            Do, Lo = reference(v)
            assert np.array_equal(D[:mp_], Do[:mp_]) and np.array_equal(L[:mp_], Lo[:mp_])
            if mg_:
                tol = 1e-12 * (np.max(Rg, axis=1) / gg)[:, None]
                assert np.all(np.abs(D[mp_:] - Do[mp_:]) <= tol) and np.all(np.abs(L[mp_:] - Lo[mp_:]) <= tol)
            check_psi(oracle, A, D, L, v, n, psi, acc)
            last_mat = (D, L)
        elif op == "push":
            lo = int(rng.integers(0, mp_))
            hi = int(rng.integers(lo, mp_)) + 1
            R[lo:hi] *= rng.uniform(0.5, 1.5, size=(hi - lo, 1))
            p.update_reserves(0, lo, R[lo:hi])
            last_mat = None
        elif op == "apply" and last_mat is not None:
            D, L = last_mat
            p.apply_trades()
            R = R + g[:, None] * D[:mp_] - L[:mp_]
            if mg_:
                Rg = Rg + gg[:, None] * D[mp_:] - L[mp_:]
            last_mat = None
        elif op == "toggle":
            p.set_option(str(rng.choice(["gradient_math", "use_tma", "psi_fixed_point"])), int(rng.integers(0, 2)))
    p.close()


def test_nan_propagates_like_julia_max(cr, oracle):
    # Julia's max(x, 0) propagates NaN (CUDA fmax would not)
    R = np.array([[np.nan, 1.0], [1.0, 2.0]])
    g = np.array([1.0, 1.0])
    Ai = np.array([[1, 2], [2, 3]])
    v = np.array([1.0, 2.0, 3.0])
    p = make_pools(cr, 3, product=(R, g, Ai))
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_product(R, g, Ai, v)
    assert np.array_equal(np.isnan(D), np.isnan(Do)) and np.isnan(D[0]).all()
    assert np.array_equal(D[1], Do[1]) and np.array_equal(L[1], Lo[1])
    assert np.isnan(psi[0]) and np.isnan(acc)
    p.close()


# ---------------------------------------------------------------------------
# BASELINE-size properties
# ---------------------------------------------------------------------------

def test_full_size_config5_10M_pools(cr, oracle, synth):
    """configs[4] on one GPU: 10M ProductTwoCoin pools, 50k tokens.  The C
    oracle still finishes in seconds, so this is a direct per-pool parity check
    at full size, plus conservation properties of Ψ."""
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n)
    v = synth.dual_prices(n, "near")
    p = make_pools(cr, n, product=(R, g, Ai))
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=oracle.max_threads())
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    # idempotence: a second sweep at the same ν reproduces Ψ to rounding
    psi2, acc2 = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi2, acc2, R=R, g=g)
    p.set_option("gradient_math", 0)
    psi3, acc3 = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi3, acc3, Rq=R)
    # invariant: every pool's trade keeps ϕ(R+γΔ−Λ) ≥ ϕ(R) − sqrt(eps) (test/arb.jl:11)
    Rp = R + g[:, None] * D - L
    assert np.all(Rp[:, 0] * Rp[:, 1] >= R[:, 0] * R[:, 1] - np.sqrt(np.finfo(float).eps))
    p.close()


def test_config3_mixed_1M(cr, oracle, synth):
    """configs[2]: 500k ProductTwoCoin + 500k GeometricMeanTwoCoin, 10k tokens."""
    n = 10_000
    Rp, gp, Ap = synth.product_pools(500_000, n)
    Rg, gg, Ag, wg = synth.geomean_pools(500_000, n)
    v = synth.dual_prices(n, "near")
    p = make_pools(cr, n, product=(Rp, gp, Ap), geomean=(Rg, gg, Ag, wg))
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    D1, L1 = oracle.sweep_product(Rp, gp, Ap, v, threads=8)
    D2, L2 = oracle.sweep_geomean(Rg, gg, Ag, wg, v, threads=8)
    assert np.array_equal(D[:500_000], D1) and np.array_equal(L[:500_000], L1)
    tol = 1e-12 * (np.max(Rg, axis=1) / gg)[:, None]
    assert np.all(np.abs(D[500_000:] - D2) <= tol) and np.all(np.abs(L[500_000:] - L2) <= tol)
    check_psi(oracle, np.concatenate([Ap, Ag]), D, L, v, n, psi, acc)
    p.close()


def test_config4_univ3_500k(cr, oracle, synth):
    """configs[3]: 500k UniV3 pools (examples/Univ3.jl shape), 5k tokens."""
    n = 5_000
    cp, g, Ai, off, lt, lq = synth.univ3_pools(500_000, n)
    rng = np.random.default_rng(3)
    v = np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n))
    p = make_pools(cr, n, univ3=(cp, g, Ai, off, lt, lq))
    psi, acc = p.sweep(v, materialize=True)
    D, L = p.trades()
    Do, Lo = oracle.sweep_univ3(cp, g, Ai, off, lt, lq, v, threads=8)
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    p.close()


# ---------------------------------------------------------------------------
# route! end to end (test/arb.jl, test/swap.jl)
# ---------------------------------------------------------------------------

TOL = 1e-4


def check_primal_feasibility(cr, r, arb=True):
    # test/arb.jl:5-23
    flows = np.zeros_like(r.v)
    for D, L, c in zip(r.Δs, r.Λs, r.cfmms):
        assert np.all(D >= -TOL) and np.all(L >= -TOL)
        assert c.phi(c.R + c.gamma * D - L) >= c.phi() - np.sqrt(np.finfo(float).eps)
        flows[c.Ai - 1] += L - D
    assert np.array_equal(flows, cr.netflows(r))
    if arb:
        assert np.all(flows >= -TOL)
    else:
        assert np.sum(flows >= -TOL) == 1


def check_dual_feasibility(r):
    # test/arb.jl:25-28
    assert np.all(r.v >= r.objective.lower_limit() - TOL)
    assert np.all(r.v <= r.objective.upper_limit() + TOL)


def test_route_readme_quickstart(cr):
    # configs[0]: README quick-start / test/arb.jl:42-58
    # README.md:25-39
    pools = [cr.ProductTwoCoin([1e6, 1e6], 1, [1, 2]), cr.ProductTwoCoin([1e3, 2e3], 1, [1, 2])]
    r = cr.Router(cr.LinearNonnegative(np.ones(2)), pools, 2)
    cr.route(r)
    psi = cr.netflows(r)
    # (the absolute ϕ slack of test/arb.jl:11 is only meaningful for the small
    # pools that test uses; with R = 1e6 one ulp of ϕ is already 1e-4)
    assert np.all(r.Δs >= -TOL) and np.all(r.Λs >= -TOL) and np.all(psi >= -TOL)
    check_dual_feasibility(r)
    assert abs(psi[1] - 171.40) < 0.05 and abs(psi[0]) < 1e-3  # SURVEY App. B


def test_route_simple_and_random_markets(cr):
    # test/arb.jl:42-58: pools appended after construction are ignored
    eq, sm = cr.ProductTwoCoin([100, 100], 1, [1, 2]), cr.ProductTwoCoin([1, 2], 1, [1, 2])
    r = cr.Router(cr.LinearNonnegative(np.ones(2)), [eq, sm], 2)
    r.cfmms += [eq, sm]
    cr.route(r)
    check_primal_feasibility(cr, r)
    check_dual_feasibility(r)
    # test/arb.jl:60-85
    rng = np.random.default_rng(1234)
    pools = []
    for _ in range(100):
        Ai = rng.choice(np.arange(1, 11), size=2, replace=False)
        pools.append(cr.ProductTwoCoin(1000 * rng.random(2), 1.0, Ai))
    r = cr.Router(cr.LinearNonnegative(rng.random(10) + 1e-3), pools, 10)
    cr.route(r)
    check_primal_feasibility(cr, r)
    check_dual_feasibility(r)


def test_route_swap_markets(cr):
    # test/swap.jl:2-46
    eq, sm = cr.ProductTwoCoin([100, 100], 1, [1, 2]), cr.ProductTwoCoin([1, 2], 1, [1, 2])
    r = cr.Router(cr.BasketLiquidation(1, [5.0, 0.0]), [eq, sm], 2)
    cr.route(r)
    check_primal_feasibility(cr, r)
    check_dual_feasibility(r)
    rng = np.random.default_rng(1234)
    pools = []
    for _ in range(100):
        Ai = rng.choice(np.arange(1, 11), size=2, replace=False)
        pools.append(cr.ProductTwoCoin(1000 * rng.random(2), 1.0, Ai))
    delta_in = np.concatenate([[0.0], 100 * rng.random(9)])
    r = cr.Router(cr.BasketLiquidation(1, delta_in), pools, 10)
    cr.route(r)
    check_primal_feasibility(cr, r, arb=False)
    check_dual_feasibility(r)
