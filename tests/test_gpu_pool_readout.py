"""Per-pool checks of the gradient-only sweeps, read out through Ψ on token-disjoint pool sets.

In a token-disjoint set (pool i holds tokens 2i+1 and 2i+2, nobody else does) Ψ[2i+1] and
Ψ[2i+2] of a gradient-only sweep are pool i's own Λ−Δ: no summation order is involved, so
the per-pool results of the kernels that route! runs on every evaluation can be checked
directly, most of them bit for bit:
  * reference operation order (ProductTwoCoin, UniV3): Ψ == the oracle's L−D exactly;
  * fixed-point Ψ[b] slice: for one pool S_b = R2, so the kernel's quantum 2^(e−54) with
    e = ilogb(R2·(1+2^-30)) + 1 is known on the host, and Ψ[b] == rint(flow / quantum)·quantum
    exactly (the flow itself when |flow| > 256·R2: the fp64 RED fallback);
  * compact (20-byte) and wide (32-byte) ProductTwoCoin streams: identical Ψ;
  * economized math: |Ψ − truth| <= C·eps·(R + γ|truth|)/γ (+ half a quantum), with the truth
    from the reference closed forms (src/cfmms.jl:125-126, :180-181) in extended precision.
The host reference and the quantisation predictor have CPU tests of their own here.
"""
import itertools
import json
import os

import numpy as np
import pytest

from test_layout import layout

LD = np.longdouble
EPS = np.finfo(np.float64).eps

# Per-pool error bounds, as multiples of eps·(R + γ|flow|)/γ of the pool's own token
# (R = its reserve of that token).  Measured on an H100 80GB HBM3 (700 W) over this file's sets:
#   ProductTwoCoin economized (rsqrt form): 2.05; reference order: 2.02 (= the oracle, bit for bit).
#   GeometricMean: the error grows with the size of the exponent of the power (see
#   geomean_log_exponent), so the bound is C + 2·|e·log2 t|.  Pools the economized form takes
#   (geomean_economized) are held to C_GEOMEAN_ECON: their largest excess over 2·|e·log2 t| is 1.4
#   for the exp2/log2 power.  Pools that run the reference's own four-pow forms (reference order,
#   exact = 1, and the economized sweeps' fallback outside the certified range or inside the tie
#   margin) are held to C_GEOMEAN: largest excess 16.2 (CUDA pow; glibc pow in the oracle
#   measures the same).  Largest totals: 38.4 (exp2/log2), 19.2 (economized pow), 16.7
#   (reference forms).
C_PRODUCT_ECON = 4.0
C_GEOMEAN_ECON = 4.0
C_GEOMEAN = 24.0


# ---------------------------------------------------------------------------
# host reference: the reference closed forms in extended precision
# ---------------------------------------------------------------------------

def _ld(*xs):
    assert np.finfo(LD).nmant >= 63, "the reference needs an x87 80-bit (or wider) long double"
    return [np.asarray(x, dtype=np.float64).astype(LD) for x in xs]


def product_truth(R, g, va, vb):
    """(Λ1−Δ1, Λ2−Δ2) of ProductTwoCoin pools, src/cfmms.jl:125-126 and :130-140, evaluated in
    long double from the exact fp64 inputs."""
    R1, R2, g, v1, v2 = _ld(R[:, 0], R[:, 1], g, va, vb)
    k = R1 * R2
    m21, m12 = v2 / v1, v1 / v2
    zero = LD(0)
    d1 = np.maximum(np.sqrt(g * m21 * k) - R1, zero) / g
    d2 = np.maximum(np.sqrt(g * m12 * k) - R2, zero) / g
    l1 = np.maximum(R1 - np.sqrt(k / (m12 * g)), zero)
    l2 = np.maximum(R2 - np.sqrt(k / (m21 * g)), zero)
    return l1 - d1, l2 - d2


def geomean_truth(R, w, g, va, vb):
    """(Λ1−Δ1, Λ2−Δ2) of GeometricMeanTwoCoin pools, src/cfmms.jl:180-181 and :185-196, in long
    double from the exact fp64 inputs."""
    R1, R2, w1, w2, g, v1, v2 = _ld(R[:, 0], R[:, 1], w[:, 0], w[:, 1], g, va, vb)
    one, zero = LD(1), LD(0)
    eta = w1 / w2

    def delta(m, r1, r2, e):
        return np.maximum((g * m * e * r1 * r2 ** e) ** (one / (e + one)) - r2, zero) / g

    def lam(m, r1, r2, e):
        return np.maximum(r1 - ((r2 * r1 ** (one / e)) / (e * g * m)) ** (e / (one + e)), zero)

    m21, m12 = v2 / v1, v1 / v2
    d1 = delta(m21, R2, R1, eta)
    d2 = delta(m12, R1, R2, one / eta)
    l1 = lam(m12, R1, R2, one / eta)
    l2 = lam(m21, R2, R1, eta)
    return l1 - d1, l2 - d2


def geomean_log_exponent(R, w, g, va, vb):
    """|e·log2 t| of the economized GeometricMean power u = t^e (t = γ·uB/uA or γ·uA/uB > 1, e the
    received token's weight share).  The power is taken as exp2(e·log2 t); the absolute rounding
    error of that exponent grows with its size, and u inherits it as a relative error: about
    ln2·(1 + 1/2 + 1)·eps·|e·log2 t| for log2 (1 ulp), the product (1/2 ulp) and e itself (1 ulp).
    The bounds of the GeometricMean paths are therefore C + 2·|e·log2 t| error units."""
    uA = (np.asarray(va) * w[:, 1]) * R[:, 0]
    uB = (np.asarray(vb) * w[:, 0]) * R[:, 1]
    lt = np.log2(g * uB / uA)
    e = np.where(lt > 0, w[:, 1], w[:, 0]) / (w[:, 0] + w[:, 1])
    return np.abs(e * lt)


def geomean_economized(R, w, g, va, vb, kernel):
    """Per pool: does the economized GeometricMean form run, or the reference's forms?  The
    side and range test of the TMA kernel (product_tma.cuh, POOL = 1) or of the first-generation
    kernel (geomean_arb_econ, arb_math.cuh), with the same IEEE products in the same order."""
    geo = lambda x: (x >= 2.0 ** -32) & (x < 2.0 ** 32)
    R1, R2, w1, w2 = R[:, 0], R[:, 1], w[:, 0], w[:, 1]
    va, vb = np.asarray(va), np.asarray(vb)
    uA = (va * w2) * R1
    uB = (vb * w1) * R2
    tA, tB = g * uB, g * uA
    lo, hi = 1.0 - 2.0 ** -30, 1.0 + 2.0 ** -30
    zA, zB = tA < uA * lo, tB < uB * lo
    fA, fB = (tA > uA * hi) & zB, (tB > uB * hi) & zA
    if kernel == "tma":
        sane = geo(uA) & geo(uB) & (va >= 2.0 ** -100) & (va < 2.0 ** 101) & (w1 < 24.0 * w2) & \
            (w2 < 24.0 * w1) & (g <= 1.0) & geo(g)
    else:
        eta = w1 / w2
        sane = geo(R1) & geo(R2) & geo(va) & geo(vb) & geo(g) & (eta > 1.0 / 24.0) & (eta < 24.0)
    return sane & (fA | fB)


def fixed_exponent(R2):
    """e of the kernel's fixed-point scale for a token whose pools' total reserve is R2
    (token_scale_kernel): e = ilogb(R2·(1 + 2^-30)) + 1, quantum 2^(e−54)."""
    _, e = np.frexp(np.asarray(R2, dtype=np.float64) * (1.0 + 2.0 ** -30))
    return e.astype(np.int64)          # frexp's exponent is ilogb + 1


def quantise_b(fb, R2):
    """Ψ[b] of a one-pool token on the fixed-point slice: the flow rounded to the nearest
    multiple of the quantum (ties to even, __double2ll_rn), or the flow itself when
    |flow| > 256·R2 (the fp64 RED fallback; NaN too)."""
    fb = np.asarray(fb, dtype=np.float64)
    e = fixed_exponent(R2)
    q = np.ldexp(np.rint(np.ldexp(fb, 54 - e)), e - 54)
    return np.where(np.abs(fb) <= 256.0 * np.asarray(R2), q, fb)


def half_quantum(R2):
    return np.ldexp(1.0, fixed_exponent(R2) - 55)


def error_units(psi, truth, R, g):
    """|Ψ − truth| in units of eps·(R + γ|truth|)/γ."""
    t = truth.astype(np.float64)
    unit = EPS * (np.asarray(R) + g * np.abs(t)) / g
    return np.abs((psi.astype(LD) - truth).astype(np.float64)) / unit


# ---------------------------------------------------------------------------
# CPU tests of the reference and the predictor
# ---------------------------------------------------------------------------

def test_reference_matches_golden_vectors():
    """The long-double closed forms against the 40-digit golden vectors (tests/golden)."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "closed_forms.json")) as f:
        gold = json.load(f)
    for kind in ("product", "geomean"):
        for case in gold[kind]:
            R = np.array([case["R"]], dtype=float)
            g = np.array([case["gamma"]])
            v = case["v"]
            if kind == "product":
                fa, fb = product_truth(R, g, [v[0]], [v[1]])
            else:
                fa, fb = geomean_truth(R, np.array([case["w"]], dtype=float), g, [v[0]], [v[1]])
            for flow, k in ((fa[0], 0), (fb[0], 1)):
                want = LD(case["Lambda"][k]) - LD(case["Delta"][k])
                scale = LD(max(case["R"])) / LD(min(case["gamma"], 1.0)) + abs(want)
                assert abs(flow - want) <= LD(2.0 ** -58) * scale, (kind, case, flow, want)


def test_reference_against_mpmath():
    """A few hundred pools of the adversarial generators: long double against 50-digit
    arithmetic, to 1/64 of the error unit the GPU bounds are stated in."""
    mpmath = pytest.importorskip("mpmath")
    from cfmmrouter_b200 import synth
    mp = mpmath.mp
    mp.dps = 50
    R, g, Ai, v = synth.disjoint_product(300, seed=3)
    fa, fb = product_truth(R, g, v[0::2], v[1::2])
    Rg, gg, Ag, w, vg = synth.disjoint_geomean(300, seed=4)
    ga, gb = geomean_truth(Rg, w, gg, vg[0::2], vg[1::2])
    for i in range(300):
        R1, R2, G, v1, v2 = (mp.mpf(float(x)) for x in (R[i, 0], R[i, 1], g[i], v[2 * i], v[2 * i + 1]))
        k = R1 * R2
        d1 = max(mp.sqrt(G * (v2 / v1) * k) - R1, 0) / G
        d2 = max(mp.sqrt(G * (v1 / v2) * k) - R2, 0) / G
        l1 = max(R1 - mp.sqrt(k / ((v1 / v2) * G)), 0)
        l2 = max(R2 - mp.sqrt(k / ((v2 / v1) * G)), 0)
        for got, want, r in ((fa[i], l1 - d1, R1), (fb[i], l2 - d2, R2)):
            unit = (r + G * abs(want)) / G * mp.mpf(EPS)
            assert abs(mp.mpf(str(got)) - want) <= unit / 64, (i, got, want)
        R1, R2, G, v1, v2, w1, w2 = (mp.mpf(float(x)) for x in
                                     (Rg[i, 0], Rg[i, 1], gg[i], vg[2 * i], vg[2 * i + 1], w[i, 0], w[i, 1]))
        eta = w1 / w2

        def delta(m, r1, r2, e):
            return max((G * m * e * r1 * r2 ** e) ** (1 / (e + 1)) - r2, 0) / G

        def lam(m, r1, r2, e):
            return max(r1 - ((r2 * r1 ** (1 / e)) / (e * G * m)) ** (e / (1 + e)), 0)

        ta = lam(v1 / v2, R1, R2, 1 / eta) - delta(v2 / v1, R2, R1, eta)
        tb = lam(v2 / v1, R2, R1, eta) - delta(v1 / v2, R1, R2, 1 / eta)
        for got, want, r in ((ga[i], ta, R1), (gb[i], tb, R2)):
            unit = (r + G * abs(want)) / G * mp.mpf(EPS)
            assert abs(mp.mpf(str(got)) - want) <= unit / 64, (i, got, want)


def test_quantisation_predictor():
    # the scale exponent: ceil(log2 S) with the 2^-30 slack (powers of two, and totals within
    # 2^-30 below one, go one up)
    R2 = np.array([1.0, 3.0, 2.0 ** -100, 2.0 ** 100, 1.5 * 2.0 ** 40, 2.0 - 2.0 ** -40, 2.0 - 2.0 ** -20])
    assert fixed_exponent(R2).tolist() == [1, 2, -99, 101, 41, 2, 1]
    # R2 = 1: quantum 2^-53; ties round to even; results are multiples of the quantum
    q = 2.0 ** -53
    fb = np.array([2.5 * q, 3.5 * q, -2.5 * q, 1.0 / 3.0, -0.7, 256.0, 256.0 + 2.0 ** -44, -300.0, np.nan])
    out = quantise_b(fb, np.ones_like(fb))
    assert out[:3].tolist() == [2 * q, 4 * q, -2 * q]
    assert out[3] == np.rint((1.0 / 3.0) / q) * q and out[4] == np.rint(-0.7 / q) * q
    assert out[5] == 256.0                                   # |flow| <= 256 R2: the integer slice
    assert out[6] == fb[6] and out[7] == -300.0 and np.isnan(out[8])  # beyond: the flow itself
    rng = np.random.default_rng(0)
    R2 = np.exp2(rng.uniform(-100, 100, size=10_000))
    fb = R2 * rng.uniform(-256, 256, size=10_000)
    out = quantise_b(fb, R2)
    quantum = np.ldexp(1.0, fixed_exponent(R2) - 54)
    assert np.all(np.abs(out - fb) <= quantum / 2)
    assert np.all(np.mod(out / quantum, 1.0) == 0.0)
    assert np.all(quantum <= R2 * 2.0 ** -53) and np.all(quantum > R2 * 2.0 ** -55)


def test_disjoint_generators():
    from cfmmrouter_b200 import synth
    R, g, Ai, v = synth.disjoint_product(5000, seed=1)
    assert np.array_equal(np.sort(Ai.ravel()), np.arange(1, 10_001)) and len(v) == 10_000
    assert fast_range_ok(R, g) and len(np.unique(g)) == 256 and 1.0 in g
    Rg, gg, Ag, w, vg = synth.disjoint_geomean(2000, seed=2)
    assert np.array_equal(np.sort(Ag.ravel()), np.arange(1, 4001)) and np.all(Rg > 0) and np.all(w > 0)
    cp, gu, Au, off, lt, lq, vu = synth.disjoint_univ3(200, seed=3, ragged=True)
    assert off[-1] == len(lt) == len(lq) and np.any(np.diff(off) == 1)
    for i in range(200):
        t = lt[off[i]:off[i + 1]]
        assert t[0] >= cp[i] and np.all(np.diff(t) < 0)


# ---------------------------------------------------------------------------
# helpers of the GPU tests
# ---------------------------------------------------------------------------

def fast_range_ok(R, g):
    """The host's pools_in_range rule (fast_range_ok in cfmm_capi.cu): every reserve and fee in
    [2^-100, 2^100], γ <= 1.  It is set-wide: one pool outside sends the whole set to the generic
    path.  (The device's per-value test, in_fast_range, admits [2^-100, 2^101); the host rule is
    the narrower one.)"""
    x = np.concatenate([np.ravel(R), np.ravel(g)])
    return bool(np.all((x >= 2.0 ** -100) & (x <= 2.0 ** 100)) and np.all(np.asarray(g) <= 1.0))


def max_chunk_span(lay, Ai):
    """Largest first-token span of a 96-pool chunk of the device order (compact stream: <= 8191)."""
    order = lay["order"].reshape(-1, 96)
    a = np.asarray(Ai)[:, 0]
    span = 0
    for row in order:
        r = row[row >= 0]
        if len(r):
            span = max(span, int(a[r[-1]] - a[r[0]]))
    return span


def make(cr, n, pre=None, product=None, geomean=None, univ3=None):
    p = cr.DevicePools(n)
    p.set_option("orient_by_degree", 0)
    for k, val in (pre or {}).items():
        p.set_option(k, val)
    if product is not None:
        p.add_product(*product)
    if geomean is not None:
        p.add_geomean(*geomean)
    if univ3 is not None:
        p.add_univ3(*univ3)
    p.finalize()
    return p


def set_options(p, **opts):
    for k, val in opts.items():
        p.set_option(k, int(val))


def check_acc(acc, v, truth_a, truth_b, slack_a=0.0, slack_b=0.0):
    """acc = Σ ν·Ψ over the pools, summed across CTAs in varying order."""
    va, vb = v[0::2].astype(LD), v[1::2].astype(LD)
    ref = float(np.sum(va * truth_a + vb * truth_b))
    scale = float(np.sum(np.abs(va * truth_a) + np.abs(vb * truth_b)))
    slack = float(np.sum(v[0::2] * slack_a + v[1::2] * slack_b))
    assert abs(acc - ref) <= 1e-12 * scale + slack + 1e-300, (acc, ref, scale, slack)


def assert_same(got, want, what):
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not bad.any(), (what, np.argwhere(bad)[:5].ravel(), got[bad][:5], want[bad][:5])


MEASURED = {}


def record(key, units):
    """Largest error seen per path (printed with -s; DESIGN §4 quotes them)."""
    if len(units):
        MEASURED[key] = max(MEASURED.get(key, 0.0), float(np.max(units)))
        print(f"[measured] {key}: max {MEASURED[key]:.3f}")


# ---------------------------------------------------------------------------
# ProductTwoCoin
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("variant", [0, -1])
@pytest.mark.parametrize("m", [1, 95, 96, 97, 5_000, 100_003, 400_000])
def test_product_reference_order_per_pool(cr, oracle, synth, m, variant):
    """gradient_math = 0: every kernel, slice and grid shape gives the oracle's Λ−Δ per pool, bit
    for bit (quantised on the fixed-point slice of the TMA kernel)."""
    R, g, Ai, v = synth.disjoint_product(m, seed=m)
    n = 2 * m
    assert fast_range_ok(R, g)
    lay = layout(cr, n, Ai, orient=0, variant=variant)
    assert lay["bucketed"] == (variant == 0)
    if variant == 0 and m == 400_000:
        assert 450 <= lay["tile_bucket"][-1] + 1 <= 640       # near the 640-entry bucket table
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    fa, fb = Lo[:, 0] - Do[:, 0], Lo[:, 1] - Do[:, 1]
    qb = quantise_b(fb, R[:, 1])
    p = make(cr, n, pre={"tma_variant": variant}, product=(R, g, Ai))
    p.set_option("gradient_math", 0)
    for per_sm, fixed, tma, exact in itertools.product((0, 1), (0, 1), (0, 1), (0, 1)):
        set_options(p, blocks_per_sm=per_sm, psi_fixed_point=fixed, use_tma=tma, exact=exact)
        psi, acc = p.sweep(v)
        on_slice = variant == 0 and tma and fixed
        what = dict(per_sm=per_sm, fixed=fixed, tma=tma, exact=exact)
        assert_same(psi[0::2], fa, what)
        assert_same(psi[1::2], qb if on_slice else fb, what)
        check_acc(acc, v, fa.astype(LD), fb.astype(LD))
    p.close()


def generic_buckets(v, R2, nb, fixed):
    """Per pool: does the TMA kernel run its bucket in the generic (reference-order) form?  It does
    when any price of the bucket's slice lies outside [2^-100, 2^101).  On the fixed-point slice the
    slice holds ν_b·2^(e_b−54) (e_b: the token's scale exponent), so a bucket with a very small (or
    very large) second reserve goes generic there and not on the fp64 slice."""
    n = len(v)
    x = np.array(v, dtype=np.float64)
    if fixed:
        x[1::2] = np.ldexp(x[1::2], fixed_exponent(R2) - 54)
    bad = ~((x >= 2.0 ** -100) & (x < 2.0 ** 101))
    bad_bucket = np.zeros(-(-n // nb), dtype=bool)
    np.logical_or.at(bad_bucket, np.arange(n) // nb, bad)
    return bad_bucket[np.arange(1, n, 2) // nb]      # b = 2i+2 (1-based): 0-based index 2i+1


def _nu_out_of_range(v, lay, m):
    """ν of one b-token of bucket 1 at 2^-110 (that bucket's slice leaves the guard-free range:
    the whole bucket takes the generic form, its neighbours do not) and ν of one a-token at
    2^105 (that pool alone takes it)."""
    nb = lay["nb"]
    b_tok = nb + 1 + (nb + 1) % 2            # an even 1-based token (a b) in bucket 1
    v[b_tok - 1] = 2.0 ** -110
    v[2 * (m // 3)] = 2.0 ** 105
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("m", [97, 5_000, 100_003, 400_000])
def test_product_economized_per_pool(cr, oracle, synth, m):
    """gradient_math = 1: the rsqrt form within C·eps·(R + γ|flow|)/γ of the truth per pool;
    compact and wide streams bit-identical; the fixed-point slice equals the fp64 slice
    quantised; the first-generation kernel stays in reference order."""
    R, g, Ai, v = synth.disjoint_product(m, seed=m + 1)
    n = 2 * m
    lay = layout(cr, n, Ai, orient=0)
    assert lay["bucketed"] and fast_range_ok(R, g)
    assert max_chunk_span(lay, Ai) <= 8191 and len(np.unique(g)) <= 256   # compact stream eligible
    if m >= 5_000:
        assert lay["tile_bucket"][-1] >= 2
        v = _nu_out_of_range(v, lay, m)
    fa, fb = product_truth(R, g, v[0::2], v[1::2])
    p = make(cr, n, product=(R, g, Ai))
    out = {}
    for compact, fixed in itertools.product((1, 0), (1, 0)):
        set_options(p, compact_stream=compact, psi_fixed_point=fixed)
        out[compact, fixed] = p.sweep(v)
    for fixed in (1, 0):
        assert_same(out[1, fixed][0], out[0, fixed][0], f"compact vs wide, fixed={fixed}")
    psi, acc = out[1, 0]
    psiq, accq = out[1, 1]
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    fa_o, fb_o = Lo[:, 0] - Do[:, 0], Lo[:, 1] - Do[:, 1]
    # the same path on both slices: the fixed-point Ψ is the fp64 one quantised; buckets that only
    # the fixed-point slice sends to the generic form give the reference's flows there
    gen_q = generic_buckets(v, R[:, 1], lay["nb"], fixed=True)
    gen = generic_buckets(v, R[:, 1], lay["nb"], fixed=False)
    assert not np.any(gen & ~gen_q)
    if m >= 5_000:
        assert gen.any() and not gen.all() and (~gen_q).any()
    want_a = np.where(gen_q == gen, psi[0::2], fa_o)
    want_b = quantise_b(np.where(gen_q == gen, psi[1::2], fb_o), R[:, 1])
    assert_same(psiq[0::2], want_a, "fixed vs fp64 slice, a side")
    assert_same(psiq[1::2], want_b, "fixed vs fp64 slice, b side")
    # the economized form ran: its roundings differ from the reference order's
    assert np.count_nonzero((psi[0::2] != fa_o) | (psi[1::2] != fb_o)) >= max(1, m // 100)
    ua = error_units(psi[0::2], fa, R[:, 0], g)
    ub = error_units(psi[1::2], fb, R[:, 1], g)
    record("product economized", np.concatenate([ua, ub]))
    assert np.all(ua <= C_PRODUCT_ECON), np.argsort(ua)[-5:]
    assert np.all(ub <= C_PRODUCT_ECON), np.argsort(ub)[-5:]
    hq = half_quantum(R[:, 1])
    assert np.all(np.abs(psiq[1::2] - fb.astype(np.float64)) <= C_PRODUCT_ECON * EPS * (R[:, 1] + g * np.abs(fb.astype(np.float64))) / g + hq)
    slack_a = C_PRODUCT_ECON * EPS * (R[:, 0] + g * np.abs(fa.astype(np.float64))) / g
    slack_b = C_PRODUCT_ECON * EPS * (R[:, 1] + g * np.abs(fb.astype(np.float64))) / g
    check_acc(acc, v, fa, fb, slack_a, slack_b)
    check_acc(accq, v, fa, fb, slack_a, slack_b)
    # the reference order on the same set, measured against the truth in the same units
    record("product reference order", np.concatenate([error_units(Lo[:, 0] - Do[:, 0], fa, R[:, 0], g),
                                                      error_units(Lo[:, 1] - Do[:, 1], fb, R[:, 1], g)]))
    set_options(p, use_tma=0)                       # ProductTwoCoin has no economized form there
    psi, acc = p.sweep(v)
    assert_same(psi[0::2], Lo[:, 0] - Do[:, 0], "first-generation kernel, a")
    assert_same(psi[1::2], Lo[:, 1] - Do[:, 1], "first-generation kernel, b")
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("edge", ["lo", "hi", "below", "above"])
def test_product_reserve_range_edges(cr, oracle, synth, edge):
    """Reserves at the edges of the host's range [2^-100, 2^100] stay on the fast path (a set of
    their own: the range test is set-wide), and the economized sweep really runs there; one
    reserve just outside sends the whole set to the generic form, so even the economized sweep
    then equals the reference bit for bit."""
    m = 3_000
    n = 2 * m
    rng = np.random.default_rng(11)
    _, g, Ai, v = synth.disjoint_product(m, seed=12, adversarial=False)
    v = np.exp2(rng.uniform(-4, 4, size=n))
    spread = np.exp2(rng.uniform(0, 30, size=m))
    if edge in ("lo", "below"):
        R = np.stack([np.full(m, 2.0 ** -100), 2.0 ** -100 * spread], axis=1)
    else:
        top = 2.0 ** 100
        R = np.stack([np.full(m, top), top / spread], axis=1)
    R[1::2] = R[1::2, ::-1].copy()                 # the edge reserve on either side
    if edge == "below":
        R[7, 0] = 2.0 ** -100 * (1 - 2.0 ** -53)
    if edge == "above":
        R[7, 0] = 2.0 ** 100 * (1 + 2.0 ** -52)
    assert fast_range_ok(R, g) == (edge in ("lo", "hi"))
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    fa_o, fb_o = Lo[:, 0] - Do[:, 0], Lo[:, 1] - Do[:, 1]
    fa, fb = product_truth(R, g, v[0::2], v[1::2])
    # at the 2^-100 edge the scaled prices of the fixed-point slice leave the range: generic form
    same = generic_buckets(v, R[:, 1], layout(cr, n, Ai, orient=0)["nb"], fixed=True) == \
        generic_buckets(v, R[:, 1], layout(cr, n, Ai, orient=0)["nb"], fixed=False)
    p = make(cr, n, product=(R, g, Ai))
    for gm in (0, 1):
        set_options(p, gradient_math=gm, psi_fixed_point=0)
        psi, _ = p.sweep(v)
        set_options(p, psi_fixed_point=1)
        psiq, _ = p.sweep(v)
        same_path = same | (gm == 0) | (edge in ("below", "above"))
        assert_same(psiq[0::2], np.where(same_path, psi[0::2], fa_o), f"gm={gm}: fixed vs fp64 slice, a")
        assert_same(psiq[1::2], quantise_b(np.where(same_path, psi[1::2], fb_o), R[:, 1]),
                    f"gm={gm}: fixed vs fp64 slice, b")
        if gm == 0 or edge in ("below", "above"):
            assert_same(psi[0::2], fa_o, f"gm={gm}, a")
            assert_same(psi[1::2], fb_o, f"gm={gm}, b")
        else:
            ua = error_units(psi[0::2], fa, R[:, 0], g)
            ub = error_units(psi[1::2], fb, R[:, 1], g)
            record("product economized", np.concatenate([ua, ub]))
            assert np.all(ua <= C_PRODUCT_ECON) and np.all(ub <= C_PRODUCT_ECON)
            # the economized form ran: its roundings differ from the reference order's
            differs = (psi[0::2] != fa_o) | (psi[1::2] != fb_o)
            assert np.count_nonzero(differs) >= m // 100, np.count_nonzero(differs)
    p.close()


# ---------------------------------------------------------------------------
# GeometricMeanTwoCoin
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("m", [700, 60_000])          # one b-bucket, 75 b-buckets
def test_geomean_gradient_paths_per_pool(cr, oracle, synth, m):
    """Every GeometricMean gradient path: the TMA kernel (economized exp2/log2 power and
    reference order, fixed-point and fp64 slices), the first-generation kernel (exp2/log2,
    pow, reference order) and exact = 1, each per pool against the truth."""
    R, g, Ai, w, v = synth.disjoint_geomean(m, seed=m)
    n = 2 * m
    assert fast_range_ok(R, g)
    fa, fb = geomean_truth(R, w, g, v[0::2], v[1::2])
    Do, Lo = oracle.sweep_geomean(R, g, Ai, w, v, threads=8)
    p = make(cr, n, geomean=(R, g, Ai, w))

    def run(**opts):
        base = dict(gradient_math=1, geomean_tma=1, geomean_log2=1, psi_fixed_point=1, exact=0)
        base.update(opts)
        set_options(p, **base)
        return p.sweep(v)

    L = geomean_log_exponent(R, w, g, v[0::2], v[1::2])
    # which pools each kernel's economized form takes (the rest run the reference's forms)
    econ_tma = geomean_economized(R, w, g, v[0::2], v[1::2], "tma")
    econ_gen1 = geomean_economized(R, w, g, v[0::2], v[1::2], "first-generation")
    nu_q = v.copy()
    nu_q[1::2] = np.ldexp(v[1::2], fixed_exponent(R[:, 1]) - 54)
    assert np.all((nu_q >= 2.0 ** -100) & (nu_q < 2.0 ** 101))    # no bucket leaves the fast form
    for econ in (econ_tma, econ_gen1):
        assert np.count_nonzero(econ) >= 0.8 * m and np.count_nonzero(~econ) >= 20
    none = np.zeros(m, dtype=bool)

    def within(psi, econ, key):
        u = np.maximum(error_units(psi[0::2], fa, R[:, 0], g), error_units(psi[1::2], fb, R[:, 1], g))
        record(key, u)
        record(key + ", economized pools beyond 2·|e·log2 t|", (u - 2 * L)[econ])
        record(key + ", reference-form pools beyond 2·|e·log2 t|", (u - 2 * L)[~econ])
        bound = np.where(econ, C_GEOMEAN_ECON, C_GEOMEAN) + 2 * L
        assert np.all(u <= bound), (key, np.argsort(u - bound)[-5:], np.sort(u - bound)[-5:])

    def near_oracle(psi):
        tol = 1e-12 * np.max(R, axis=1) / g
        assert np.all(np.abs(psi[0::2] - (Lo[:, 0] - Do[:, 0])) <= tol)
        assert np.all(np.abs(psi[1::2] - (Lo[:, 1] - Do[:, 1])) <= tol)

    # TMA kernel: the fixed-point slice is the fp64 slice quantised (and differs from it: the slice ran)
    for gm in (1, 0):
        psi, acc = run(gradient_math=gm, psi_fixed_point=0)
        psiq, accq = run(gradient_math=gm, psi_fixed_point=1)
        assert_same(psiq[0::2], psi[0::2], f"geomean TMA gm={gm}: fixed vs fp64, a")
        assert_same(psiq[1::2], quantise_b(psi[1::2], R[:, 1]), f"geomean TMA gm={gm}: fixed vs fp64, b")
        assert np.any(psiq[1::2] != psi[1::2])
        within(psi, econ_tma if gm else none, "geomean TMA exp2/log2" if gm else "geomean TMA reference order")
        if gm == 0:
            near_oracle(psi)
    # first-generation kernel: exp2/log2, pow, reference order; then exact = 1 on both kernels
    within(run(geomean_tma=0)[0], econ_gen1, "geomean first-gen exp2/log2")
    within(run(geomean_log2=0)[0], econ_gen1, "geomean first-gen pow")
    psi, _ = run(geomean_tma=0, gradient_math=0)
    within(psi, none, "geomean first-gen reference order")
    near_oracle(psi)
    for tma in (1, 0):
        psi, _ = run(geomean_tma=tma, exact=1, psi_fixed_point=0)
        within(psi, none, "geomean exact")
        near_oracle(psi)
    psi, acc = run()
    slack = [(C_GEOMEAN + 2 * L) * EPS * (R[:, k] + g * np.abs(f.astype(float))) / g + (half_quantum(R[:, 1]) if k else 0)
             for k, f in ((0, fa), (1, fb))]
    check_acc(acc, v, fa, fb, *slack)
    p.close()


# ---------------------------------------------------------------------------
# UniV3
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("m", [1, 31, 33, 64, 65, 20_000])
def test_univ3_gradient_sweep_per_pool(cr, oracle, synth, m, ragged):
    """The gradient-only UniV3 kernel (MAT = false): per-pool Λ−Δ bit-exact against the oracle,
    ladder edges included, with one wave of CTAs and with one CTA per 512 pools."""
    cp, g, Ai, off, lt, lq, v = synth.disjoint_univ3(m, seed=m, ragged=ragged)
    n = 2 * m
    Do, Lo = oracle.sweep_univ3(cp, g, Ai, off, lt, lq, v, threads=8)
    fa, fb = Lo[:, 0] - Do[:, 0], Lo[:, 1] - Do[:, 1]
    if m >= 40:
        assert np.count_nonzero(fa) and np.count_nonzero(fb) and np.count_nonzero((fa == 0) & (fb == 0))
    p = make(cr, n, univ3=(cp, g, Ai, off, lt, lq))
    for waves in (-1, 0):
        p.set_option("grid_waves", waves)
        psi, acc = p.sweep(v)
        assert_same(psi[0::2], fa, f"grid_waves={waves}, a")
        assert_same(psi[1::2], fb, f"grid_waves={waves}, b")
        check_acc(acc, v, fa.astype(LD), fb.astype(LD))
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hubs", [False, True])
def test_univ3_gradient_sweep_shared_tokens(cr, oracle, synth, hubs):
    """The same gradient-only path on shared-token sets (uniform, and Zipf hubs): Ψ and acc
    within summation-order noise of the oracle's per-pool trades."""
    from test_gpu_parity import check_psi
    m, n = 60_000, 800
    cp, g, Ai, off, lt, lq = synth.univ3_pools(m, n, seed=5, ragged=True)
    if hubs:
        Ai = synth.product_pools_skewed(m, n, alpha=1.0, seed=6)[2]
    rng = np.random.default_rng(7)
    v = np.exp(rng.uniform(np.log(0.5), np.log(2.0), size=n))
    Do, Lo = oracle.sweep_univ3(cp, g, Ai, off, lt, lq, v, threads=8)
    p = make(cr, n, univ3=(cp, g, Ai, off, lt, lq))
    for waves in (-1, 0):
        p.set_option("grid_waves", waves)
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    p.close()


# ---------------------------------------------------------------------------
# repeated sweeps at one ν
# ---------------------------------------------------------------------------

def _from_ptr(torch, ptr, count, dev):
    class _Holder:
        pass
    h = _Holder()
    h.__cuda_array_interface__ = {"shape": (count,), "typestr": "<f8", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device=dev)


def cta_chunk_counts(p):
    """Chunks each CTA of the last TMA sweep processed (option "trace", cfmm_debug_read_trace):
    the lengths of the range table it ran under."""
    import ctypes as C
    grid = C.c_int64(0)
    buf = (C.c_uint64 * (8 * 4096))()
    p._chk(p._lib.cfmm_debug_read_trace(p._ctx, buf, 4096, C.byref(grid)))
    words = np.frombuffer(buf, dtype=np.uint64)[:8 * grid.value].reshape(-1, 8)
    return tuple(int(x) for x in words[:, 7] & np.uint64(0xffffffff))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["product", "geomean", "univ3"])
def test_repeated_sweeps_bitwise_identical(cr, synth, kind):
    """20 gradient-only sweeps at one ν: eager, graph-captured and replayed, device-resident
    (cfmm_sweep_device_view), across materialising sweeps and, for ProductTwoCoin, under two
    range tables: the one cfmm_finalize's calibration sweeps derived from measured CTA speeds,
    then the even split (option "balance" = 0).  The per-CTA chunk counts of the phase trace
    show which table a sweep ran under.  Ψ is bitwise identical every time; acc (summed across
    CTAs in varying order) within summation noise."""
    import torch
    if kind == "product":
        m = 450_000
        R, g, Ai, v = synth.disjoint_product(m, seed=21)
        data = dict(product=(R, g, Ai))
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        lay = layout(cr, 2 * m, Ai, orient=0)
        # one CTA per SM: enough chunks per CTA for the speed feedback to re-size the ranges
        assert lay["bucketed"] and lay["m_padded"] // 96 >= 32 * sms
        pre = {"blocks_per_sm": 1}
    elif kind == "geomean":
        m = 200_000
        R, g, Ai, w, v = synth.disjoint_geomean(m, seed=22)
        data = dict(geomean=(R, g, Ai, w))
        pre = {}
    else:
        m = 100_000
        cp, g, Ai, off, lt, lq, v = synth.disjoint_univ3(m, seed=23, ragged=True)
        data = dict(univ3=(cp, g, Ai, off, lt, lq))
        pre = {}
    n = 2 * m
    p = make(cr, n, pre=pre, **data)
    if kind == "product":
        p.set_option("trace", 1)
    first, acc0 = p.sweep(v)
    ranges = []
    dev = torch.device("cuda", 0)
    d_v = torch.from_numpy(v).to(dev)
    stream = torch.cuda.current_stream().cuda_stream
    accs = []
    for k in range(19):
        if k % 5 == 3:
            ptr = p.sweep_device_view(d_v.data_ptr(), False, stream)
            torch.cuda.synchronize()
            h = _from_ptr(torch, ptr, n + 1, dev).clone().cpu().numpy()
            psi, acc = h[:n], float(h[n])
        else:
            if k == 9:
                p.sweep(v, materialize=True)            # flips the accumulator parity
            if k == 14:
                p.set_option("sweep_graphs", 0)     # eager from here: option changes take effect
            if k == 16:
                p.set_option("balance", 0)
            psi, acc = p.sweep(v)
        assert np.array_equal(psi.view(np.int64), first.view(np.int64)), (k, np.argwhere(psi != first)[:5])
        accs.append(acc)
        if kind == "product":
            ranges.append(cta_chunk_counts(p))
            assert sum(ranges[-1]) == lay["m_padded"] // 96
    if kind == "product":
        grid = len(ranges[0])
        even = tuple(((c + 1) * lay["m_padded"] // 96) // grid - (c * lay["m_padded"] // 96) // grid
                     for c in range(grid))
        assert ranges[0] != even and ranges[-1] == even, (ranges[0][:8], ranges[-1][:8])
    scale = float(np.sum(np.abs(first) * v))
    assert max(abs(a - acc0) for a in accs) <= 1e-12 * scale
    p.close()
