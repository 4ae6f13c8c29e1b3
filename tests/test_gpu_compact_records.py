"""GPU tests of the 192-pool compact records of the headline sweep: two consecutive 96-pool chunks
of one b-bucket share a record (the second half of a bucket's last record is 96 no-trade pools
when the bucket has an odd chunk count), pools sit lane-interleaved in it, and the first tokens
of the whole record must span at most 8191.  Option compact_record forces the record size (0, the
default, takes 192-pool records only on sets with several of them per resident warp)."""
import numpy as np
import pytest

from test_gpu_parity import EPS, check_psi, make_pools

pytestmark = pytest.mark.gpu


def bucket0_set(synth, k, span, n=20_000, seed=23):
    """Random pools whose second tokens all lie beyond 1600 (so outside b-bucket 0), plus k pools
    in bucket 0 whose first tokens run from 2001 to 2001 + span."""
    R, g, Ai = synth.product_pools(60_000, n, seed=seed)
    Ai[:, 1] = 1601 + (Ai[:, 1] - 1) % (n - 1600)
    clash = Ai[:, 0] == Ai[:, 1]
    Ai[clash, 0] = Ai[clash, 0] % 1600 + 1
    a0 = np.round(np.linspace(2001, 2001 + span, k)).astype(np.int64)
    b0 = 1 + (np.arange(k, dtype=np.int64) * 7) % 1200
    rng = np.random.default_rng(seed)
    R0 = np.maximum(1000.0 * rng.random((k, 2)), 1e-3)
    g0 = rng.choice(np.array([0.997, 0.9995, 1.0]), size=k)
    return (np.concatenate([R0, R]), np.concatenate([g0, g]), np.concatenate([np.stack([a0, b0], axis=1), Ai]))


def sweep_checked(p, oracle, R, g, Ai, n, kinds=("near", "wide"), synth=None):
    for kind in kinds:
        v = synth.dual_prices(n, kind)
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
        for fixed in (1, 0):
            p.set_option("psi_fixed_point", fixed)
            psi, acc = p.sweep(v)
            check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g, Rq=R if fixed else np.zeros_like(R))


@pytest.mark.parametrize("k", [40, 150, 200, 300])
@pytest.mark.parametrize("record", [192, 96])
def test_odd_and_even_bucket_chunk_counts(cr, oracle, synth, k, record):
    """Bucket 0 holds 1, 2, 3 or 4 chunks: with 1 and 3 its last 192-pool record is half padding."""
    n = 20_000
    R, g, Ai = bucket0_set(synth, k, span=3000, n=n)
    p = make_pools(cr, n, product=(R, g, Ai), pre={"orient_by_degree": 0})
    assert p.pool_set_info(0)["compact_stream"] == 1
    p.set_option("compact_record", record)
    sweep_checked(p, oracle, R, g, Ai, n, synth=synth)
    p.close()


@pytest.mark.parametrize("span,compact", [(8191, 1), (12_000, 0)])
def test_record_span_at_the_field_limit(cr, oracle, synth, span, compact):
    """150 pools in bucket 0 (two chunks, one record) whose first tokens span 8191 (the largest
    offset the record holds) or 12000: each chunk alone would fit the field at 12000 (7.7k and 4.3k),
    the record does not, so the set takes the 32-byte stream."""
    n = 20_000
    R, g, Ai = bucket0_set(synth, 150, span=span, n=n)
    p = make_pools(cr, n, product=(R, g, Ai), pre={"orient_by_degree": 0})
    assert p.pool_set_info(0)["compact_stream"] == compact
    for record in (192, 96):
        p.set_option("compact_record", record)
        sweep_checked(p, oracle, R, g, Ai, n, synth=synth)
    p.close()


@pytest.mark.parametrize("skewed", [False, True])
@pytest.mark.parametrize("fixed,per_sm", [(1, 0), (0, 0), (1, 1), (1, 2)])
def test_option_grid_on_1m_pools(cr, oracle, synth, skewed, fixed, per_sm):
    """~1M pools over 5k tokens (many buckets, about half with an odd chunk count), with and
    without hub tokens (SKEW), fixed-point and fp64 Ψ[b] slices, CTAs per SM, two price vectors."""
    m, n = 1_000_000, 5_000
    if skewed:
        R, g, Ai = synth.product_pools_skewed(m, n, alpha=1.0, seed=78)
    else:
        R, g, Ai = synth.product_pools(m, n, seed=79)
    p = make_pools(cr, n, product=(R, g, Ai))
    assert p.pool_set_info(0)["compact_stream"] == 1
    p.set_option("compact_record", 192)
    p.set_option("psi_fixed_point", fixed)
    p.set_option("blocks_per_sm", per_sm)
    for kind in ("near", "wide"):
        v = synth.dual_prices(n, kind)
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g, Rq=R if fixed else np.zeros_like(R))
    p.close()


def test_record_sizes_and_wide_stream_agree(cr, oracle, synth):
    """The same set through 192-pool records, 96-pool records and the 32-byte stream: Ψ and acc
    agree within the summation-order noise (the per-pool math is the same operation for
    operation; only the order of the Ψ[a] and acc adds differs)."""
    m, n = 1_000_000, 5_000
    R, g, Ai = synth.product_pools(m, n, seed=80)
    p = make_pools(cr, n, product=(R, g, Ai))
    v = synth.dual_prices(n, "near")
    out = {}
    for name, opts in (("r192", {"compact_record": 192}), ("r96", {"compact_record": 96}),
                       ("wide", {"compact_stream": 0})):
        p.set_option("compact_stream", 1)
        for k, val in opts.items():
            p.set_option(k, val)
        out[name] = p.sweep(v)
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    _, _, absG = oracle.fold_compensated(Ai, Do, Lo, v, n)
    psi0, acc0 = out["r192"]
    check_psi(oracle, Ai, Do, Lo, v, n, psi0, acc0, R=R, g=g)
    for name in ("r96", "wide"):
        psi, acc = out[name]
        assert np.all(np.abs(psi - psi0) <= 1e-12 * absG + 1e-300), name
        assert abs(acc - acc0) <= 1e-12 * float(np.sum(absG * v)), name
    p.close()


def test_repeated_sweeps_and_graph_replay(cr, oracle, synth):
    """Repeated sweeps with the same buffers (replayed as one CUDA graph once captured) pass the
    oracle check every time.  Ψ of the tokens that are only ever second tokens comes from the
    exact fixed-point slices; what may still move between sweeps is the order in which the CTAs
    sharing a bucket add their partials in fp64, so it repeats to within a few ulp."""
    m, n = 1_000_000, 5_000
    R, g, Ai = synth.product_pools(m, n, seed=81)
    Ai[:, 0] = 1 + (Ai[:, 0] - 1) % 2500          # first tokens 1..2500, second tokens 2501..5000
    Ai[:, 1] = 2501 + (Ai[:, 1] - 1) % 2500
    p = make_pools(cr, n, product=(R, g, Ai), pre={"orient_by_degree": 0})
    p.set_option("compact_record", 192)
    v = synth.dual_prices(n, "near")
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    _, _, absG = oracle.fold_compensated(Ai, Do, Lo, v, n)
    b_only = np.arange(n) >= 2500
    first = None
    for _ in range(6):
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
        if first is None:
            first = psi.copy()
        assert np.all(np.abs(psi[b_only] - first[b_only]) <= 16 * EPS * absG[b_only])
    p.close()
