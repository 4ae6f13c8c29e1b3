"""GPU tests of the compact ProductTwoCoin stream (20-byte pool records): its first token is
stored as a 13-bit offset from the first token of its 96-pool chunk, so a pool set takes the
compact stream only when every chunk's first tokens span at most 8191; any other set takes the
32-byte stream.  Both sides of that rule must give the oracle's Ψ and acc."""
import numpy as np
import pytest

from test_gpu_parity import check_psi, make_pools

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("variant,fixed,per_sm,compact", [(-1, 1, 0, 1), (0, 1, 0, 1), (0, 0, 0, 1), (0, 1, 1, 1),
                                                           (0, 1, 0, 0), (0, 0, 0, 0)])
def test_sparse_pool_set_takes_the_wide_stream(cr, oracle, synth, variant, fixed, per_sm, compact):
    """5k pools over 50k tokens: the first tokens of one chunk span about 35k, far beyond the compact
    record's offset field, so even with compact_stream=1 the 32-byte stream runs.  Same option grid
    as the other gradient-sweep variants."""
    m, n = 5_000, 50_000
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
    p.set_option("use_tma", 0)
    psi, acc = p.sweep(v)
    check_psi(oracle, Ai, Do, Lo, v, n, psi, acc)
    p.sweep(v, materialize=True)
    D, L = p.trades()
    assert np.array_equal(D, Do) and np.array_equal(L, Lo)
    p.close()


@pytest.mark.parametrize("span", [8191, 8192])
def test_chunk_token_span_at_the_field_limit(cr, oracle, synth, span):
    """One chunk whose first tokens span exactly 8191 (the largest offset the compact record holds:
    20-byte stream) or 8192 (one more: 32-byte stream).  An off-by-one in the field width or in the
    host's span check would add Ψ[a] of that chunk's last pool to the wrong token."""
    n = 12_000                 # 8 b-buckets of 1500 tokens
    R, g, Ai = synth.product_pools(60_000, n, seed=23)
    # every random pool's second token in buckets 1.. (b > 1600 > bucket width)
    Ai[:, 1] = 1601 + (Ai[:, 1] - 1) % (n - 1600)
    clash = Ai[:, 0] == Ai[:, 1]
    Ai[clash, 0] = Ai[clash, 0] % 1600 + 1
    # bucket 0 holds 40 pools (one chunk, padded with copies of its last first token) whose first
    # tokens run from 2001 to 2001 + span
    k = 40
    a0 = np.round(np.linspace(2001, 2001 + span, k)).astype(np.int64)
    b0 = 1 + np.arange(k, dtype=np.int64) * 17
    rng = np.random.default_rng(3)
    R0 = np.maximum(1000.0 * rng.random((k, 2)), 1e-3)
    g0 = rng.choice(np.array([0.997, 1.0]), size=k)
    R = np.concatenate([R0, R])
    g = np.concatenate([g0, g])
    Ai = np.concatenate([np.stack([a0, b0], axis=1), Ai])
    assert Ai[:k, 0].max() - Ai[:k, 0].min() == span
    p = make_pools(cr, n, product=(R, g, Ai), pre={"orient_by_degree": 0})
    for kind in ("wide", "near"):
        v = synth.dual_prices(n, kind)
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
        for fixed in (1, 0):
            p.set_option("psi_fixed_point", fixed)
            psi, acc = p.sweep(v)
            check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g, Rq=R if fixed else np.zeros_like(R))
    p.close()
