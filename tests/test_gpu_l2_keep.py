"""The L2 kept across headline sweeps (option l2_keep): on a ProductTwoCoin set whose packed stream
is larger than the L2, the TMA sweep's bulk copies keep the first records of every CTA's range in the
L2 (evict_last) and stream the rest (evict_first).  Only the later sweeps of a run read kept records from the L2, so
several gradient sweeps in a row, at two ν, are each checked against the oracle's per-pool trades,
with the hints on and off.  A set whose stream fits in the L2 runs without hints whatever l2_keep says."""
import numpy as np
import pytest

from test_gpu_parity import check_psi, make_pools

pytestmark = pytest.mark.gpu

SWEEPS = 4  # per ν and setting: the first reads HBM only, the later ones the kept records too


def test_l2_keep_repeated_sweeps(cr, oracle, synth):
    # 4M pools over 20k tokens: 20,834 records of 3520 B, 73 MB > the H100's 50 MB L2
    m, n = 4_000_000, 20_000
    R, g, Ai = synth.product_pools(m, n, seed=11)
    p = make_pools(cr, n, product=(R, g, Ai))
    assert p.compact_record(0) == 192
    keep = p.l2_keep(0)
    assert keep > 1, keep
    for kind in ("near", "wide"):
        v = synth.dual_prices(n, kind)
        Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=oracle.max_threads())
        for setting in (-1, 0):
            p.set_option("l2_keep", setting)
            assert p.l2_keep(0) == (keep if setting else 0)
            for _ in range(SWEEPS):
                psi, acc = p.sweep(v)
                check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    # an explicit count of kept records per CTA range runs as given; values below -1 are refused
    p.set_option("l2_keep", 3)
    assert p.l2_keep(0) == 3
    v = synth.dual_prices(n, "near")
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=oracle.max_threads())
    for _ in range(2):
        psi, acc = p.sweep(v)
        check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    with pytest.raises(cr.CFMMError):
        p.set_option("l2_keep", -2)
    p.close()


def test_l2_keep_no_effect_in_l2(cr, oracle, synth):
    # 300k pools over 4k tokens: a stream of a few MB, which the L2 holds without hints
    m, n = 300_000, 4_000
    R, g, Ai = synth.product_pools(m, n, seed=4)
    v = synth.dual_prices(n, "near")
    Do, Lo = oracle.sweep_product(R, g, Ai, v, threads=8)
    p = make_pools(cr, n, product=(R, g, Ai))
    p.sweep(v)  # (the first gradient sweep also packs the stream)
    for setting in (-1, 0, 1, 8):
        p.set_option("l2_keep", setting)
        assert p.l2_keep(0) == 0
        for _ in range(2):
            l0 = p.launch_count
            psi, acc = p.sweep(v)
            assert p.launch_count == l0 + 1
            check_psi(oracle, Ai, Do, Lo, v, n, psi, acc, R=R, g=g)
    p.close()
