"""GPU tests of the 18-byte pool record of the 192-pool compact stream: a 16-bit word per pool
holds b within its bucket, a relative to the first a of its lane (six pools per lane) and a slot of
the record's table of four γ codes; the record header holds every lane's first a relative to the
record's first a.  A set takes these records only when every record fits: lane spans <= 7, lane
offsets <= 255, at most four fees among a record's real pools; otherwise the 192-pool option falls
back to the 96-pool records.  Each case runs both sides of its boundary, asks the library which
record it streams and checks Ψ and acc against the oracle."""
import numpy as np
import pytest

from test_gpu_compact_records import sweep_checked
from test_gpu_parity import make_pools

pytestmark = pytest.mark.gpu

N = 1500  # tokens: one b-bucket
TIERS = np.array([0.997, 0.998, 0.999, 0.9995, 0.9999])  # none of them 1.0, the padding pools' fee


def lane_ladder(k, step=8):
    """First tokens of k pools in device order: every lane of six pools on one token, the next lane
    `step` tokens further (lane offsets up to 31·step within a record)."""
    return 10 + step * (np.arange(k) // 6)


def pool_set(a, gamma, seed=7):
    """Pools inserted in device order (first tokens a, non-decreasing), second tokens spread over
    bucket 0, random reserves."""
    a = np.asarray(a, dtype=np.int64)
    k = len(a)
    b = 1 + (np.arange(k, dtype=np.int64) * 37 + 11) % N
    b = np.where(b == a, b % N + 1, b)
    R = np.maximum(1000.0 * np.random.default_rng(seed).random((k, 2)), 1e-3)
    return R, np.asarray(gamma, dtype=np.float64), np.stack([a, b], axis=1)


def check(cr, oracle, synth, R, g, Ai, record):
    p = make_pools(cr, N, product=(R, g, Ai), pre={"orient_by_degree": 0})
    assert p.pool_set_info(0)["compact_stream"] == 1
    p.set_option("compact_record", 192)
    assert p.compact_record(0) == record
    sweep_checked(p, oracle, R, g, Ai, N, synth=synth)
    p.close()


@pytest.mark.parametrize("span,record", [(7, 192), (8, 96)])
def test_lane_span(cr, oracle, synth, span, record):
    """Lane 5 of the first record: its six first tokens span 7 (the largest offset a pool word holds)
    or 8."""
    a = lane_ladder(384)
    a[35] = a[30] + span
    rng = np.random.default_rng(1)
    check(cr, oracle, synth, *pool_set(a, rng.choice([0.997, 1.0], size=384)), record)


@pytest.mark.parametrize("off,record", [(255, 192), (256, 96)])
def test_lane_offset(cr, oracle, synth, off, record):
    """Lanes 0-30 of the first record on one token, lane 31 `off` tokens further (the header's lane
    offsets are bytes)."""
    a = np.full(384, 10, dtype=np.int64)
    a[186:192] = 10 + off
    a[192:] = 10 + off + 1 + (np.arange(192) // 6)
    rng = np.random.default_rng(2)
    check(cr, oracle, synth, *pool_set(a, rng.choice([0.997, 1.0], size=384)), record)


@pytest.mark.parametrize("fees,record", [(4, 192), (5, 96)])
def test_fees_per_record(cr, oracle, synth, fees, record):
    """The first record's pools use 4 or 5 fee tiers; the second record one."""
    g = np.full(384, 0.997)
    g[:192] = TIERS[np.arange(192) % fees]
    check(cr, oracle, synth, *pool_set(lane_ladder(384), g), record)


def test_half_padding_record_with_four_fees(cr, oracle, synth):
    """242 pools: three chunks, the third holding 50 real pools and 46 padding pools, so the second
    record is half padding.  Its real pools use four fees, none of them the padding pools' 1.0, so
    the padding pools take a slot whose fee belongs to real pools (zero reserves: no trade)."""
    g = np.where(np.arange(242) % 2 == 0, 0.997, 1.0)
    g[192:] = TIERS[np.arange(50) % 4]
    check(cr, oracle, synth, *pool_set(lane_ladder(242), g), 192)


@pytest.mark.parametrize("chunks", [1, 2, 3, 4])
def test_bucket_chunk_counts(cr, oracle, synth, chunks):
    """Bucket 0 holds 1 to 4 chunks (the last one partly padding): with 1 and 3 the last record's
    second half is padding."""
    k = 96 * chunks - 10
    rng = np.random.default_rng(3 + chunks)
    check(cr, oracle, synth, *pool_set(lane_ladder(k), rng.choice(TIERS[:3], size=k)), 192)


def test_reserve_updates_apply_and_retire(cr, oracle, synth):
    """The packed records follow every reserve change: apply the trades of a materialising sweep,
    push new reserves, retire pools, then sweep and compare with the oracle on the resulting state
    (retired pools absent)."""
    k = 96 * 4 - 10
    rng = np.random.default_rng(11)
    R, g, Ai = pool_set(lane_ladder(k), rng.choice(TIERS[:4], size=k), seed=12)
    p = make_pools(cr, N, product=(R, g, Ai), pre={"orient_by_degree": 0})
    p.set_option("compact_record", 192)
    assert p.compact_record(0) == 192
    sweep_checked(p, oracle, R, g, Ai, N, kinds=("near",), synth=synth)
    p.sweep(synth.dual_prices(N, "wide"), materialize=True)
    p.apply_trades()
    upd = np.arange(5, k, 17)
    p.update_reserves(0, int(upd[0]), R[upd[0]:upd[0] + 3] * 1.5)
    for i in upd[1:]:
        p.update_reserves(0, int(i), R[i:i + 1] * 0.75)
    active = rng.random(k) >= 0.2
    p.set_active(0, 0, active)
    assert p.compact_record(0) == 192
    state, act = p.pool_state(0)
    assert np.array_equal(act, active)
    assert np.array_equal(state[upd[1:]], R[upd[1:]] * 0.75)
    sweep_checked(p, oracle, state[active], g[active], Ai[active], N, synth=synth)
    p.close()
