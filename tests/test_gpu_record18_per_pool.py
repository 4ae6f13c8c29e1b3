"""Per-pool checks of the headline sweep's 192-pool compact records (18 bytes per pool).

The sets here are laid out so that they fit the 18-byte record (lane spans <= 7, lane offsets
<= 255, at most four fees among a record's real pools) while their Ψ can still be read out pool by
pool.  Every token lives in one b-bucket of 1600 tokens (n is a multiple of 1600): the first tokens
fill the low buckets, the second tokens the high ones, and pools are inserted in device order
(bucket of b, a), so the generators decide which pools share a lane, a record and a bucket.
  * token-disjoint sets: every pool has its own a and b, Ψ is that pool's flow;
  * run sets: every pool has its own b, the a tokens form runs of 1 to 200 pools;
  * hub sets: run sets plus one token held by the first record of every bucket (the layout then
    detects a hub and the SKEW kernels run);
  * the default-rule set: 2.1M pools in runs of six on a and groups of four on b, large enough
    that the 192-pool record is chosen without being forced.
The rule upload_set applies is restated on the layout's order (rec18_rule) and checked on the CPU,
together with the edges each set is meant to hold and a twin one step past every limit.  The GPU
tests then hold every pool to the truth (single-pool tokens: per pool, bit for bit where the
same operations run; shared tokens: the sum of the pools' bounds, each pool's flow larger than it).
"""
import itertools

import numpy as np
import pytest

from test_gpu_pool_readout import (C_PRODUCT_ECON, _nu_out_of_range, check_acc, error_units, product_truth,
                                   quantise_b, assert_same, fixed_exponent, make, set_options, record, LD, EPS)
from test_layout import layout

NB = 1600                                          # tokens per b-bucket (kTmaNbMax)
# pools per b-bucket, cycled: 15 chunks (odd: the last record is half padding, 40 padding pools in
# its first half), 16 (no padding), 16 (36 padding), 17 (odd, one real pool in the last chunk)
BUCKET_POOLS = (1400, 1536, 1500, 1537, 1450)
# runs of a tokens, cycled: inside a lane, across lane boundaries, whole lanes, across records
RUNS = (1, 1, 1, 1) + tuple(range(2, 14)) + (24, 200)
REC, LANE = 192, 6


# ---------------------------------------------------------------------------
# the 18-byte record rule, restated on the layout's device order (upload_set)
# ---------------------------------------------------------------------------

def records(lay):
    """The 192-pool records of a bucketed layout: (first chunk, odd) per record; odd: the bucket's
    last chunk without a partner (the record's second half is padding)."""
    tb = np.asarray(lay["tile_bucket"])
    nc = len(tb)
    new = np.r_[True, tb[1:] != tb[:-1]]
    first = np.nonzero(new)[0]
    k = np.arange(nc) - np.repeat(first, np.diff(np.r_[first, nc]))
    starts = np.nonzero(k % 2 == 0)[0]
    odd = (starts + 1 >= nc) | (tb[np.minimum(starts + 1, nc - 1)] != tb[starts])
    return starts, odd


def record_positions(lay):
    """Per record its 192 logical pools: the device position each one reads its a from (the second
    half of an odd record repeats the first half's last a) and whether it is a real pool."""
    starts, odd = records(lay)
    q = np.arange(REC)
    pos = starts[:, None] * 96 + q[None, :]
    half = odd[:, None] & (q[None, :] >= 96)
    pos = np.where(half, starts[:, None] * 96 + 95, pos)
    order = lay["order"]
    real = (order[pos] >= 0) & ~half
    return pos, real, odd


def device_first_tokens(lay, Ai):
    """0-based first token (after orientation) of every device position; padding pools repeat the
    last real pool before them."""
    Ai = np.asarray(Ai).reshape(-1, 2) - 1
    sw = lay["swapped"].astype(bool)
    oa = np.where(sw, Ai[:, 1], Ai[:, 0])
    order = lay["order"]
    idx = np.where(order >= 0, np.arange(len(order)), -1)
    last = np.maximum.accumulate(idx)
    return oa[order[last]]


def rec18_rule(lay, Ai, g):
    """Does the set fit the 18-byte record (cfmm_capi.cu upload_set)?  Also returns what the
    generators' edges are checked against: per record the largest lane span, the largest lane
    offset, the fee count, whether fee 1.0 is among its real pools, and whether it is odd."""
    assert lay["bucketed"]
    g = np.asarray(g, dtype=np.float64)
    pos, real, odd = record_positions(lay)
    a = device_first_tokens(lay, Ai)[pos]
    lanes = a.reshape(len(a), 32, LANE)
    span = (lanes[:, :, -1] - lanes[:, :, 0]).max(axis=1)
    off = (lanes[:, :, 0] - a[:, :1]).max(axis=1)
    order = lay["order"]
    gg = np.where(real, g[np.maximum(order[pos], 0)], 2.0)         # 2.0: no pool (fees are <= 1)
    gs = np.sort(gg, axis=1)
    fees = np.count_nonzero((np.diff(gs, axis=1) != 0) & (gs[:, 1:] <= 1.0), axis=1) + (gs[:, 0] <= 1.0)
    fee1 = np.any(real & (gg == 1.0), axis=1)
    rec_span = a[:, -1] - a[:, 0]
    compact = rec_span.max() <= 8191 and len(np.unique(np.r_[g, 1.0])) <= 256
    fits = bool(compact and span.max() <= 7 and off.max() <= 255 and fees.max() <= 4)
    return dict(fits=fits, span=span, off=off, fees=fees, fee1=fee1, odd=odd, real=real, pos=pos)


def run_shapes(lay, Ai):
    """Which run shapes of first tokens the device order holds: a run of >= 2 pools inside one
    lane, one across a lane boundary, one covering a whole lane, one across a record's end."""
    pos, real, _ = record_positions(lay)
    a = device_first_tokens(lay, Ai)[pos]
    r = real.reshape(len(a), 32, LANE)
    la = a.reshape(len(a), 32, LANE)
    same = la[:, :, 1:] == la[:, :, :-1]
    inside = np.any(same & r[:, :, 1:] & r[:, :, :-1])
    across = np.any((la[:, 1:, 0] == la[:, :-1, -1]) & r[:, 1:, 0] & r[:, :-1, -1])
    whole = np.any(np.all(la == la[:, :, :1], axis=2) & np.all(r, axis=2))
    nxt = a[1:, 0] == a[:-1, -1]
    rec_end = np.any(nxt & real[1:, 0] & real[:-1, -1])
    return dict(inside=bool(inside), across=bool(across), whole=bool(whole), record_end=bool(rec_end))


# ---------------------------------------------------------------------------
# generators
# ---------------------------------------------------------------------------

def _bucket_sizes(m, sizes=BUCKET_POOLS):
    out = []
    while sum(out) < m:
        out.append(sizes[len(out) % len(sizes)])
    out[-1] -= sum(out) - m
    return np.array(out, dtype=np.int64)


def _place(cr, a, per_bucket, b_per_pool=None, orient=0):
    """Token labels and layout for pools given in device order: first tokens a (1-based, non-
    decreasing inside each bucket), per_bucket pools per b-bucket; second tokens in the buckets
    above the first tokens' (each pool its own, or b_per_pool pools each)."""
    k_b = np.repeat(np.arange(len(per_bucket)), per_bucket)
    pos = np.arange(len(a)) - np.repeat(np.cumsum(per_bucket) - per_bucket, per_bucket)
    ba = -(-int(a.max()) // NB) + 1               # buckets of first tokens, one spare for appends
    step = b_per_pool or 1
    b = NB * (ba + k_b) + 1 + pos // step
    n = NB * (ba + len(per_bucket))
    Ai = np.stack([a, b], axis=1).astype(np.int64)
    lay = layout(cr, n, Ai, orient=orient)
    return Ai, n, lay


def _fee_groups(n_recs, fees, extra=None):
    """Every record's fees: three codes cycling over 1..255, plus 1.0 (code 0) on every third record
    (four fees); extra: {record: fees to add}."""
    groups = []
    for r in range(n_recs):
        grp = [fees[1 + (3 * r + t) % 255] for t in range(3)]
        if r % 3 == 0:
            grp.append(1.0)
        for f in (extra or {}).get(r, []):
            if f not in grp:
                grp.append(f)
        groups.append(grp)
    return groups


def _assign_fees(lay, groups):
    """γ per pool (insertion index) from its record's group: logical pool q takes group[q % len]
    (_place_adversarial relies on it)."""
    pos, real, _ = record_positions(lay)
    order = lay["order"]
    m = int(np.count_nonzero(order >= 0))
    g = np.full(m, np.nan)
    for r in range(len(pos)):
        grp = groups[r]
        q = np.nonzero(real[r])[0]
        g[order[pos[r, q]]] = np.array(grp)[q % len(grp)]
    assert not np.isnan(g).any()
    return g


def _adversarial(synth, seed):
    """disjoint_product's adversarial rows (economized-margin ties, 2^±80, the fixed-point guard),
    then eight rows with reserves at 2^-100 and 2^100: (R, γ, ν_a, ν_b) per row."""
    R, g, _, v = synth.disjoint_product(53, seed=seed)
    rng = np.random.default_rng(seed)
    fee = synth.fee_levels()[7]
    rows = [(R[i], g[i], v[2 * i], v[2 * i + 1]) for i in range(53)]
    for j in range(8):
        spread = 2.0 ** rng.uniform(4, 30)
        r = [2.0 ** -100, 2.0 ** -100 * spread] if j < 4 else [2.0 ** 100, 2.0 ** 100 / spread]
        rows.append((np.array(r if j % 2 else r[::-1]), fee, 2.0 ** rng.uniform(-4, 4), 2.0 ** rng.uniform(-4, 4)))
    return rows


def _place_adversarial(lay, groups, rows, eligible):
    """A pool for every adversarial row: a real pool of a record with four fees (every third record)
    at a logical position q = 3 mod 4, so that it takes the record's fourth fee (1.0), which the
    row's fee replaces.  eligible: per insertion index, may the pool take a row (a single-pool
    token).  Returns [(insertion index, row)]; groups are updated in place."""
    pos, real, _ = record_positions(lay)
    order = lay["order"]
    out = []
    rows = list(rows)
    for r in range(3, len(pos), 3):
        if not rows:
            break
        q = [q for q in range(3, REC, 4) if real[r, q] and eligible[order[pos[r, q]]]]
        if q:
            row = rows.pop(0)
            groups[r][3] = row[1]
            out.append((int(order[pos[r, q[0]]]), row))
    return out


def _apply_rows(placed, R, v, Ai):
    for i, (R0, _, va, vb) in placed:
        R[i] = R0
        v[Ai[i, 0] - 1], v[Ai[i, 1] - 1] = va, vb
    return np.array([i for i, _ in placed], dtype=np.int64)


def disjoint18(cr, synth, m, seed=1, past=None):
    """Token-disjoint set of m pools (n <= 1,024,000) on 192-pool records.  Edges: a lane whose six
    first tokens span 7 (record 1), a lane offset of 255 (record 2), four fees on every third
    record, the adversarial rows in records of four fees, odd buckets ending on a half-padding record; past = "span" / "offset" / "fees" builds
    the twin one step beyond that limit (span 8, offset 256, five fees in record 4)."""
    rng = np.random.default_rng(seed)
    per_bucket = _bucket_sizes(m)
    gap = np.zeros(m, dtype=np.int64)
    # positions inside bucket 0 (1400 pools: records 0-7, all but the last full)
    gap[REC * 1 + 5 * LANE + 3] = 2 + (past == "span")          # lane 5 of record 1 spans 5 + 2
    gap[REC * 2 + 31 * LANE] = 69 + (past == "offset")          # lane 31 of record 2 at 186 + 69
    a = 1 + np.arange(m) + np.cumsum(gap)
    Ai, n, lay = _place(cr, a, per_bucket)
    n_recs = len(records(lay)[0])
    fees = synth.fee_levels()
    extra = {4: [fees[200], fees[201]]} if past == "fees" else None      # record 4: five fees
    groups = _fee_groups(n_recs, fees, extra)
    placed = _place_adversarial(lay, groups, _adversarial(synth, seed), np.ones(m, dtype=bool))
    g = _assign_fees(lay, groups)
    # random rows as in disjoint_product: log2 R2 in U(-25, 40), log2(γP/Q) in U(-40, 40), log2 ν in U(-6, 6)
    va = np.exp2(rng.uniform(-6, 6, size=m))
    vb = np.exp2(rng.uniform(-6, 6, size=m))
    R2 = np.exp2(rng.uniform(-25, 40, size=m))
    rho = np.exp2(rng.uniform(-40, 40, size=m))
    R = np.stack([R2 * g * vb / (rho * va), R2], axis=1)
    v = np.ones(n)
    v[Ai[:, 0] - 1] = va
    v[Ai[:, 1] - 1] = vb
    adv = _apply_rows(placed, R, v, Ai)
    return dict(R=R, g=g, Ai=Ai, v=v, n=n, lay=lay, adv=adv)


def _shared_values(rng, Ai, g, n):
    """Reserves and prices where every pool trades and the pools of one token have flows of one
    order of magnitude: |log2(γP/Q)| in [2, 8], R1 within a factor 4 of a per-token scale.  The
    second reserves of a token's pools stay within 2^40 of each other (the fixed-point slice runs)."""
    m = len(g)
    v = np.exp2(rng.uniform(-2, 2, size=n))
    scale = np.exp2(rng.uniform(-4, 4, size=n))
    a, b = Ai[:, 0] - 1, Ai[:, 1] - 1
    R1 = scale[a] * np.exp2(rng.uniform(0, 2, size=m))
    rho = np.exp2(rng.uniform(2, 8, size=m) * rng.choice([-1.0, 1.0], size=m))
    R2 = rho * v[a] * R1 / (g * v[b])
    return np.stack([R1, R2], axis=1), v


def _run_tokens(m, runs=RUNS, first=1):
    lens = np.array([runs[i % len(runs)] for i in range(m)])
    ends = np.cumsum(lens)
    k = int(np.searchsorted(ends, m)) + 1
    return first + np.repeat(np.arange(k), lens[:k])[:m]


def runs18(cr, synth, m, seed=2, hub=False):
    """Every pool its own b; first tokens in runs of RUNS.  hub: one more token (1) holding the first
    192 pools of every bucket, so the hub's pools fill whole records and the layout detects a hub."""
    rng = np.random.default_rng(seed)
    per_bucket = _bucket_sizes(m, tuple(x - REC for x in BUCKET_POOLS) if hub else BUCKET_POOLS)
    a = _run_tokens(m, first=2 if hub else 1)
    if hub:
        a = np.asarray(a)
        starts = np.cumsum(per_bucket) - per_bucket
        a = np.insert(a, np.repeat(starts, REC), 1)
        per_bucket = per_bucket + REC
    Ai, n, lay = _place(cr, a, per_bucket, orient=-1 if hub else 0)
    n_recs = len(records(lay)[0])
    fees = synth.fee_levels()
    groups = _fee_groups(n_recs, fees)
    single = np.bincount(Ai[:, 0], minlength=n + 1)[Ai[:, 0]] == 1    # runs of length 1
    placed = _place_adversarial(lay, groups, _adversarial(synth, seed), single)
    g = _assign_fees(lay, groups)
    R, v = _shared_values(rng, Ai, g, n)
    adv = _apply_rows(placed, R, v, Ai)
    return dict(R=R, g=g, Ai=Ai, v=v, n=n, lay=lay, adv=adv)


def default_rule18(cr, synth, m=2_100_000, seed=3):
    """Large enough for the default choice of the 192-pool record (4 records per resident warp on
    132 SMs: 2.03M pools): first tokens in runs of six, second tokens shared by four pools."""
    rng = np.random.default_rng(seed)
    per_bucket = 4 * _bucket_sizes(-(-m // 4))
    per_bucket[-1] -= per_bucket.sum() - m
    a = 1 + np.arange(m) // 6
    Ai, n, lay = _place(cr, a, per_bucket, b_per_pool=4)
    n_recs = len(records(lay)[0])
    g = _assign_fees(lay, _fee_groups(n_recs, synth.fee_levels()))
    R, v = _shared_values(rng, Ai, g, n)
    return dict(R=R, g=g, Ai=Ai, v=v, n=n, lay=lay, adv=np.zeros(0, dtype=np.int64))


# ---------------------------------------------------------------------------
# CPU tests of the generators
# ---------------------------------------------------------------------------

def _common_requirements(s):
    rule = rec18_rule(s["lay"], s["Ai"], s["g"])
    assert rule["fits"], (rule["span"].max(), rule["off"].max(), rule["fees"].max())
    assert len(np.unique(s["g"])) == 256 and 1.0 in s["g"]          # every code of the dictionary
    assert rule["fee1"].any() and not rule["fee1"].all()            # 1.0 in some records only
    assert np.count_nonzero(rule["fees"] == 4) > 0
    assert rule["odd"].any() and (~rule["odd"]).any()               # half-padding records
    R = s["R"]
    assert np.all((R >= 2.0 ** -100) & (R <= 2.0 ** 100)) and np.all(s["g"] <= 1.0)
    return rule


def test_disjoint_sets_fit_with_their_edges(cr, synth):
    s = disjoint18(cr, synth, 40_000, seed=5)
    Ai = s["Ai"]
    assert len(np.unique(Ai)) == 2 * len(Ai) and s["n"] <= 1_024_000
    rule = _common_requirements(s)
    assert rule["span"].max() == 7 and rule["off"].max() == 255
    assert len(s["adv"]) == 61 and np.any(s["R"][s["adv"]] == 2.0 ** -100) and np.any(s["R"][s["adv"]] == 2.0 ** 100)
    assert np.all(rule["real"][rule["odd"]][:, 96:] == False)        # noqa: E712
    for past in ("span", "offset", "fees"):
        t = disjoint18(cr, synth, 40_000, seed=5, past=past)
        assert not rec18_rule(t["lay"], t["Ai"], t["g"])["fits"], past
    # the largest token-disjoint set of the GPU tests fits the bucket table
    big = disjoint18(cr, synth, 450_000, seed=7)
    assert big["lay"]["tile_bucket"][-1] + 1 <= 640 and big["n"] <= 1_024_000
    assert rec18_rule(big["lay"], big["Ai"], big["g"])["fits"]


@pytest.mark.parametrize("hub", [False, True])
def test_run_sets_fit_with_every_run_shape(cr, synth, hub):
    s = runs18(cr, synth, 40_000, hub=hub)
    _common_requirements(s)
    shapes = run_shapes(s["lay"], s["Ai"])
    assert all(shapes.values()), shapes
    assert s["lay"]["skewed"] == hub
    assert len(s["adv"]) >= 30


def test_default_rule_set(cr, synth):
    s = default_rule18(cr, synth)
    rule = rec18_rule(s["lay"], s["Ai"], s["g"])
    assert rule["fits"] and rule["odd"].any()
    assert len(rule["odd"]) >= 4 * 132 * 2 * 10                       # the default rule on 132 SMs
    assert s["n"] <= 1_024_000 and s["lay"]["tile_bucket"][-1] + 1 <= 640
    assert np.bincount(s["Ai"][:, 1]).max() == 4 and np.bincount(s["Ai"][:, 0]).max() == 6
    b = s["Ai"][:, 1]
    R2 = s["R"][:, 1]
    assert np.all(R2 * 2.0 ** 40 >= np.bincount(b, weights=R2)[b])   # the fixed-point slice runs


# ---------------------------------------------------------------------------
# GPU tests
# ---------------------------------------------------------------------------

def _in_range(x):
    return (x >= 2.0 ** -100) & (x < 2.0 ** 101)


def generic_pools(v, Ai, R, nb, fixed):
    """Per pool: does the TMA kernel take the generic (reference-order) form?  When any price of its
    b-bucket's slice is out of range (on the fixed-point slice the slice holds ν_b·2^(e_b−54), e_b
    from the token's total second reserve) or its ν_a is."""
    a, b = Ai[:, 0] - 1, Ai[:, 1] - 1
    x = np.array(v, dtype=np.float64)
    if fixed:
        S = np.bincount(b, weights=R[:, 1], minlength=len(v))
        held = np.unique(b[R[:, 1] != 0])
        x[held] = np.ldexp(x[held], fixed_exponent(S[held]) - 54)
    bad = np.zeros(-(-len(v) // nb), dtype=bool)
    np.logical_or.at(bad, np.arange(len(v)) // nb, ~_in_range(x))
    return bad[b // nb] | ~_in_range(np.asarray(v)[a])


def _interleaved(v, Ai):
    """ν in the (a, b) pairs check_acc reads: [ν_a0, ν_b0, ν_a1, ...]."""
    out = np.empty(2 * len(Ai))
    out[0::2], out[1::2] = v[Ai[:, 0] - 1], v[Ai[:, 1] - 1]
    return out


def _units(R, g, f):
    return C_PRODUCT_ECON * EPS * (R + g * np.abs(f.astype(np.float64))) / g


def check_disjoint(p, oracle, R, g, Ai, v, nb, key, active=None):
    """Every active pool of a token-disjoint set on the 192-pool record: fp64 slice within
    C_PRODUCT_ECON units of the truth, bit for bit the 96-pool record's and the 32-byte stream's;
    generic pools bit for bit the oracle's; the fixed-point slice the fp64 one quantised; acc.
    Retired pools' tokens read 0.  Returns the fp64 Ψ."""
    act = np.ones(len(g), dtype=bool) if active is None else active
    a, b = Ai[:, 0] - 1, Ai[:, 1] - 1
    out = {}
    for rec, fixed in itertools.product((192, 96, 0), (0, 1)):
        set_options(p, compact_record=rec or 192, compact_stream=rec != 0, psi_fixed_point=fixed)
        if rec:
            assert p.compact_record(0) == rec
        out[rec, fixed] = p.sweep(v)
    set_options(p, compact_record=192, compact_stream=1)
    for fixed in (0, 1):
        for rec in (96, 0):
            assert_same(out[rec, fixed][0], out[192, fixed][0], f"192 vs {rec}, fixed={fixed}")
    psi, acc = out[192, 0]
    psiq, accq = out[192, 1]
    Ra, ga, Aa = R[act], g[act], Ai[act]
    fa, fb = product_truth(Ra, ga, v[Aa[:, 0] - 1], v[Aa[:, 1] - 1])
    pa, pb = psi[Aa[:, 0] - 1], psi[Aa[:, 1] - 1]
    ua, ub = error_units(pa, fa, Ra[:, 0], ga), error_units(pb, fb, Ra[:, 1], ga)
    record(key, np.concatenate([ua, ub]))
    assert np.all(ua <= C_PRODUCT_ECON), np.argsort(ua)[-5:]
    assert np.all(ub <= C_PRODUCT_ECON), np.argsort(ub)[-5:]
    Do, Lo = oracle.sweep_product(Ra, ga, Aa, v, threads=8)
    fa_o, fb_o = Lo[:, 0] - Do[:, 0], Lo[:, 1] - Do[:, 1]
    gen = generic_pools(v, Aa, Ra, nb, fixed=False)
    gen_q = generic_pools(v, Aa, Ra, nb, fixed=True)
    assert_same(pa[gen], fa_o[gen], "generic pools, a")
    assert_same(pb[gen], fb_o[gen], "generic pools, b")
    same = gen_q == gen
    assert_same(psiq[Aa[:, 0] - 1], np.where(same, pa, fa_o), "fixed vs fp64 slice, a")
    assert_same(psiq[Aa[:, 1] - 1], quantise_b(np.where(same, pb, fb_o), Ra[:, 1]), "fixed vs fp64 slice, b")
    if not act.all():
        gone = np.concatenate([a[~act], b[~act]])
        assert np.all(psi[gone] == 0.0) and np.all(psiq[gone] == 0.0)
    vv = _interleaved(v, Aa)
    sa, sb = _units(Ra[:, 0], ga, fa), _units(Ra[:, 1], ga, fb)
    check_acc(acc, vv, fa, fb, sa, sb)
    check_acc(accq, vv, fa, fb, sa, sb + np.ldexp(1.0, fixed_exponent(Ra[:, 1]) - 55))
    return psi


@pytest.mark.gpu
@pytest.mark.parametrize("m", [40_000, 450_000])
def test_disjoint_per_pool(cr, oracle, synth, m):
    """Token-disjoint sets on the forced 192-pool record, with ν out of range on one b-bucket and
    on single a tokens; Ψ bitwise the same under every CTA shape and range table."""
    s = disjoint18(cr, synth, m, seed=m)
    R, g, Ai, n, lay = s["R"], s["g"], s["Ai"], s["n"], s["lay"]
    v = _nu_out_of_range(s["v"].copy(), lay, m)
    v[Ai[m // 2, 1] - 1] = 2.0 ** -110                     # a b-bucket's slice out of range
    gen = generic_pools(v, Ai, R, lay["nb"], fixed=False)
    assert gen.any() and not gen.all()
    p = make(cr, n, product=(R, g, Ai))
    p.set_option("compact_record", 192)
    assert p.compact_record(0) == 192
    check_disjoint(p, oracle, R, g, Ai, v, lay["nb"], "product economized, 192-pool record")
    set_options(p, psi_fixed_point=1)
    first, _ = p.sweep(v)
    for per_sm, balance in itertools.product((0, 1, 2), (1, 0)):
        set_options(p, blocks_per_sm=per_sm, balance=balance)
        psi, _ = p.sweep(v)
        assert np.array_equal(psi.view(np.int64), first.view(np.int64)), (per_sm, balance)
    p.close()


def check_shared(psi, R, g, Ai, v, n, fixed):
    """Tokens held by several pools: |Ψ − Σ truth| <= Σ_k C·unit_k + (r−1)·eps·Σ|f_k| (+ r half
    quanta of the b side on the fixed-point slice), and every pool's |f_k| above that bound, so a
    dropped or double-counted pool cannot pass."""
    a, b = Ai[:, 0] - 1, Ai[:, 1] - 1
    fa, fb = product_truth(R, g, v[a], v[b])
    tok = np.concatenate([a, b])
    f = np.concatenate([fa, fb])
    fabs = np.abs(f.astype(np.float64))
    unit = _units(np.concatenate([R[:, 0], R[:, 1]]), np.concatenate([g, g]), f)
    r = np.bincount(tok, minlength=n)
    truth = np.zeros(n, dtype=LD)
    np.add.at(truth, tok, f)
    bound = np.bincount(tok, weights=unit, minlength=n) + np.maximum(r - 1, 0) * EPS * \
        np.bincount(tok, weights=fabs, minlength=n)
    if fixed:
        S = np.bincount(b, weights=R[:, 1], minlength=n)
        rb = np.bincount(b, minlength=n)
        held = rb > 0
        bound[held] += rb[held] * np.ldexp(1.0, fixed_exponent(S[held]) - 55)
    err = np.abs((psi.astype(LD) - truth).astype(np.float64))
    held = r > 0
    assert np.all(err[held] <= bound[held]), np.argsort(np.where(held, err - bound, -np.inf))[-5:]
    multi = r[tok] >= 2
    assert np.all(fabs[multi] > bound[tok[multi]])
    ratio = np.where(held, err / np.maximum(bound, 1e-300), 0.0)
    return float(ratio.max())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["runs", "hubs", "default"])
def test_shared_tokens_per_pool(cr, oracle, synth, kind):
    """Runs of first tokens (forced 192-pool record), hub sets (SKEW kernels) and the 2.1M-pool set
    that takes the 192-pool record under the default options."""
    if kind == "default":
        s = default_rule18(cr, synth)
    else:
        s = runs18(cr, synth, 200_000, hub=kind == "hubs")
    R, g, Ai, v, n, lay = s["R"], s["g"], s["Ai"], s["v"], s["n"], s["lay"]
    p = make(cr, n, pre={"orient_by_degree": -1 if kind == "hubs" else 0}, product=(R, g, Ai))
    assert lay["skewed"] == (kind == "hubs")
    if kind != "default":
        p.set_option("compact_record", 192)
    assert p.compact_record(0) == 192
    assert p.pool_set_info(0)["fixed_point"] == 1
    fa, fb = product_truth(R, g, v[Ai[:, 0] - 1], v[Ai[:, 1] - 1])
    vv = _interleaved(v, Ai)
    for fixed in (0, 1):
        set_options(p, psi_fixed_point=fixed)
        psi, acc = p.sweep(v)
        print(f"[measured] {kind}, fixed={fixed}: largest |Ψ − Σ truth| / bound {check_shared(psi, R, g, Ai, v, n, fixed):.3g}")
        sa, sb = _units(R[:, 0], g, fa), _units(R[:, 1], g, fb)
        check_acc(acc, vv, fa, fb, sa, sb + (np.ldexp(1.0, fixed_exponent(R[:, 1]) - 55) if fixed else 0.0))
    p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["padding", "retired"])
def test_edge_prices(cr, oracle, synth, where):
    """ν = 0, +inf, NaN, 2^-1074 on the last first token of a bucket ending on a half-padding record
    (its padding pools repeat that token), or on a retired pool's tokens: padding and retired pools
    add nothing to Ψ or acc, the active pools give the oracle's flows (generic form) or what they
    gave at ordinary prices, on the 192- and 96-pool records, the 32-byte stream and the
    first-generation kernel."""
    s = disjoint18(cr, synth, 40_000, seed=17)
    R, g, Ai, v0, n, lay = s["R"], s["g"], s["Ai"], s["v"], s["n"], s["lay"]
    rule = rec18_rule(lay, Ai, g)
    assert rule["odd"][records(lay)[0] * 96 < 1400].any() and BUCKET_POOLS[0] == 1400
    last = 1399                                          # bucket 0: 1400 pools, 15 chunks
    retired = np.array([700, 5_003, 20_011])
    active = np.ones(len(g), dtype=bool)
    active[retired] = False
    p = make(cr, n, product=(R, g, Ai))
    p.set_active(0, 0, active)
    edge_tokens = [Ai[last, 0] - 1] if where == "padding" else list(Ai[retired].ravel() - 1)
    Ra, ga, Aa = R[active], g[active], Ai[active]
    streams = {"192": dict(use_tma=1, compact_stream=1, compact_record=192),
               "96": dict(use_tma=1, compact_stream=1, compact_record=96),
               "32": dict(use_tma=1, compact_stream=0), "first-generation": dict(use_tma=0)}
    for name, opts in streams.items():
        set_options(p, psi_fixed_point=0, **opts)
        if name in ("192", "96"):
            assert p.compact_record(0) == int(name)
        base, _ = p.sweep(v0)
        for price in (0.0, np.inf, np.nan, 2.0 ** -1074):
            v = v0.copy()
            v[edge_tokens] = price
            Do, Lo = oracle.sweep_product(Ra, ga, Aa, v, threads=8)
            acc_o, _ = oracle.fold(Aa, Do, Lo, v, n)
            gen = generic_pools(v, Aa, Ra, lay["nb"], fixed=False) if name != "first-generation" else \
                np.ones(len(ga), dtype=bool)
            want = base.copy()
            want[Aa[gen, 0] - 1] = Lo[gen, 0] - Do[gen, 0]
            want[Aa[gen, 1] - 1] = Lo[gen, 1] - Do[gen, 1]
            psi, acc = p.sweep(v)
            assert_same(psi, want, (where, name, price))
            assert np.isnan(acc) == np.isnan(acc_o), (where, name, price, acc, acc_o)
            if where == "retired":
                assert np.isfinite(acc)
            if name != "first-generation":              # the fixed-point slice: same NaN / inf pattern
                set_options(p, psi_fixed_point=1)
                psiq, accq = p.sweep(v)
                set_options(p, psi_fixed_point=0)
                assert_same(np.isnan(psiq), np.isnan(psi), (where, name, price, "fixed"))
                assert_same(np.isinf(psiq), np.isinf(psi), (where, name, price, "fixed"))
                assert np.isnan(accq) == np.isnan(acc)
    p.close()


def _moved(prev, psi, R_old, R_new, g, Ai, v):
    """Pools whose state changed: where the truth moved by more than both bounds, Ψ moved too (a
    stale record keeps the old value).  Returns how many such pools there were."""
    a, b = Ai[:, 0] - 1, Ai[:, 1] - 1
    changed = np.any(R_old != R_new, axis=1)
    fo = product_truth(R_old, g, v[a], v[b])
    fn = product_truth(R_new, g, v[a], v[b])
    count = 0
    for k, tok in ((0, a), (1, b)):
        room = _units(R_old[:, k], g, fo[k]) + _units(R_new[:, k], g, fn[k])
        big = changed & (np.abs((fn[k] - fo[k]).astype(np.float64)) > 2 * room)
        assert np.all(np.abs(psi[tok[big]] - prev[tok[big]]) > room[big])
        count += int(np.count_nonzero(big))
    return count


@pytest.mark.gpu
def test_records_follow_state_changes(cr, oracle, synth):
    """One context through reserve pushes (one R2 across a power of two: a new fixed-point scale),
    a materialising sweep and its trades, swaps, retire and restore, appends folded in by compact
    (still fitting, then a fifth fee in one record: 96-pool records) and record sizes switched
    between sweeps; every step read back from the device and checked pool by pool."""
    m = 40_000
    s = disjoint18(cr, synth, m, seed=23)
    R, g, Ai, v, n, lay = s["R"], s["g"], s["Ai"], s["v"].copy(), s["n"], s["lay"]
    nb = lay["nb"]
    p = make(cr, n, product=(R, g, Ai))
    p.set_option("compact_record", 192)
    assert p.compact_record(0) == 192
    key = "product economized, 192-pool record"
    prev = check_disjoint(p, oracle, R, g, Ai, v, nb, key)
    state = R.copy()

    def step(expect_moved=True):
        nonlocal prev, state
        new, act = p.pool_state(0)
        assert p.compact_record(0) == 192
        psi = check_disjoint(p, oracle, new, g, Ai, v, nb, key, active=act)
        if expect_moved:
            assert _moved(prev, psi, state[act], new[act], g[act], Ai[act], v) > 0
        prev, state = psi, new

    rng = np.random.default_rng(5)
    # reserve pushes: small relative changes, and one R2 across a power of two
    upd = np.sort(rng.choice(m, size=400, replace=False))
    newR = state[upd] * (1.0 + rng.uniform(-2.0 ** -10, 2.0 ** -10, size=(len(upd), 2)))
    j = int(np.argmin(np.abs(np.log2(state[upd, 1]) - np.round(np.log2(state[upd, 1])) + 0.5)))
    newR[j, 1] = 2.0 ** np.ceil(np.log2(state[upd[j], 1])) * 1.25     # past the next power of two
    for i, r in zip(upd, newR):
        p.update_reserves(0, int(i), r[None, :])
    step()
    assert fixed_exponent(state[upd[j], 1]) == fixed_exponent(newR[j, 1])
    # a materialising sweep, then its trades
    p.sweep(v, materialize=True)
    p.apply_trades()
    step()
    # swaps: tender 1/64 of the first reserve
    pools = np.sort(rng.choice(m, size=300, replace=False))
    p.execute_swaps(0, pools, np.stack([state[pools, 0] / 64, np.zeros(len(pools))], axis=1))
    step()
    # retire, then restore
    act = np.ones(m, dtype=bool)
    act[rng.choice(m, size=500, replace=False)] = False
    p.set_active(0, 0, act)
    step(expect_moved=False)
    p.set_active(0, 0, np.ones(m, dtype=bool))
    step(expect_moved=False)
    # appends into the last bucket's free second tokens, folded in by compact: still 192-pool records
    a_free = int(Ai[:, 0].max()) + 1
    b_free = int(Ai[:, 1].max()) + 1
    k = 60
    assert b_free + k - 1 <= n and (b_free + k - 2) // nb == (Ai[-1, 1] - 1) // nb
    A2 = np.stack([a_free + np.arange(k), b_free + np.arange(k)], axis=1)
    g2 = np.full(k, g[-1])
    R2 = np.exp2(rng.uniform(-4, 4, size=(k, 2)))
    v[A2[:, 0] - 1] = 1.5
    v[A2[:, 1] - 1] = 0.5
    p.append_product(R2, g2, A2)
    p.compact()
    Ai, g = np.concatenate([Ai, A2]), np.concatenate([g, g2])
    state = np.concatenate([state, R2])
    step(expect_moved=False)
    # one record of five fees: the set falls back to the 96-pool record, the flows stay
    fees = synth.fee_levels()
    A3 = np.stack([a_free + k + np.arange(5), b_free + k + np.arange(5)], axis=1)
    g3 = np.array([f for f in fees[1:] if f not in set(g[-200:])][:5])
    R3 = np.exp2(rng.uniform(-4, 4, size=(5, 2)))
    p.append_product(R3, g3, A3)
    p.compact()
    Ai, g = np.concatenate([Ai, A3]), np.concatenate([g, g3])
    assert p.compact_record(0) == 96
    new, act = p.pool_state(0)
    Aa = Ai[act]
    fa, fb = product_truth(new[act], g[act], v[Aa[:, 0] - 1], v[Aa[:, 1] - 1])
    psi, _ = p.sweep(v)
    assert np.all(error_units(psi[Aa[:, 0] - 1], fa, new[act, 0], g[act]) <= C_PRODUCT_ECON)
    assert np.all(error_units(psi[Aa[:, 1] - 1], fb, new[act, 1], g[act]) <= C_PRODUCT_ECON)
    p.close()
    # record sizes switched between sweeps on one context: 192 -> 96 -> 192, bitwise the same
    p = make(cr, n, product=(s["R"], s["g"], s["Ai"]))
    out = []
    for rec in (192, 96, 192):
        p.set_option("compact_record", rec)
        assert p.compact_record(0) == rec
        out.append(p.sweep(s["v"])[0])
    assert_same(out[1], out[0], "96 after 192")
    assert_same(out[2], out[0], "192 after 96")
    p.close()
