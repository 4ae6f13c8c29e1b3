"""The 50-digit optimality certificate of order_certificate.py for arbitrage rows
(cfmm_quote_arbitrage / cfmm_execute_arbitrage), for the tests.

An arbitrage row (base p, other x, hubs y) is the routed exact-in row j = x, i = p with δ = 0 that
runs its search.  Weak duality at the device's (s*, t_y*) with δ = 0 bounds the profit of every
cycle through the row's pools that leaves neither x nor a hub short:

    profit ≤ UB = Σ_k π_k(ν*),

and the row's profit must reach UB less order_certificate's allowance (rounding per trading pool,
one ordinal of s*, one ordinal of each t_y*).  The checks are order_certificate.certify_row's for an
exact-in row with δ = 0: feasible legs, retired pools idle, the sums equal to the exact sums of the
legs within the warp tree's rounding, N(s*) ≤ 0, the ordinal checks (N(pred s*) > 0,
H_y(pred t_y*) < 0, in 50 digits) and the bound.  The row's outputs are mapped to a routed row's:
paid = N(s*) = −surplus_in, received = profit.  An unreachable row is checked for its legs only
(with δ = 0 a row is unreachable when it has no pool of {x, p} or no active pool).
"""
from __future__ import annotations

import mpmath as mp
import numpy as np

import order_certificate as oc
from order_certificate import C_ORD, C_ROUND, DBL_MIN, DPS, EPS, FILLED, LIMIT, UNREACHABLE


def certify_arbitrage(row, out, nested=True, limit=None):
    """Certify one arbitrage row.  row: order_certificate.Row with j = x, i = p; out: profit,
    surplus_in, price, status, hub_price [nh], hub_surplus [nh], D, L [n, 2] in list order; limit: the
    row's min_profit when it reverted.  Returns dict(status, gap, allowance, rounding, bound, kinds)
    (gap None for rows without a trade) and asserts the checks."""
    with mp.workdps(DPS):
        return _certify(row, out, nested, limit)


def _certify(row, out, nested, limit):
    pools, nh = row.pools, len(row.hubs)
    D, L = np.asarray(out["D"], float).reshape(-1, 2), np.asarray(out["L"], float).reshape(-1, 2)
    assert len(D) == len(pools) and len(L) == len(pools), "the legs are not the row's pools"
    st = int(out["status"])
    res = dict(status=st, gap=None, allowance=None, kinds={p.kind for p in pools if p.active})
    if st != FILLED:
        assert not D.any() and not L.any(), "legs on a row that did not fill"
        assert out["profit"] == 0.0 and out["surplus_in"] == 0.0
    if st == UNREACHABLE:
        return res
    paid, received = -float(out["surplus_in"]), float(out["profit"])
    s = float(out["price"])
    ts = [float(x) for x in out["hub_price"]]
    assert s > 0.0 and all(t > 0.0 for t in ts)
    ms = oc._m(s)
    prices = lambda k: {row.j: ms, row.i: mp.mpf(1), **({row.hubs[k][0]: oc._m(ts[k])} if k is not None else {})}
    owner = [None] * len(row.direct) + [k for k, (_, A, B) in enumerate(row.hubs) for _ in A + B]
    # 1. legs feasible; the value scales and Σπ at ν*
    pi, allow_r, scale = mp.mpf(0), mp.mpf(0), {}
    for n, p in enumerate(pools):
        d, l = D[n], L[n]
        if not p.active:
            assert not d.any() and not l.any(), ("a retired pool traded", n)
            continue
        assert np.all(np.isfinite(d)) and np.all(np.isfinite(l)) and np.all(d >= 0.0) and np.all(l >= 0.0), n
        pr = prices(owner[n])
        nu = [pr[p.Ai[0]], pr[p.Ai[1]]]
        _, _, v, _ = oc.response(p, nu)
        pi += v
        V = oc.value_scale(p, nu, d, l, bool(d.any() or l.any()))
        a = 0 if nu[0] * oc._m(d[0]) >= nu[1] * oc._m(d[1]) else 1
        assert oc._m(d[1 - a]) <= C_ROUND[p.kind] * EPS * V[1 - a], ("both sides tendered", n)
        X = oc._u3_base(p) if p.kind == "univ3" else [oc._m(p.R[0]), oc._m(p.R[1])]
        for sd in (0, 1):
            scale[p.Ai[sd]] = scale.get(p.Ai[sd], mp.mpf(0)) + C_ROUND[p.kind] * (V[sd] + X[sd]) / 64
        allow_r += C_ROUND[p.kind] * EPS * (nu[0] * V[0] + nu[1] * V[1])
        fx = oc.forward(p, a, oc._m(d[a]))
        tol = C_ROUND[p.kind] * EPS
        assert oc._m(l[1 - a]) <= fx + tol * V[1 - a], ("pays out more than F(Δ)", n, float(l[1 - a]), float(fx))
        assert oc._m(l[a]) <= tol * V[a], ("pays out on the tendered side", n)
    # 2. accounting: the device's sums against the exact sums of its legs
    tn, to, th = [], [], [[] for _ in range(nh)]
    for n, p in enumerate(pools):
        k = owner[n]
        if row.j in p.Ai:
            x = p.Ai.index(row.j)
            tn.append(D[n, x] - L[n, x])
        if row.i in p.Ai:
            x = p.Ai.index(row.i)
            to.append(L[n, x] - D[n, x])
        if k is not None:
            x = p.Ai.index(row.hubs[k][0])
            th[k].append(L[n, x] - D[n, x])
    if st == FILLED:
        paid_x, recv_x = oc._exact_sum(tn), oc._exact_sum(to)
        assert abs(float(oc._frac(paid) - paid_x)) <= oc._tree_bound(len(tn), nh, tn), "N is not the sum of the legs"
        assert abs(float(oc._frac(received) - recv_x)) <= oc._tree_bound(len(to), nh, to), "profit is not the sum"
        for k in range(nh):
            hx = oc._exact_sum(th[k])
            assert abs(float(oc._frac(out["hub_surplus"][k]) - hx)) <= oc._tree_bound(len(th[k]), 0, th[k]), \
                ("hub surplus", k)
            assert out["hub_surplus"][k] >= 0.0, ("hub short", k)
        assert paid <= 0.0, "the row takes x from the trader"
    # 3. the one-ordinal terms and the ordinal checks (50 digits)
    sn = float(np.nextafter(s, 0.0))
    if nested and nh:
        at_s, at_n = row.sums_resolved(s, ts), row.sums_resolved(sn, ts)
    else:
        at_s, at_n = row.sums(s, ts), row.sums(sn, ts)
    rnd = lambda tok: C_ORD * EPS * scale.get(tok, mp.mpf(0))
    step = ms * max(at_n[0] - at_s[0], 0)
    if nested or not nh:
        assert at_n[0] > -rnd(row.j), ("the ordinal below s* takes x from the pools", float(at_n[0]))
    hstep = mp.mpf(0)
    H_s = row.sums(s, ts)[2]
    for k, (h, _, _) in enumerate(row.hubs):
        t = ts[k]
        if t <= DBL_MIN:
            continue
        Hp = row.hub_net(k, ms, oc._m(float(np.nextafter(t, 0.0))))
        assert Hp < rnd(h), ("the ordinal below t_y* leaves hub y short of nothing", k, float(Hp))
        hstep += oc._m(t) * max(H_s[k] - Hp, 0)
    allowance = allow_r + step + hstep
    # 4. the bound: profit ≤ Σπ_k(ν*)
    res.update(allowance=float(allowance), rounding=float(allow_r), bound=float(pi))
    if st == LIMIT:
        assert float(limit) > float(pi - allowance), ("a min_profit the optimum meets", float(limit), float(pi))
        return res
    gap = pi - oc._mf(recv_x)
    res.update(gap=float(gap))
    assert -allow_r <= gap <= allowance, ("not optimal", float(gap), float(allowance), received)
    return res
