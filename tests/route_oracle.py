"""Host mirror of cfmm_quote_routed_orders / cfmm_execute_routed_orders (include/cfmm_b200.h), for
the tests.  Built on split_oracle.py: its pool classes (find_arb! of the CPU oracle at any two prices
of a pool's tokens), its warp tree and the split's search on the ordinals of the doubles.  A row
sells j for i over the direct pools of {j, i} and, per hub h, the pools of {j, h} then {h, i}; for
each s of the outer search, each hub's t_h is the inner search's smallest ordinal with H_h >= 0.
For ProductTwoCoin and UniV3 pools the mirror gives the device's bits.

  search                      the split's gallop and bisection (0: bracket, 1: top, 2: bottom)
  hub_sums                    N_h, O_h, H_h and the legs of one hub's pools at (s, t)
  route_row                   one row on the current state of its pools (optionally executed)
  quote_routed / replay_routed  rows on their own / in batch order
"""
from __future__ import annotations

import numpy as np

import split_oracle as so
from swap_order_oracle import ORD_MAX, from_ordinal, ordinal

F = np.float64
ORD_MIN = so.ORD_MIN
EXACT_IN, EXACT_OUT = so.EXACT_IN, so.EXACT_OUT
FILLED, LIMIT, UNREACHABLE = so.FILLED, so.LIMIT, so.UNREACHABLE
MAX_OUTER = so.MAX_EVALS             # evaluations of the direct pools: 126 in the search, 1 for the legs
MAX_INNER = 126 * 126 + 1            # evaluations of one hub's pools
MAX_HUBS = 7


def start(e) -> int:
    """o(e) clamped to [o(DBL_MIN), o(DBL_MAX)]; o(DBL_MIN) for a NaN or e < DBL_MIN."""
    return ORD_MIN if not (e >= so.DBL_MIN) else min(ordinal(e), ORD_MAX)


def search(o, test):
    """The split's search from o: (rc, lo, hi).  rc 0: test(lo), not test(hi), hi = lo + 1; rc 1: test
    holds at o(DBL_MAX); rc 2: it fails at o(DBL_MIN) (hi = o(DBL_MIN))."""
    lo = hi = None
    if test(o):
        lo, step = o, 1
        while True:
            if lo == ORD_MAX:
                return 1, lo, hi
            c = ORD_MAX if ORD_MAX - lo <= step else lo + step
            if test(c):
                lo = c
            else:
                hi = c
                break
            step *= 2
    else:
        hi, step = o, 1
        while True:
            if hi == ORD_MIN:
                return 2, lo, hi
            c = ORD_MIN if hi - ORD_MIN <= step else hi - step
            if test(c):
                lo = c
                break
            hi = c
            step *= 2
    while hi - lo > 1:
        mid = lo + ((hi - lo) >> 1)
        if test(mid):
            lo = mid
        else:
            hi = mid
    return 0, lo, hi


def tree(terms):
    """The warp tree over list positions; None adds nothing at its position."""
    p = np.zeros(32, dtype=F)
    for k, t in enumerate(terms):
        if t is not None:
            p[k % 32] = p[k % 32] + F(t)
    for m in (16, 8, 4, 2, 1):
        p = p + p[so._LANE ^ m]
    return float(p[0])


def legs_at(p, prices):
    """(Δ, Λ) of pool p at the prices {token: ν} of its tokens; (0, 0) when retired."""
    if not p.active:
        return np.zeros(2), np.zeros(2)
    return p.legs(np.array([prices[int(a)] for a in p.Ai], dtype=F))


def hub_sums(A, B, j, h, i, s, t):
    """(N_h, O_h, H_h, Δ [n, 2], Λ [n, 2]) of hub h's pools, A = its {j, h} pools, B = its {h, i}."""
    n = len(A) + len(B)
    D, L = np.zeros((n, 2)), np.zeros((n, 2))
    tn, to, th = [], [], []
    for k, p in enumerate(list(A) + list(B)):
        inb = k >= len(A)
        D[k], L[k] = legs_at(p, {h: t, i: 1.0} if inb else {j: s, h: t})
        x = 0 if int(p.Ai[0]) == (h if inb else j) else 1  # the list's first token
        if inb:
            tn.append(None)
            to.append(F(L[k, 1 - x]) - F(D[k, 1 - x]))
            th.append(F(L[k, x]) - F(D[k, x]))
        else:
            tn.append(F(D[k, x]) - F(L[k, x]))
            to.append(None)
            th.append(F(L[k, 1 - x]) - F(D[k, 1 - x]))
    return tree(tn), tree(to), tree(th), D, L


def _max(e, b):
    return b if b > e else e


def route_row(direct, hubs, token_in, token_out, kind, amount, limit=None, execute=False):
    """One row.  direct: the pools of {j, i}; hubs: [(h, A, B)], A the pools of {j, h}, B of {h, i},
    each in pair order.  Returns a dict: paid, received, price, status, hub_price, hub_surplus (per
    hub), D, L (legs in list order: direct, A₁, B₁, A₂, …; zero unless filled), outer (evaluations of
    the direct pools) and inner (per hub, evaluations of its pools)."""
    ti, tj, amt, out = int(token_out), int(token_in), float(amount), int(kind) == EXACT_OUT
    nh = len(hubs)
    n = len(direct) + sum(len(A) + len(B) for _, A, B in hubs)
    res = dict(paid=0.0, received=0.0, price=0.0, status=FILLED, hub_price=[0.0] * nh, hub_surplus=[0.0] * nh,
               D=np.zeros((n, 2)), L=np.zeros((n, 2)), outer=0, inner=[0] * nh)
    if not (amt > 0.0):
        return res
    inf = float("inf")
    e = -inf
    for p in direct:
        if p.active:
            e = _max(e, p.boundary(ti, tj))
    any_active = any(p.active for p in direct)
    tprev = []
    for h, A, B in hubs:
        b1 = b2 = -inf
        for p in A:
            if p.active:
                b1 = _max(b1, p.boundary(h, tj))
        for p in B:
            if p.active:
                b2 = _max(b2, p.boundary(ti, h))
        a1, a2 = any(p.active for p in A), any(p.active for p in B)
        any_active = any_active or a1 or a2
        if a1 and a2:
            with np.errstate(all="ignore"):
                e = _max(e, float(F(b1) * F(b2)))
        tprev.append(start(b2))
    if not any_active:
        res["status"] = UNREACHABLE
        return res
    cache = {}
    bad = False

    def test(c):
        nonlocal bad
        if bad:
            return False
        s = from_ordinal(c)
        N, O, _, _ = so.evaluate(direct, ti, tj, s)
        res["outer"] += 1
        ts, hs = [], []
        for k, (h, A, B) in enumerate(hubs):
            last = {}

            def inner(ct):
                res["inner"][k] += 1
                last[ct] = hub_sums(A, B, tj, h, ti, s, from_ordinal(ct))
                return not (last[ct][2] >= 0.0)

            rc, _, hi = search(tprev[k], inner)
            if rc == 1:
                bad = True
                ts.append(None)
                hs.append(None)
                continue
            tprev[k] = hi
            Nh, Oh, Hh = last[hi][:3]
            N, O = float(F(N) + F(Nh)), float(F(O) + F(Oh))
            ts.append(hi)
            hs.append(Hh)
        cache[c] = (N, O, ts, hs)
        if bad:
            return False
        return O >= amt if out else not (N <= amt)

    rc, lo, hi = search(start(e), test)
    if rc != 0 or bad:
        res["status"] = UNREACHABLE
        return res
    so_ = lo if out else hi
    s = from_ordinal(so_)
    N, O, ts, hs = cache[so_]
    res["price"] = s
    res["hub_price"] = [from_ordinal(t) for t in ts]
    if execute and limit is not None and (N > float(limit) if out else O < float(limit)):
        res["status"] = LIMIT
        return res
    # legs at (s*, t_h*), and on execute the transition of each pool
    parts = []
    _, _, D, L = so.evaluate(direct, ti, tj, s)
    res["outer"] += 1
    parts.append((D, L, [(p, {tj: s, ti: 1.0}) for p in direct]))
    for k, (h, A, B) in enumerate(hubs):
        t = from_ordinal(ts[k])
        _, _, _, D, L = hub_sums(A, B, tj, h, ti, s, t)
        res["inner"][k] += 1
        parts.append((D, L, [(p, {tj: s, h: t}) for p in A] + [(p, {h: t, ti: 1.0}) for p in B]))
    res.update(paid=N, received=O, hub_surplus=list(hs), D=np.concatenate([x[0] for x in parts]).reshape(-1, 2),
               L=np.concatenate([x[1] for x in parts]).reshape(-1, 2))
    if execute:
        for D, L, ps in parts:
            for k, (p, prices) in enumerate(ps):
                if p.active:
                    p.apply(D[k], L[k], np.array([prices[int(a)] for a in p.Ai], dtype=F))
    return res


def _batch(pairs, token_in, token_out, kind, amount, hub_off, hubs, limit, execute):
    """pairs(a, b) -> the pool objects of the pair (pair order)."""
    rows = []
    for r in range(len(token_in)):
        j, i = int(token_in[r]), int(token_out[r])
        hs = [(int(h), pairs(j, int(h)), pairs(int(h), i)) for h in hubs[int(hub_off[r]):int(hub_off[r + 1])]]
        rows.append(route_row(pairs(j, i), hs, j, i, kind[r], amount[r], None if limit is None else limit[r],
                              execute))
    return rows


def quote_routed(pairs, token_in, token_out, kind, amount, hub_off, hubs):
    """cfmm_quote_routed_orders on the host: every row on the current state on its own."""
    return _batch(pairs, token_in, token_out, kind, amount, hub_off, hubs, None, False)


def replay_routed(pairs, token_in, token_out, kind, amount, hub_off, hubs, limit=None):
    """cfmm_execute_routed_orders on the host, in batch order; the pool objects change in place."""
    return _batch(pairs, token_in, token_out, kind, amount, hub_off, hubs, limit, True)
