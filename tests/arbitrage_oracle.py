"""Host mirror of cfmm_quote_arbitrage / cfmm_execute_arbitrage / cfmm_scan_arbitrage
(include/cfmm_b200.h), for the tests.  An arbitrage row is route_oracle's routed row in its
arbitrage mode (j = the other token x, i = the base token p, δ = 0); the scan follows the header's
steps (adjacency, rates, screen, solve, select) in plain Python.  The row repeats route_oracle's
routed row with δ = 0 and its search switched on, from route_oracle's search, start and hub sums.  For ProductTwoCoin and UniV3 pools
the mirror gives the device's bits.

  arb_row                     one arbitrage row (optionally executed): profit, surplus_in, …
  quote_arbitrage / replay_arbitrage   rows on their own / in batch order
  rates                       r(a → b) of every directed pair
  candidates                  the screen's rows (base index, p, x, hubs) in (base index, x) order
  scan                        cfmm_scan_arbitrage: (found, rows)
"""
from __future__ import annotations

import numpy as np

import route_oracle as ro

F = np.float64
FILLED, LIMIT, UNREACHABLE = ro.FILLED, ro.LIMIT, ro.UNREACHABLE
SCREEN = 1.0 - 2.0 ** -40
MAX_HUBS = ro.MAX_HUBS


def arb_row(direct, hubs, base, other, min_profit=None, execute=False):
    """One row over direct = the pools of {x, p} and hubs = [(y, pools of {x, y}, pools of {y, p})], each
    in pair order: route_oracle.route_row's exact-in row with j = x, i = p and δ = 0, except that the
    search runs (enough(s) = N(s) > 0) and a row without a pool of {x, p} is unreachable.  Returns a
    dict: profit = O(s*), surplus_in = 0.0 − N(s*), price, status, hub_price, hub_surplus (per hub),
    D, L (legs in list order; zero unless filled), outer and inner (evaluation counts)."""
    ti, tj = int(base), int(other)
    nh = len(hubs)
    n = len(direct) + sum(len(A) + len(B) for _, A, B in hubs)
    res = dict(profit=0.0, surplus_in=0.0, price=0.0, status=FILLED, hub_price=[0.0] * nh, hub_surplus=[0.0] * nh,
               D=np.zeros((n, 2)), L=np.zeros((n, 2)), outer=0, inner=[0] * nh)
    if not direct:
        res["status"] = UNREACHABLE
        return res
    inf = float("inf")
    e = -inf
    for p in direct:
        if p.active:
            e = ro._max(e, p.boundary(ti, tj))
    any_active = any(p.active for p in direct)
    tprev = []
    for h, A, B in hubs:
        b1 = b2 = -inf
        for p in A:
            if p.active:
                b1 = ro._max(b1, p.boundary(h, tj))
        for p in B:
            if p.active:
                b2 = ro._max(b2, p.boundary(ti, h))
        a1, a2 = any(p.active for p in A), any(p.active for p in B)
        any_active = any_active or a1 or a2
        if a1 and a2:
            with np.errstate(all="ignore"):
                e = ro._max(e, float(F(b1) * F(b2)))
        tprev.append(ro.start(b2))
    if not any_active:
        res["status"] = UNREACHABLE
        return res
    cache = {}
    bad = False

    def test(c):
        nonlocal bad
        if bad:
            return False
        s = ro.from_ordinal(c)
        N, O, _, _ = ro.so.evaluate(direct, ti, tj, s)
        res["outer"] += 1
        ts, hs = [], []
        for k, (h, A, B) in enumerate(hubs):
            last = {}

            def inner(ct):
                res["inner"][k] += 1
                last[ct] = ro.hub_sums(A, B, tj, h, ti, s, ro.from_ordinal(ct))
                return not (last[ct][2] >= 0.0)

            rc, _, hi = ro.search(tprev[k], inner)
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
        return not (N <= 0.0)  # N > 0, a NaN counts as true

    rc, lo, hi = ro.search(ro.start(e), test)
    if rc != 0 or bad:
        res["status"] = UNREACHABLE
        return res
    s = ro.from_ordinal(hi)
    N, O, ts, hs = cache[hi]
    res["price"] = s
    res["hub_price"] = [ro.from_ordinal(t) for t in ts]
    if execute and min_profit is not None and O < float(min_profit):
        res["status"] = LIMIT
        return res
    parts = []
    _, _, D, L = ro.so.evaluate(direct, ti, tj, s)
    parts.append((D, L, [(p, {tj: s, ti: 1.0}) for p in direct]))
    for k, (h, A, B) in enumerate(hubs):
        t = ro.from_ordinal(ts[k])
        _, _, _, D, L = ro.hub_sums(A, B, tj, h, ti, s, t)
        parts.append((D, L, [(p, {tj: s, h: t}) for p in A] + [(p, {h: t, ti: 1.0}) for p in B]))
    res.update(profit=O, surplus_in=float(F(0.0) - F(N)), hub_surplus=list(hs),
               D=np.concatenate([x[0] for x in parts]).reshape(-1, 2),
               L=np.concatenate([x[1] for x in parts]).reshape(-1, 2))
    if execute:
        for D, L, ps in parts:
            for k, (p, prices) in enumerate(ps):
                if p.active:
                    p.apply(D[k], L[k], np.array([prices[int(a)] for a in p.Ai], dtype=F))
    return res


def _batch(pairs, base, other, hub_off, hubs, min_profit, execute):
    """pairs(a, b) -> the pool objects of the pair (pair order)."""
    rows = []
    for r in range(len(base)):
        p, x = int(base[r]), int(other[r])
        hs = [(int(y), pairs(x, int(y)), pairs(int(y), p)) for y in hubs[int(hub_off[r]):int(hub_off[r + 1])]]
        rows.append(arb_row(pairs(x, p), hs, p, x, None if min_profit is None else min_profit[r], execute))
    return rows


def quote_arbitrage(pairs, base, other, hub_off, hubs):
    """cfmm_quote_arbitrage on the host: every row on the current state on its own."""
    return _batch(pairs, base, other, hub_off, hubs, None, False)


def replay_arbitrage(pairs, base, other, hub_off, hubs, min_profit=None):
    """cfmm_execute_arbitrage on the host, in batch order; the pool objects change in place.  A null
    min_profit is 0."""
    if min_profit is None:
        min_profit = np.zeros(len(base))
    return _batch(pairs, base, other, hub_off, hubs, min_profit, True)


def rates(by_pair):
    """{(a, b): r(a → b)} for every pair {a, b} of by_pair ({(lo, hi): pools}) and both directions: the
    largest start boundary over the active pools with a in j's role, NaNs ignored, 0 when none."""
    r = {}
    for (a, b), pools in by_pair.items():
        for u, v in ((a, b), (b, a)):
            best = 0.0
            for p in pools:
                if p.active:
                    x = p.boundary(v, u)
                    if x > best:
                        best = x
            r[(u, v)] = best
    return r


def _passing(t1, t2):
    q1, q2 = t1 > SCREEN, t2 > SCREEN
    if not (q1 or q2):
        return None
    return t1 if not q2 else t2 if not q1 else (t2 if t2 > t1 else t1)


def candidates(by_pair, base, max_hubs):
    """The screen: [(b, p, x, hubs)] in (base index, x) order."""
    r = rates(by_pair)
    nbr = {}
    for a, b in by_pair:
        nbr.setdefault(a, set()).add(b)
        nbr.setdefault(b, set()).add(a)
    out = []
    with np.errstate(all="ignore"):
        for bi, p in enumerate(int(t) for t in base):
            for x in sorted(nbr.get(p, ())):
                pair_pass = float(F(r[(p, x)]) * F(r[(x, p)])) > SCREEN
                tri = []
                for y in sorted(nbr[p] & nbr[x]):
                    t1 = float((F(r[(p, x)]) * F(r[(x, y)])) * F(r[(y, p)]))
                    t2 = float((F(r[(p, y)]) * F(r[(y, x)])) * F(r[(x, p)]))
                    s = _passing(t1, t2)
                    if s is not None:
                        tri.append((-s, y))
                if pair_pass or tri:
                    tri.sort()
                    out.append((bi, p, x, [y for _, y in tri[:max_hubs]]))
    return out


def scan(by_pair, pairs, base, min_profit, max_hubs, cap=None, memo=None):
    """cfmm_scan_arbitrage on the host: (found, [dict(base, other, hubs, profit, price)]) with the
    first min(found, cap) rows in (base index, profit descending, x ascending) order.  memo (a dict)
    keeps solved rows across calls on the same state."""
    kept = []
    memo = {} if memo is None else memo
    for bi, p, x, hs in candidates(by_pair, base, max_hubs):
        key = (p, x, tuple(hs))
        if key not in memo:
            memo[key] = arb_row(pairs(x, p), [(y, pairs(x, y), pairs(y, p)) for y in hs], p, x)
        row = memo[key]
        if row["status"] == FILLED and row["profit"] >= float(min_profit[bi]):
            kept.append((bi, -row["profit"], x, dict(base=p, other=x, hubs=hs, profit=row["profit"],
                                                     price=row["price"])))
    kept.sort(key=lambda k: k[:3])
    rows = [k[3] for k in kept]
    return len(rows), rows if cap is None else rows[:cap]
