"""A 50-digit optimality certificate for split and routed orders (cfmm_quote_split_orders,
cfmm_quote_routed_orders and their executes), for the tests.  It works from each pool's trading
function in mpmath and shares nothing with the host mirrors (split_oracle.py, route_oracle.py) or
the CPU oracle: a mistake common to a kernel and its mirror does not pass it.

Pools are plain state (Pool: reserves, fee, weights, price and ladder, active flag) with their
tokens in ingest order.  Per pool and direction (tender side a, receive side 1 − a):

  forward(p, a, x)     the exact amount out for a tender x, fee on the input (δ = γx)
  best(p, a, ν)        max_x ν_out·F(x) − ν_in·x, from the first-order condition: the pool's post-trade
                       marginal price reaches ν_in/(γ·ν_out) (closed forms for the two-coin types, a
                       walk to the target price for UniV3)
  response(p, ν)       the optimal flows (Δ, Λ) at ν and π(ν) = their value, the larger direction
  depth(p, a)          the most input the pool absorbs and the most output it gives tendering side a

Weak duality.  A row sells j for i over the direct pools {j, i} and, per hub h, the pools {j, h}
and {h, i}.  At any prices ν (ν_i = 1, ν_j = s, ν_h = t_h) each pool's trade is worth at most
π_k(ν), so every route that pays at most δ of j and leaves no hub short receives at most

    UB(δ) = s·δ + Σ_k π_k(ν),

and every route that delivers at least y pays at least (y − Σ_k π_k)/s.  certify_row evaluates the
bound at the device's (s*, t_h*) and compares it with the exact (fractions.Fraction) sums of the
device's legs: received_exact ≥ UB − allowance for exact-in, paid_exact ≤ LB + allowance/s* for
exact-out.  The legs at ν* are the pools' optimal responses, so received − s*·paid + Σ t_h·H_h =
Σ_k ν*·(Λ_k − Δ_k), and the gap is s*·(δ − paid) (exact-out: received − y) + Σ_h t_h*·H_h plus the
rounding of the legs.

Error model of the allowance (in value units of token i, ε = 2⁻⁵²):

  * rounding: c_type·ε·V_k per pool that trades (in the device's legs or the 50-digit response),
    V_k = Σ_side ν_side·(X_side + |Δ_side| + |Λ_side|), X the reserves for the two-coin types and,
    for UniV3, the virtual reserves √(k/p), √(kp) at both ends of every tick the walk crosses.
    c = 64 for ProductTwoCoin and UniV3: each leg is a difference of reserve-sized terms
    (√(γmk) − R, a sum of per-tick terms), a few ulp of V each, and the warp tree adds a few
    more.  c = 256 for GeometricMeanTwoCoin: CUDA's pow is within 2 ulp and each leg chains two of
    them, one raised to 1/(η+1) and one multiplied into a reserve-sized difference.
  * one ordinal of s: s*·(N(pred s*) − N(s*)) for exact-in, O(s*) − O(succ s*) for exact-out, with
    N, O the row's j intake and i output in 50 digits (each hub's t re-solved at that s when nested),
    because the search stops within one ordinal of the boundary.
  * one ordinal of each t_h: t_h*·(H_h(t_h*) − H_h(pred t_h*)), 50-digit hub nets at s*.

A gap below −(rounding) fails: fp64 legs may sit an ulp outside the curve, not more.  The ordinal
checks test the device's searches against the 50-digit responses: exact-in N(pred s*) > δ, exact-
out O(succ s*) < y and H_h(pred t_h*) < 0, each up to C_ORD·ε times the scales of the pools summed.

UNREACHABLE rows are certified against the depth of the row's pools: exact-out y above the
reachable output (direct pools plus, per hub, the most its {h, i} pools deliver from all the h its
{j, h} pools can give) must be UNREACHABLE and y below it by a relative REACH_MARGIN must fill;
exact-in likewise with the input the direct and {j, h} pools absorb when that is finite, and, with
no hubs, N(DBL_MIN) ≤ δ when it is not (the search's range ends there).
"""
from __future__ import annotations

from fractions import Fraction

import mpmath as mp
import numpy as np

EPS = 2.0 ** -52
DPS = 50
EXACT_IN, EXACT_OUT = 0, 1
FILLED, LIMIT, UNREACHABLE = 0, 1, 2
DBL_MIN = 2.0 ** -1022
C_ROUND = {"product": 64, "geomean": 256, "univ3": 64}
C_ORD = 16          # rounding of the fp64 sums N, O, H against the 50-digit ones, per unit of scale
REACH_MARGIN = 1e-12


def _m(x):
    return mp.mpf(float(x))


def _frac(x):
    return Fraction(float(x))


class Pool:
    """One pool's plain state; Ai are its two tokens in ingest order."""

    def __init__(self, kind, Ai, g, R=None, w=None, price=None, lt=None, lq=None, active=True):
        self.kind, self.Ai, self.g, self.active = kind, (int(Ai[0]), int(Ai[1])), float(g), bool(active)
        self.R = None if R is None else (float(R[0]), float(R[1]))
        self.w = None if w is None else (float(w[0]), float(w[1]))
        self.price = None if price is None else float(price)
        self.lt = None if lt is None else [float(x) for x in lt]
        self.lq = None if lq is None else [float(x) for x in lq]
        self._cache = {}


def product(R, g, Ai, active=True):
    return Pool("product", Ai, g, R=R, active=active)


def geomean(R, g, w, Ai, active=True):
    return Pool("geomean", Ai, g, R=R, w=w, active=active)


def univ3(price, lt, lq, g, Ai, active=True):
    return Pool("univ3", Ai, g, price=price, lt=lt, lq=lq, active=active)


# ---- UniV3: the ladder in 50 digits ----------------------------------------------------------
def _ticks(p):
    """[(lo, hi, k)] of ticks 1 … n (tick idx spans (lower_ticks[idx], lower_ticks[idx − 1]], the last
    down to 0) and the current tick cur = #(lower_ticks ≥ price)."""
    n = len(p.lt)
    T = [(_m(p.lt[i]) if i < n else mp.mpf(0), _m(p.lt[i - 1]), _m(p.lq[i - 1])) for i in range(1, n + 1)]
    cur = sum(1 for x in p.lt if x >= p.price)
    assert cur >= 1, "a UniV3 price above its ladder"
    return T, cur


def _walk(p, a, target=None, budget=None):
    """Move the price from p.price: down tendering token 0 (a = 0), up tendering token 1, to target
    (None: as far as the ladder goes) or until the fee-adjusted input reaches budget.  Returns
    (input after the fee, output, (X₀, X₁) virtual reserves of the ticks crossed)."""
    T, cur = _ticks(p)
    q = _m(p.price)
    xin, yout, sc = mp.mpf(0), mp.mpf(0), [mp.mpf(0), mp.mpf(0)]
    for idx in (range(cur, len(T) + 1) if a == 0 else range(cur, 0, -1)):
        lo, hi, k = T[idx - 1]
        if a == 0:
            ps = q if idx == cur else hi
            if target is not None and target >= ps:
                break
            pe = lo if target is None else max(target, lo)
        else:
            ps = q if idx == cur else lo
            if target is not None and target <= ps:
                break
            pe = hi if target is None else min(target, hi)
        if k > 0 and pe != ps:  # (a price at the edge of its tick moves on to the next)
            if a == 0:
                cap = mp.inf if pe == 0 else mp.sqrt(k / pe) - mp.sqrt(k / ps)
                if budget is not None and budget - xin < cap:
                    pe = k / (mp.sqrt(k / ps) + (budget - xin)) ** 2
                    cap = budget - xin
                out = mp.sqrt(k * ps) - mp.sqrt(k * pe)
            else:
                cap = mp.sqrt(k * pe) - mp.sqrt(k * ps)
                if budget is not None and budget - xin < cap:
                    pe = ((mp.sqrt(k * ps) + (budget - xin)) ** 2) / k
                    cap = budget - xin
                out = mp.sqrt(k / ps) - mp.sqrt(k / pe)
            xin += cap
            yout += out
            if pe > 0:
                sc[0] += mp.sqrt(k / ps) + mp.sqrt(k / pe)
                sc[1] += mp.sqrt(k * ps) + mp.sqrt(k * pe)
            if budget is not None and xin >= budget:
                break
        if (a == 0 and pe > lo) or (a == 1 and pe < hi):
            break
    return xin, yout, sc


def _u3_base(p):
    """Virtual reserves around the current price (the rounding scale of a pool at its boundary)."""
    T, cur = _ticks(p)
    q = _m(p.price)
    ks = [T[i][2] for i in range(max(cur - 2, 0), min(cur + 1, len(T)))]
    kk = max(ks)
    return [mp.sqrt(kk / q), mp.sqrt(kk * q)]


# ---- per pool --------------------------------------------------------------------------------
def forward(p, a, x):
    """The amount of token 1 − a out for a tender x of token a (fee on the input)."""
    with mp.workdps(DPS):
        x = mp.mpf(x) if not isinstance(x, mp.mpf) else x
        if not (x > 0):
            return mp.mpf(0)
        d = _m(p.g) * x
        if p.kind == "univ3":
            return _walk(p, a, budget=d)[1]
        Ri, Ro = _m(p.R[a]), _m(p.R[1 - a])
        eta = mp.mpf(1) if p.kind == "product" else _m(p.w[a]) / _m(p.w[1 - a])
        return Ro * (1 - (Ri / (Ri + d)) ** eta)


def best(p, a, n_in, n_out):
    """(x, y, scale): the tender x of side a maximising n_out·F(x) − n_in·x, its output y, and the
    pool's value scale in token units per side."""
    g = _m(p.g)
    if p.kind == "univ3":
        target = n_in / (g * n_out) if a == 0 else g * n_out / n_in
        xin, y, sc = _walk(p, a, target=target)
        return xin / g, y, sc
    Ri, Ro = _m(p.R[a]), _m(p.R[1 - a])
    sc = [_m(p.R[0]), _m(p.R[1])]
    if p.kind == "product":
        S = mp.sqrt(g * n_out * Ro * Ri / n_in)
        eta = mp.mpf(1)
    else:
        eta = _m(p.w[a]) / _m(p.w[1 - a])
        S = (n_out * g * eta * Ro * Ri ** eta / n_in) ** (1 / (eta + 1))
    if not (S > Ri):
        return mp.mpf(0), mp.mpf(0), sc
    return (S - Ri) / g, Ro * (1 - (Ri / S) ** eta), sc


def response(p, nu):
    """(Δ [2], Λ [2], π, scale [2]) of pool p at the prices nu of its tokens (ingest order)."""
    key = (mp.nstr(nu[0], 60), mp.nstr(nu[1], 60))
    if key in p._cache:
        return p._cache[key]
    with mp.workdps(DPS):
        D, L = [mp.mpf(0), mp.mpf(0)], [mp.mpf(0), mp.mpf(0)]
        val, sc = mp.mpf(0), None
        for a in (0, 1):
            x, y, s = best(p, a, nu[a], nu[1 - a])
            v = nu[1 - a] * y - nu[a] * x
            if x > 0 and v > val:
                D, L = [mp.mpf(0), mp.mpf(0)], [mp.mpf(0), mp.mpf(0)]
                D[a], L[1 - a], val, sc = x, y, v, s
        out = (D, L, val, sc)
    p._cache[key] = out
    return out


def depth(p, a):
    """(most input of side a absorbed, most output of side 1 − a given), 50 digits (inf: no bound)."""
    with mp.workdps(DPS):
        if p.kind == "univ3":
            xin, y, _ = _walk(p, a)
            return xin / _m(p.g), y
        return mp.inf, _m(p.R[1 - a])


def value_scale(p, nu, D, L, dev_trades):
    """V of the error model, per side in token units: [X₀ + |Δ₀| + |Λ₀|, X₁ + …]; zero when neither the
    device nor the 50-digit response trades."""
    d, l, _, sc = response(p, nu)
    if sc is None:
        if not dev_trades:
            return [mp.mpf(0), mp.mpf(0)]
        sc = _u3_base(p) if p.kind == "univ3" else [_m(p.R[0]), _m(p.R[1])]
    return [sc[s] + abs(d[s]) + abs(l[s]) + abs(_m(D[s])) + abs(_m(L[s])) for s in (0, 1)]


# ---- a row in 50 digits ----------------------------------------------------------------------
class Row:
    """The pools of one row: direct {j, i} and per hub (h, A = {j, h}, B = {h, i}), in list order."""

    def __init__(self, direct, hubs, j, i):
        self.direct, self.hubs, self.j, self.i = list(direct), [(int(h), list(A), list(B)) for h, A, B in hubs], int(j), int(i)
        self.pools = self.direct + [p for _, A, B in self.hubs for p in A + B]

    def _flows(self, pools, prices):
        """{token: Σ (Λ − Δ)} of the active pools at prices."""
        tot = {}
        for p in pools:
            if not p.active:
                continue
            D, L, _, _ = response(p, [prices[p.Ai[0]], prices[p.Ai[1]]])
            for s in (0, 1):
                tot[p.Ai[s]] = tot.get(p.Ai[s], mp.mpf(0)) + L[s] - D[s]
        return tot

    def hub_net(self, k, s, t):
        h, A, B = self.hubs[k]
        with mp.workdps(DPS):
            return self._flows(A + B, {self.j: _m(s) if not isinstance(s, mp.mpf) else s, h: t, self.i: mp.mpf(1)}).get(h, mp.mpf(0))

    def hub_root(self, k, s, t0):
        """The smallest t with H_h(s, t) ≥ 0 in 50 digits, searched from t0 (H is nondecreasing in t)."""
        with mp.workdps(DPS):
            f = lambda t: self.hub_net(k, s, t)
            b = _m(max(t0, DBL_MIN))
            if f(b) >= 0:
                a, r = b, mp.mpf(2) ** -40
                while True:
                    a = b * (1 - r) if r < 1 else b / (1 + r)
                    if a < DBL_MIN:
                        a = _m(DBL_MIN)
                        if f(a) >= 0:
                            return a
                        break
                    if f(a) < 0:
                        break
                    b, r = a, r * 16
            else:
                a, r = b, mp.mpf(2) ** -40
                while True:
                    b = a * (1 + r)
                    if f(b) >= 0:
                        break
                    a, r = b, r * 16
            fa, fb = f(a), f(b)
            side = 0
            for _ in range(400):  # Illinois on [a, b], f(a) < 0 <= f(b)
                if b - a <= b * mp.mpf(10) ** -(DPS - 8):
                    break
                c = b - fb * (b - a) / (fb - fa) if fb != fa else (a + b) / 2
                if not (a < c < b):
                    c = (a + b) / 2
                fc = f(c)
                if fc >= 0:
                    b, fb = c, fc
                    if side == 1:
                        fa /= 2
                    side = 1
                else:
                    a, fa = c, fc
                    if side == -1:
                        fb /= 2
                    side = -1
            return b

    def sums(self, s, ts):
        """(N, O, [H_h]) in 50 digits at ν_j = s, ν_h = ts[h], ν_i = 1 (s, ts mp or float)."""
        with mp.workdps(DPS):
            s = s if isinstance(s, mp.mpf) else _m(s)
            f = self._flows(self.direct, {self.j: s, self.i: mp.mpf(1)})
            N, O = -f.get(self.j, mp.mpf(0)), f.get(self.i, mp.mpf(0))
            H = []
            for k, (h, A, B) in enumerate(self.hubs):
                t = ts[k] if isinstance(ts[k], mp.mpf) else _m(ts[k])
                fa = self._flows(A, {self.j: s, h: t})
                fb = self._flows(B, {h: t, self.i: mp.mpf(1)})
                N -= fa.get(self.j, mp.mpf(0))
                O += fb.get(self.i, mp.mpf(0))
                H.append(fa.get(h, mp.mpf(0)) + fb.get(h, mp.mpf(0)))
            return N, O, H

    def sums_resolved(self, s, t0):
        """sums at s with every hub's t re-solved in 50 digits (from the starting points t0)."""
        with mp.workdps(DPS):
            s = _m(s)
            ts = [self.hub_root(k, s, t0[k]) for k in range(len(self.hubs))]
            return self.sums(s, ts)

    def reach_out(self):
        """The most i the row's pools can deliver for any amount of j."""
        with mp.workdps(DPS):
            tot = mp.mpf(0)
            for p in self.direct:
                if p.active:
                    tot += depth(p, p.Ai.index(self.j))[1]
            for h, A, B in self.hubs:
                X = sum((depth(p, p.Ai.index(self.j))[1] for p in A if p.active), mp.mpf(0))
                tot += _deliver([p for p in B if p.active], h, X)
            return tot

    def reach_in(self):
        """The most j the direct and {j, h} pools absorb (inf: no bound)."""
        with mp.workdps(DPS):
            return sum((depth(p, p.Ai.index(self.j))[0] for p in self.direct + [p for _, A, _ in self.hubs for p in A]
                        if p.active), mp.mpf(0))


def _deliver(B, h, X):
    """max Σ F_b(x_b) over the pools B selling h, Σ x_b ≤ X: water-filling on the price μ of h."""
    if not B or X == 0:
        return mp.mpf(0)
    full = sum(depth(p, p.Ai.index(h))[1] for p in B)
    cap = sum(depth(p, p.Ai.index(h))[0] for p in B)
    if X == mp.inf or cap <= X:
        return full
    take = lambda lm: sum(best(p, p.Ai.index(h), mp.exp(lm), mp.mpf(1))[0] for p in B)
    lo, hi = mp.mpf(-2000), mp.mpf(2000)  # log μ: take(lo) ≥ X > take(hi)
    for _ in range(120):
        mid = (lo + hi) / 2
        if take(mid) >= X:
            lo = mid
        else:
            hi = mid
    return sum(best(p, p.Ai.index(h), mp.exp(hi), mp.mpf(1))[1] for p in B)


# ---- the certificate -------------------------------------------------------------------------
def _exact_sum(xs):
    return sum((_frac(x) for x in xs), Fraction(0))


def _tree_bound(n, extra, terms):
    """Rounding bound of the device's fixed-order sum of n terms (lane loop, then 5 shuffle levels,
    then `extra` further additions), ε per level on the sum of |terms|."""
    return (-(-n // 32) + 5 + 1 + extra) * EPS * float(sum(abs(float(x)) for x in terms))


def _mf(x):
    return mp.mpf(x.numerator) / x.denominator


def certify_row(row, kind, amount, out, nested=True, limit=None):
    """Certify one row.  row: Row; out: dict of the device's (or the mirror's) outputs — paid,
    received, price, status, hub_price [nh], hub_surplus [nh], D, L [n, 2] in list order.  Returns a
    dict with gap and allowance (value units of i; None for rows without a trade) and asserts the
    checks of the module docstring."""
    with mp.workdps(DPS):
        return _certify(row, int(kind), float(amount), out, nested, limit)


def _certify(row, kind, amount, out, nested, limit):
    pools, nh = row.pools, len(row.hubs)
    D, L = np.asarray(out["D"], float).reshape(-1, 2), np.asarray(out["L"], float).reshape(-1, 2)
    assert len(D) == len(pools) and len(L) == len(pools), "the legs are not the row's pools"
    st = int(out["status"])
    res = dict(status=st, gap=None, allowance=None, kinds={p.kind for p in pools if p.active})
    if st != FILLED or amount == 0.0:
        assert not D.any() and not L.any(), "legs on a row that did not fill"
        if amount == 0.0:
            assert st == FILLED and out["paid"] == 0.0 and out["received"] == 0.0
            return res
    if st == UNREACHABLE:
        _unreachable(row, kind, amount)
        return res
    if st == FILLED:
        _reachable(row, kind, amount)
    s = float(out["price"])
    ts = [float(x) for x in out["hub_price"]]
    assert s > 0.0 and all(t > 0.0 for t in ts)
    ms = _m(s)
    prices = lambda p, k: {row.j: ms, row.i: mp.mpf(1), **({row.hubs[k][0]: _m(ts[k])} if k is not None else {})}
    owner = [None] * len(row.direct) + [k for k, (_, A, B) in enumerate(row.hubs) for _ in A + B]
    # 1. legs feasible; the value scales and Σπ at ν*
    pi, allow_r, scale = mp.mpf(0), mp.mpf(0), {}
    for n, p in enumerate(pools):
        d, l = D[n], L[n]
        if not p.active:
            assert not d.any() and not l.any(), ("a retired pool traded", n)
            continue
        assert np.all(np.isfinite(d)) and np.all(np.isfinite(l)) and np.all(d >= 0.0) and np.all(l >= 0.0), n
        pr = prices(p, owner[n])
        nu = [pr[p.Ai[0]], pr[p.Ai[1]]]
        _, _, v, _ = response(p, nu)
        pi += v
        V = value_scale(p, nu, d, l, bool(d.any() or l.any()))
        a = 0 if nu[0] * _m(d[0]) >= nu[1] * _m(d[1]) else 1
        # at most one side tendered, up to rounding (a fee-free pool at its price can show both)
        assert _m(d[1 - a]) <= C_ROUND[p.kind] * EPS * V[1 - a], ("both sides tendered", n)
        # the scales of the ordinal checks: every active pool counts (one at its no-trade boundary
        # may trade a rounding's worth in fp64), weighted like the rounding constants
        X = _u3_base(p) if p.kind == "univ3" else [_m(p.R[0]), _m(p.R[1])]
        for sd in (0, 1):
            scale[p.Ai[sd]] = scale.get(p.Ai[sd], mp.mpf(0)) + C_ROUND[p.kind] * (V[sd] + X[sd]) / 64
        allow_r += C_ROUND[p.kind] * EPS * (nu[0] * V[0] + nu[1] * V[1])
        fx = forward(p, a, _m(d[a]))
        tol = C_ROUND[p.kind] * EPS
        assert _m(l[1 - a]) <= fx + tol * V[1 - a], ("pays out more than F(Δ)", n, float(l[1 - a]), float(fx))
        assert _m(l[a]) <= tol * V[a], ("pays out on the tendered side", n)
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
    paid_x, recv_x = _exact_sum(tn), _exact_sum(to)
    assert abs(float(_frac(out["paid"]) - paid_x)) <= _tree_bound(len(tn), nh, tn), "paid is not the sum of the legs"
    assert abs(float(_frac(out["received"]) - recv_x)) <= _tree_bound(len(to), nh, to), "received is not the sum"
    H_x = []
    for k in range(nh):
        hx = _exact_sum(th[k])
        H_x.append(hx)
        assert abs(float(_frac(out["hub_surplus"][k]) - hx)) <= _tree_bound(len(th[k]), 0, th[k]), ("hub surplus", k)
        assert out["hub_surplus"][k] >= 0.0, ("hub short", k)
    if st == FILLED:
        assert out["paid"] <= amount if kind == EXACT_IN else out["received"] >= amount
    # 3. the one-ordinal terms and the ordinal checks (50 digits)
    sn = float(np.nextafter(s, 0.0)) if kind == EXACT_IN else float(np.nextafter(s, np.inf))
    if nested and nh:
        at_s = row.sums_resolved(s, ts)
        at_n = row.sums_resolved(sn, ts)
    else:
        at_s, at_n = row.sums(s, ts), row.sums(sn, ts)
    rnd = lambda tok: C_ORD * EPS * scale.get(tok, mp.mpf(0))
    rj, ri = rnd(row.j), rnd(row.i)
    if kind == EXACT_IN:
        step = ms * max(at_n[0] - at_s[0], 0)
        if nested or not nh:
            assert at_n[0] > amount - rj, ("the ordinal below s* takes at most δ", float(at_n[0]), amount)
    else:
        step = max(at_s[1] - at_n[1], 0)
        if nested or not nh:
            assert at_n[1] < amount + ri, ("the ordinal above s* delivers y", float(at_n[1]), amount)
    hstep = mp.mpf(0)
    H_s = row.sums(s, ts)[2]
    for k, (h, _, _) in enumerate(row.hubs):
        t = ts[k]
        if t <= DBL_MIN:
            continue
        tp = float(np.nextafter(t, 0.0))
        Hp = row.hub_net(k, ms, _m(tp))
        rh = rnd(h)
        assert Hp < rh, ("the ordinal below t_h* leaves hub h short of nothing", k, float(Hp), float(rh))
        hstep += _m(t) * max(H_s[k] - Hp, 0)
    allowance = allow_r + step + hstep
    # 4. the bound
    if kind == EXACT_IN:
        bound = ms * _m(amount) + pi
        gap = bound - _mf(recv_x)
        chk, val = _mf(recv_x), out["received"]
    else:
        bound = (_m(amount) - pi) / ms
        gap = (_mf(paid_x) - bound) * ms
        chk, val = _mf(paid_x), out["paid"]
    res.update(gap=float(gap), allowance=float(allowance), rounding=float(allow_r), bound=float(bound))
    if st == LIMIT:
        lim = float(limit)
        if kind == EXACT_IN:  # the best route receives at most the bound, and at least bound − allowance
            assert lim > float(bound - allowance), ("a limit the optimum meets", lim, float(bound))
        else:
            assert lim < float(bound + allowance / ms), ("a limit the optimum meets", lim, float(bound))
        return res
    assert -allow_r <= gap <= allowance, ("not optimal", float(gap), float(allowance), float(chk), val)
    return res


def _reachable(row, kind, amount):
    if kind == EXACT_OUT:
        assert _m(amount) <= row.reach_out() * (1 + REACH_MARGIN), "filled beyond the depth"
    else:
        cap = row.reach_in()
        if cap != mp.inf:
            assert _m(amount) <= cap * (1 + REACH_MARGIN), "absorbed beyond the depth"


def _unreachable(row, kind, amount):
    if kind == EXACT_OUT:
        reach = row.reach_out()
        assert _m(amount) >= reach * (1 - REACH_MARGIN), ("unreachable below the depth", amount, float(reach))
        return
    cap = row.reach_in()
    if cap != mp.inf:
        assert _m(amount) >= cap * (1 - REACH_MARGIN), ("unreachable below the depth", amount, float(cap))
    elif not row.hubs:
        N = row.sums(DBL_MIN, [])[0]
        assert N <= _m(amount) * (1 + REACH_MARGIN), ("unreachable though N(DBL_MIN) > δ", amount, float(N))
