"""A 50-digit certificate for a route! result (cfmm_solve, route(..., optimizer="device"), and the host
path), for the tests.  It works from each pool's optimal response in mpmath (order_certificate.response)
and shares nothing with the kernels or the optimizer.

route! minimises the dual g(ν) = linᵀν + Σ_k π_k(ν) over the box ℓ ≤ ν ≤ u (π_k the value of pool k's
optimal trade at ν).  The objectives map to a box and a reference lower bound ℓ̂ ≤ ℓ, the one of the
primal problem the box stands for:
  LinearNonnegative(c)     lin = 0, ℓ = c + 1e-8, ℓ̂ = c              (primal: max cᵀΨ, Ψ ≥ 0)
  BasketLiquidation(i, Δ)  lin = Δ (0 at i), ℓ = √eps (1 + √eps at i), ℓ̂ = 0 (1 at i)
                                                                  (primal: max Ψ_i, Ψ_j + Δ_j ≥ 0)
  a raw (lin, ℓ, u) box    ℓ̂ = ℓ                                   (primal: max_Ψ min_box (lin + Ψ)ᵀν)

With z = lin + Ψ at the result's trades Ψ = Σ_k A_k(Λ_k − Δ_k), the duality gap is
    gap = Σ_j gap_j,   gap_j = z_j·(ν_j − ℓ̂_j)   if z_j ≥ 0 or u_j = ∞,   |z_j|·(u_j − ν_j) otherwise
(LinearNonnegative: (ν − c)ᵀΨ; Basket: Σ_{j≠i} ν_j(Ψ_j + Δ_j) + (ν_i − 1)Ψ_i), and the primal
infeasibility of token j (u_j = ∞) is max(0, −z_j).

The stop.  The device stops at status 0 when ‖pg‖∞ ≤ pgtol, pg the gradient ∇g = lin + Ψ with the
clipping rule of solver_commit_kernel: pg_j = 0 when ν_j ≤ ℓ_j and ∇g_j > 0, or ν_j ≥ u_j and
∇g_j < 0 (rule "clip").  scipy's L-BFGS-B tests |P(ν − ∇g) − ν|∞ instead (rule "lbfgsb"), under which a
coordinate within pgtol of its bound counts as on it.  With ‖pg‖∞ ≤ pgtol:
  free coordinates:       |∇g_j| ≤ pgtol, so gap_j ≤ pgtol·max(ν_j − ℓ̂_j, u_j − ν_j);
  on the lower bound:     ∇g_j ≥ 0 (or |∇g_j| ≤ pgtol), so gap_j ≤ ∇g_j⁺·(ν_j − ℓ̂_j) + pgtol·(u_j − ν_j);
  on a finite upper one:  ∇g_j ≤ 0 (or |∇g_j| ≤ pgtol), so gap_j ≤ ∇g_j⁻·(u_j − ν_j) + pgtol·(ν_j − ℓ̂_j)
(terms with u_j = ∞ drop), and −∇g_j ≤ pgtol wherever u_j = ∞.  certify asserts
    gap ≤ bound + allowance,   bound = Σ_j of the terms above at the 50-digit ∇g,
    infeasibility_j ≤ pgtol + 2·E_j,
so a result certifies itself: the bound follows from the stop, not from another solver.  ℓ − ℓ̂ is
1e-8 (LinearNonnegative) or √eps (Basket): the lower-bound terms are the price of the objective's
box, not of the optimizer.

Checks, with ε = 2⁻⁵² and the per-pool rounding model of order_certificate (r_k,s = C_ROUND·ε·V_k,s,
V the value scale of pool k in token units of side s):
  1. trades are optimal responses: |Δ_k,s − Δ*_k,s| and |Λ_k,s − Λ*_k,s| ≤ r_k,s for every active pool
     (the materialising sweep, reference operation order), and retired pools trade exactly zero;
  2. the stop was honest (status 0): the 50-digit |pg*_j| ≤ pgtol + E_j for every token, with E_j the
     error bound of the gradient-only sweep at ν:
         E_j = Σ_{k∋j} r_k,j + deg_j·ε·Σ_{k∋j} |Λ*_k,j − Δ*_k,j| + deg_j·2⁻⁵³·S_j,
     the per-pool bound of the economized and reference forms (C_ROUND is at least the per-pool
     constants the readout tests measure: 4 ProductTwoCoin economized, 24 + 2·|e·log2 t| GeometricMean),
     any order of the deg_j fp64 additions into Ψ_j, and one quantum 2^(e−54) ≤ 2⁻⁵³·S_j per pool of
     the fixed-point Ψ[b] slice (S_j the token's total ProductTwoCoin reserve).  info.f agrees with
     the 50-digit g(ν) within Σ_j ν_j·E_j + (m + n)·ε·(Σ_k Σ_s ν_s(Δ*_k,s + Λ*_k,s) + Σ_j |lin_j ν_j|);
  3. the gap bound above, with allowance = Σ_k Σ_s W_s·r_k,s, W_j = max(ν_j, |ν_j − ℓ̂_j|, u_j − ν_j)
     (finite terms): the rounding of the trades the gap is computed from.
"""
from __future__ import annotations

import mpmath as mp
import numpy as np

from order_certificate import C_ROUND, DPS, EPS, response, value_scale

SQRT_EPS = float(np.sqrt(np.finfo(np.float64).eps))


class Box:
    """lin, ℓ (lower), u (upper, +inf where unbounded) and the primal's ℓ̂ (ref) of one objective."""

    def __init__(self, lin, lower, upper=None, ref=None):
        self.lower = np.asarray(lower, dtype=np.float64)
        n = len(self.lower)
        self.lin = np.zeros(n) if lin is None else np.asarray(lin, dtype=np.float64)
        self.upper = np.full(n, np.inf) if upper is None else np.asarray(upper, dtype=np.float64)
        self.ref = self.lower.copy() if ref is None else np.asarray(ref, dtype=np.float64)

    def solve_args(self):
        """The keyword arguments of DevicePools.solve for this box."""
        fin = np.isfinite(self.upper)
        return dict(lower=self.lower, lin=self.lin, upper=self.upper if fin.any() else None)


def linear_nonnegative(c):
    c = np.asarray(c, dtype=np.float64)
    return Box(np.zeros(len(c)), c + 1e-8, ref=c)


def basket(i, delta_in):
    """BasketLiquidation(i, Δin), i 1-based."""
    lin = np.array(delta_in, dtype=np.float64)
    lin[i - 1] = 0.0
    lower = np.full(len(lin), SQRT_EPS)
    lower[i - 1] = 1.0 + SQRT_EPS
    ref = np.zeros(len(lin))
    ref[i - 1] = 1.0
    return Box(lin, lower, ref=ref)


def _pair(p, nu):
    return [mp.mpf(float(nu[p.Ai[0] - 1])), mp.mpf(float(nu[p.Ai[1] - 1]))]


def oracle_sweep(pools, n):
    """sweep(ν) -> (Ψ, acc) of the active pools from their 50-digit responses, rounded to fp64: the
    callback that drives solver_restatement.solve on the exact dual."""
    def sweep(nu):
        with mp.workdps(DPS):
            psi = [mp.mpf(0)] * n
            acc = mp.mpf(0)
            for p in pools:
                if not p.active:
                    continue
                D, L, v, _ = response(p, _pair(p, nu))
                for s in (0, 1):
                    psi[p.Ai[s] - 1] += L[s] - D[s]
                acc += v
            return np.array([float(x) for x in psi]), float(acc)
    return sweep


def oracle_trades(pools, nu):
    """(Δ, Λ) [m, 2] of every pool at ν from the 50-digit responses, rounded to fp64 (retired: 0)."""
    D, L = np.zeros((len(pools), 2)), np.zeros((len(pools), 2))
    with mp.workdps(DPS):
        for k, p in enumerate(pools):
            if p.active:
                d, l, _, _ = response(p, _pair(p, nu))
                D[k], L[k] = [float(x) for x in d], [float(x) for x in l]
    return D, L


def pg_vector(box, nu, z, rule="clip"):
    """The projected gradient at ν for the gradient z (mp or float), rule "clip" or "lbfgsb"."""
    out = []
    for j in range(len(nu)):
        zj, x, lo, up = z[j], float(nu[j]), box.lower[j], box.upper[j]
        if rule == "clip":
            p = zj
            if x <= lo and zj > 0:
                p = 0 * zj
            if x >= up and zj < 0:
                p = 0 * zj
        else:
            t = mp.mpf(x) - zj
            t = max(t, mp.mpf(lo))
            if np.isfinite(up):
                t = min(t, mp.mpf(up))
            p = mp.mpf(x) - t
        out.append(p)
    return out


def certify(pools, box, nu, D, L, info=None, pgtol=1e-5, rule="clip", check_stop=True):
    """Certify a route! result.  pools: order_certificate.Pools in global insertion order (inactive
    ones included); nu: the result's ν; D, L: its trades [m, 2]; info: cfmm_solve's info dict (f is
    checked when given); check_stop: the optimizer claims ‖pg‖∞ ≤ pgtol (status 0).  Returns a dict
    (gap, bound, allowance, pg50, ...) and asserts the checks of the module docstring."""
    with mp.workdps(DPS):
        return _certify(pools, box, np.asarray(nu, dtype=np.float64), np.asarray(D, float).reshape(-1, 2),
                        np.asarray(L, float).reshape(-1, 2), info, float(pgtol), rule, check_stop)


def _certify(pools, box, nu, D, L, info, pgtol, rule, check_stop):
    n = len(nu)
    assert len(D) == len(pools) and len(L) == len(pools), "one (Δ, Λ) per pool"
    assert np.all(nu >= box.lower) and np.all(nu <= box.upper), "ν outside the box"
    psi_star, psi_dev = [mp.mpf(0)] * n, [mp.mpf(0)] * n
    E = [mp.mpf(0)] * n                   # sweep error bound per token
    absflow, deg, S = [mp.mpf(0)] * n, [0] * n, [mp.mpf(0)] * n
    r_side = []                           # (token, r) per pool side, for the gap allowance
    pi, absval = mp.mpf(0), mp.mpf(0)
    for k, p in enumerate(pools):
        d, l = D[k], L[k]
        if not p.active:
            assert not d.any() and not l.any(), ("a retired pool traded", k)
            continue
        assert np.all(np.isfinite(d)) and np.all(np.isfinite(l)) and np.all(d >= 0) and np.all(l >= 0), k
        nup = _pair(p, nu)
        Ds, Ls, v, _ = response(p, nup)
        pi += v
        V = value_scale(p, nup, d, l, bool(d.any() or l.any()))
        for s in (0, 1):
            j = p.Ai[s] - 1
            r = C_ROUND[p.kind] * EPS * V[s]
            # 1. the materialised trades are the optimal response, up to rounding
            assert abs(mp.mpf(float(d[s])) - Ds[s]) <= r, ("Δ is not the optimal response", k, s, float(d[s]), float(Ds[s]))
            assert abs(mp.mpf(float(l[s])) - Ls[s]) <= r, ("Λ is not the optimal response", k, s, float(l[s]), float(Ls[s]))
            psi_star[j] += Ls[s] - Ds[s]
            psi_dev[j] += mp.mpf(float(l[s])) - mp.mpf(float(d[s]))
            E[j] += r
            absflow[j] += abs(Ls[s] - Ds[s])
            deg[j] += 1
            if p.kind == "product":
                S[j] += mp.mpf(p.R[s])
            absval += nup[s] * (Ds[s] + Ls[s])
            r_side.append((j, r))
    for j in range(n):
        E[j] += deg[j] * EPS * absflow[j] + deg[j] * mp.mpf(2) ** -53 * S[j]
    lin = [mp.mpf(float(x)) for x in box.lin]
    z_star = [lin[j] + psi_star[j] for j in range(n)]
    z_dev = [lin[j] + psi_dev[j] for j in range(n)]
    g50 = sum((lin[j] * mp.mpf(float(nu[j])) for j in range(n)), mp.mpf(0)) + pi
    pg = pg_vector(box, nu, z_star, rule)
    pg50 = max((abs(x) for x in pg), default=mp.mpf(0))
    res = dict(g50=float(g50), pg50=float(pg50), n=n, m=len(pools))
    # 2. the stop
    if check_stop:
        for j in range(n):
            assert abs(pg[j]) <= pgtol + E[j], ("|pg| above pgtol at a claimed stop", j, float(pg[j]), pgtol, float(E[j]))
    if info is not None:
        allow_f = sum((mp.mpf(float(nu[j])) * E[j] for j in range(n)), mp.mpf(0)) + \
            (len(pools) + n) * EPS * (absval + sum((abs(lin[j] * mp.mpf(float(nu[j]))) for j in range(n)), mp.mpf(0)))
        assert abs(mp.mpf(float(info["f"])) - g50) <= allow_f, ("info.f is not g(ν)", float(info["f"]), float(g50), float(allow_f))
        res["f_err"] = float(abs(mp.mpf(float(info["f"])) - g50))
    # 3. the gap and its bound
    delta = 0.0 if rule == "clip" else pgtol
    gap, bound, infeas = mp.mpf(0), mp.mpf(0), mp.mpf(0)
    W = []
    for j in range(n):
        x, lo, up, ref = (mp.mpf(float(a)) for a in (nu[j], box.lower[j], box.upper[j] if np.isfinite(box.upper[j]) else 0.0, box.ref[j]))
        fin = bool(np.isfinite(box.upper[j]))
        zd, zs = z_dev[j], z_star[j]
        gap += zd * (x - ref) if (zd >= 0 or not fin) else -zd * (up - x)
        up_room = (up - x) if fin else mp.mpf(0)
        if nu[j] - box.lower[j] <= delta:
            bound += max(zs, 0) * (x - ref) + pgtol * up_room
        elif fin and box.upper[j] - nu[j] <= delta:
            bound += max(-zs, 0) * up_room + pgtol * (x - ref)
        else:
            bound += pgtol * max(x - ref, up_room)
        if not fin:
            inf_j = max(-zd, 0)
            infeas = max(infeas, inf_j)
            if check_stop:
                assert inf_j <= pgtol + 2 * E[j], ("primal infeasible beyond pgtol", j, float(inf_j))
        W.append(max(x, abs(x - ref), up_room))
    allowance = sum((W[j] * r for j, r in r_side), mp.mpf(0))
    res.update(gap=float(gap), bound=float(bound), allowance=float(allowance), infeasibility=float(infeas),
               sweep_err=float(max(E, default=0)))
    if check_stop:
        assert gap <= bound + allowance, ("the gap exceeds what the stop implies", float(gap), float(bound), float(allowance))
    return res
