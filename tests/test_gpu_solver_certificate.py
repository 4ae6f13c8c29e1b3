"""cfmm_solve (route(..., optimizer="device")) against a restatement of its optimizer and a 50-digit
certificate of its result.

(a) The iterates x_1 … x_12 of the device (one solve per maxiter = k) match solver_restatement.solve
    driven by the device's own sweeps, coordinate by coordinate, up to the first iteration where a
    decision margin falls below 1e-7 (fp64 atomics make Ψ non-deterministic in its last bits, so two
    runs may only part ways at a decision that close).  Token counts from 2 up to 300 000: above
    131 072 tokens the vector kernels' grid-stride loops run more than once, and the multi-block
    reduction sums partials of up to 512 blocks.
(b) Every configuration the solver runs on stops at status 0 and passes solve_certificate.certify:
    ProductTwoCoin on the first-generation kernel and on the TMA kernel (compact records, fixed-point
    Ψ[b] slice) under each sweep option, GeometricMean, UniV3 with ragged ladders, a mixed set, a set
    with appended and retired pools, LinearNonnegative, BasketLiquidation and a raw box with finite
    upper bounds, fixed coordinates and a supplied v0.  The host path (scipy L-BFGS-B over the same
    sweeps) certifies too, and the two dual values agree within the sum of their certified gaps.
(c) maxiter and maxfun are honoured, and the trades are materialised at the returned ν.

pgtol per case: the line search and the factr test compare values of f, whose fp64 resolution is
about 8·eps·|f|; below ‖pg‖ ≈ √(2·λ·8·eps·|f|) (λ the dual's curvature) no step can show a decrease
and the solve stops at status 1.  That floor is the same with exact = 1, the reference-order math and
the fp64 Ψ[b] slice (DESIGN §7), so each case runs at a pgtol above it.
"""
import time

import numpy as np
import pytest

import order_certificate as oc
import solve_certificate as sc
import solver_restatement as sr

pytestmark = pytest.mark.gpu

MARGIN = 1e-7
PGTOL = 1e-3           # LinearNonnegative markets of 60 tokens below (floor: 3e-4 … 7e-4 measured)
PGTOL_PRODUCT = 1e-2   # the 8000-pool ProductTwoCoin market (|f| ≈ 1e6: status 1 at pgtol 1e-3 with every option)
PGTOL_BASKET = 5e-3    # BasketLiquidation markets below (floor: 4e-4 … 1.3e-3 measured)


# ---- pool sets: the device context and the certificate's pools, in global insertion order ----------
def product_pools(R, g, A, active=None):
    act = np.ones(len(g), bool) if active is None else active
    return [oc.product(R[k], g[k], A[k], active=bool(act[k])) for k in range(len(g))]


def geomean_pools(R, g, A, w):
    return [oc.geomean(R[k], g[k], w[k], A[k]) for k in range(len(g))]


def univ3_pools(cp, g, A, off, lt, lq):
    return [oc.univ3(cp[k], lt[off[k]:off[k + 1]], lq[off[k]:off[k + 1]], g[k], A[k]) for k in range(len(g))]


def make(cr, n, product=None, geomean=None, univ3=None, opts=None):
    p = cr.DevicePools(n)
    for k, v in (opts or {}).items():
        p.set_option(k, v)
    pools = []
    if product is not None:
        p.add_product(*product)
        pools += product_pools(*product)
    if geomean is not None:
        p.add_geomean(*geomean)
        pools += geomean_pools(*geomean)
    if univ3 is not None:
        p.add_univ3(*univ3)
        pools += univ3_pools(*univ3)
    p.finalize()
    return p, pools


def solve_and_certify(p, pools, box, pgtol, v0=None):
    x, info = p.solve(**box.solve_args(), v0=v0, pgtol=pgtol)
    assert info["status"] == 0 and info["pg_norm"] <= pgtol, (info, pgtol)
    D, L = p.trades()
    res = sc.certify(pools, box, x, D, L, info=info, pgtol=pgtol)
    res.update(status=info["status"], iterations=info["iterations"])
    print(f"  status {info['status']}, {info['iterations']} iterations, |pg|50 {res['pg50']:.3g}, "
          f"gap {res['gap']:.3g} <= bound {res['bound']:.3g} + {res['allowance']:.3g}")
    return x, res


def host_path(p, box, pgtol):
    """route()'s host path: scipy L-BFGS-B over one device sweep per evaluation (ftol = 0: it stops
    on pgtol)."""
    from scipy.optimize import minimize
    n = len(box.lower)
    cache = {}

    def ev(x):
        k = x.tobytes()
        if k not in cache:
            cache.clear()
            cache[k] = p.sweep(x)
        return cache[k]

    res = minimize(lambda x: float(box.lin @ x) + ev(x)[1], np.maximum(np.full(n, 1.0 / n), box.lower),
                   jac=lambda x: box.lin + ev(x)[0], method="L-BFGS-B",
                   bounds=[(lo, None) for lo in box.lower],
                   options=dict(maxcor=5, ftol=0.0, gtol=pgtol, maxiter=15_000, maxfun=15_000))
    assert "PGTOL" in str(res.message), res.message
    return res.x


def certify_host_and_compare(p, pools, box, pgtol, dev):
    xh = host_path(p, box, pgtol)
    p.sweep(xh, materialize=True)
    D, L = p.trades()
    host = sc.certify(pools, box, xh, D, L, pgtol=pgtol, rule="lbfgsb")
    slack = dev["bound"] + dev["allowance"] + host["bound"] + host["allowance"]
    assert abs(dev["g50"] - host["g50"]) <= slack, (dev, host)


# ---- (a) iterate by iterate -------------------------------------------------------------------------
def _two_token(seed, m):
    rng = np.random.default_rng(seed)
    R = 1000 * rng.random((m, 2)) + 1
    g = rng.choice([0.997, 1.0], m)
    return R, g, np.tile([1, 2], (m, 1))


# (n, m, seed, iterations, compared at least, branches the compared iterations must include)
AGREE = [
    (2, 6, 3, 12, 5, ("backtrack",)),
    (31, 300, 2, 12, 6, ("activated", "wrap")),
    (257, 4000, 1, 12, 7, ("wrap",)),
    (50_000, 200_000, 1, 3, 3, ("activated",)),
    (131_073, 400_000, 1, 3, 3, ("activated",)),
    (300_000, 900_000, 1, 3, 3, ("activated",)),
]


@pytest.mark.parametrize("n,m,seed,kmax,need,branches", AGREE, ids=[str(a[0]) for a in AGREE])
def test_iterates_match_the_restatement(cr, synth, n, m, seed, kmax, need, branches):
    R, g, A = _two_token(seed, m) if n == 2 else synth.product_pools(m, n, seed=seed)
    p = cr.DevicePools(n)
    p.add_product(R, g, A)
    p.finalize()
    lower = np.random.default_rng(seed + 1).random(n) + 0.5 + 1e-8
    _, info, trace = sr.solve(lambda v: p.sweep(v), lower, lin=np.zeros(n), maxiter=kmax)
    assert info["iterations"] == kmax, info
    compared, seen = 0, set()
    for k, rec in enumerate(trace, start=1):
        if rec["min_margin"] < MARGIN:
            break
        x, dinfo = p.solve(lower, lin=np.zeros(n), maxiter=k)
        assert dinfo["status"] == 2 and dinfo["iterations"] == k, dinfo
        err = np.max(np.abs(x - rec["x"]))
        assert err <= 1e-9 * np.max(np.abs(rec["x"])), (k, err)
        compared += 1
        seen |= {b for b, hit in (("backtrack", rec["backtracks"]), ("wrap", rec["wrap"]),
                                  ("activated", rec["activated"]), ("restart", rec["restart"])) if hit}
    assert compared >= need, compared
    assert set(branches) <= seen, seen
    p.close()


# ---- (b) the certificate at convergence --------------------------------------------------------------
@pytest.mark.parametrize("opts", [{"use_tma": 0}, {}, {"exact": 1}, {"gradient_math": 0}, {"psi_fixed_point": 0}],
                         ids=["first_generation", "tma_default", "exact", "reference_math", "fp64_slice"])
def test_product_two_coin_certifies(cr, synth, opts):
    n = 300
    R, g, A = synth.product_pools(8000, n, seed=3)
    p, pools = make(cr, n, product=(R, g, A), opts=opts)
    info = p.pool_set_info(0)
    assert info["tma"] == 1 and info["compact_stream"] == 1 and info["fixed_point"] == 1, info
    box = sc.linear_nonnegative(np.random.default_rng(0).random(n) + 0.5)
    t = time.time()
    _, dev = solve_and_certify(p, pools, box, PGTOL_PRODUCT)
    if opts == {}:
        certify_host_and_compare(p, pools, box, PGTOL_PRODUCT, dev)
    print(f"  {opts}: {time.time() - t:.1f} s")
    p.close()


def _mixed(synth, n):
    return dict(product=synth.product_pools(1000, n, seed=7), geomean=synth.geomean_pools(600, n, seed=8),
                univ3=synth.univ3_pools(600, n, seed=9, ragged=True))


@pytest.mark.parametrize("kind", ["geomean", "univ3", "mixed"])
def test_other_pool_types_certify(cr, synth, kind):
    n = 60
    sets = {"geomean": dict(geomean=synth.geomean_pools(1500, n, seed=5)),
            "univ3": dict(univ3=synth.univ3_pools(1500, n, seed=6, ragged=True)),
            "mixed": _mixed(synth, n)}[kind]
    p, pools = make(cr, n, **sets)
    box = sc.linear_nonnegative(np.random.default_rng(1).random(n) + 0.5)
    _, dev = solve_and_certify(p, pools, box, PGTOL)
    if kind == "mixed":
        certify_host_and_compare(p, pools, box, PGTOL, dev)
    p.close()


@pytest.mark.parametrize("kind", ["basket", "swap"])
def test_basket_liquidation_certifies(cr, synth, kind):
    n = 60
    p, pools = make(cr, n, **_mixed(synth, n))
    if kind == "basket":
        delta_in = np.concatenate([[0.0], 10 * np.random.default_rng(2).random(n - 1)])
        i = 1
    else:
        delta_in, i = np.zeros(n), 5
        delta_in[11] = 50.0                      # Swap(5, 12, 50, n)
    box = sc.basket(i, delta_in)
    solve_and_certify(p, pools, box, PGTOL_BASKET)
    p.close()


def test_appended_and_retired_pools_certify(cr, synth):
    n = 60
    R, g, A = synth.product_pools(1200, n, seed=11)
    Rt, gt, At = synth.product_pools(300, n, seed=12)
    Rg, gg, Ag, wg = synth.geomean_pools(300, n, seed=13)
    p = cr.DevicePools(n)
    p.add_product(R, g, A)
    p.finalize()
    p.append_product(Rt, gt, At)
    p.append_geomean(Rg, gg, Ag, wg)
    rng = np.random.default_rng(14)
    act_p = rng.random(1500) > 0.2        # main and appended ProductTwoCoin pools
    act_g = rng.random(300) > 0.2
    p.set_active(0, 0, act_p)
    p.set_active(1, 0, act_g)
    assert p.pool_set_info(0)["tail"] == 300 and p.pool_set_info(0)["retired"] == int((~act_p).sum())
    Rp, gp, Ap = np.concatenate([R, Rt]), np.concatenate([g, gt]), np.concatenate([A, At])
    pools = product_pools(Rp, gp, Ap, act_p) + [oc.geomean(Rg[k], gg[k], wg[k], Ag[k], active=bool(act_g[k]))
                                                for k in range(300)]
    box = sc.linear_nonnegative(np.random.default_rng(15).random(n) + 0.5)
    _, a = solve_and_certify(p, pools, box, PGTOL)
    p.close()
    # a fresh context of just the active pools reaches the same optimum, within the certified gaps
    q, qpools = make(cr, n, product=(Rp[act_p], gp[act_p], Ap[act_p]),
                     geomean=(Rg[act_g], gg[act_g], Ag[act_g], wg[act_g]))
    _, b = solve_and_certify(q, qpools, box, PGTOL)
    assert abs(a["g50"] - b["g50"]) <= a["bound"] + a["allowance"] + b["bound"] + b["allowance"], (a, b)
    q.close()


def test_raw_box_upper_bounds_fixed_coordinates_and_v0(cr, synth):
    n = 60
    p, pools = make(cr, n, **_mixed(synth, n))
    rng = np.random.default_rng(3)
    c = rng.random(n) + 0.5
    lower, upper = c.copy(), np.full(n, np.inf)
    upper[:10] = c[:10] * 1.02               # finite upper bounds
    upper[10:14] = lower[10:14]              # fixed coordinates
    box = sc.Box(0.2 * rng.random(n), lower, upper)
    v0 = c * (1.0 + 0.05 * rng.random(n))
    x, res = solve_and_certify(p, pools, box, PGTOL, v0=v0)
    assert np.array_equal(x[10:14], lower[10:14])
    assert np.all(x <= upper) and np.any(x[:10] == upper[:10]), "no upper bound is active: the case tests nothing"
    p.close()


# ---- (c) options ----------------------------------------------------------------------------------------
def test_solve_options_and_materialised_trades(cr, synth):
    n = 300
    R, g, A = synth.product_pools(8000, n, seed=3)
    p, _ = make(cr, n, product=(R, g, A))
    lower = np.random.default_rng(0).random(n) + 0.5 + 1e-8
    x, info = p.solve(lower, maxfun=3)
    assert info["status"] == 3 and info["fun_evals"] == 3, info
    x, info = p.solve(lower, maxiter=4)
    assert info["status"] == 2 and info["iterations"] == 4, info
    D, L = p.trades()
    p.sweep(x, materialize=True)
    D2, L2 = p.trades()
    assert np.array_equal(D, D2) and np.array_equal(L, L2)
    p.close()
