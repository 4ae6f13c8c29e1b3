"""The route! certificate (solve_certificate.py) and the restatement of cfmm_solve's optimizer
(solver_restatement.py) on the exact dual: no GPU.  The restatement, driven by 50-digit pool
responses, must reach status 0 and certify; so must scipy's L-BFGS-B on the same dual; and the
certificate must reject results that are subtly wrong."""
import numpy as np
import pytest
from scipy.optimize import minimize

import order_certificate as oc
import solve_certificate as sc
import solver_restatement as sr


def market(n, m, seed, kinds=("product",)):
    """m pools over n tokens (every pool on a random pair; all on {1, 2} when n = 2)."""
    rng = np.random.default_rng(seed)
    pools = []
    for k in range(m):
        Ai = (1, 2) if n == 2 else tuple(int(x) for x in rng.choice(np.arange(1, n + 1), 2, replace=False))
        R = 1.0 + 1000.0 * rng.random(2)
        g = float(rng.choice([0.997, 1.0]))
        kind = kinds[k % len(kinds)]
        if kind == "product":
            pools.append(oc.product(R, g, Ai))
        elif kind == "geomean":
            w1 = rng.uniform(0.2, 0.8)
            pools.append(oc.geomean(R, g, (w1, 1.0 - w1), Ai))
        else:
            cp = float(np.exp(rng.uniform(-1, 1)))
            lt = [cp * x for x in (2.0, 4.0 / 3.0, 2.0 / 3.0, 1.0 / 3.0)]
            lq = [float(s) * rng.uniform(1, 100) for s in (1.0, 2.0, 1.5, 0.0)]
            pools.append(oc.univ3(cp, lt, lq, 0.997, Ai))
    c = 0.5 + rng.random(n)
    return pools, c


PGTOL = 1e-3     # above the resolution floor of f at these markets' scale (see DESIGN §7)

CASES = [(2, 6, 1, ("product",)), (31, 120, 2, ("product", "geomean", "univ3")), (200, 500, 3, ("product",))]


@pytest.mark.parametrize("n,m,seed,kinds", CASES)
def test_restatement_on_the_exact_dual_certifies(n, m, seed, kinds):
    pools, c = market(n, m, seed, kinds)
    box = sc.linear_nonnegative(c)
    x, info, trace = sr.solve(sc.oracle_sweep(pools, n), **box.solve_args(), pgtol=PGTOL)
    assert info["status"] == 0, info
    assert info["iterations"] == len(trace) and info["fun_evals"] >= info["iterations"]
    D, L = sc.oracle_trades(pools, x)
    res = sc.certify(pools, box, x, D, L, info=info, pgtol=PGTOL)
    assert res["pg50"] <= PGTOL * (1 + 1e-9) and res["gap"] <= res["bound"] + res["allowance"], res


def test_restatement_basket_certifies():
    n = 31
    pools, _ = market(n, 120, 4, ("product", "geomean"))
    delta_in = np.concatenate([[0.0], 10.0 * np.random.default_rng(5).random(n - 1)])
    box = sc.basket(1, delta_in)
    x, info, _ = sr.solve(sc.oracle_sweep(pools, n), **box.solve_args(), pgtol=PGTOL)
    assert info["status"] == 0, info
    D, L = sc.oracle_trades(pools, x)
    res = sc.certify(pools, box, x, D, L, info=info, pgtol=PGTOL)
    assert res["gap"] <= res["bound"] + res["allowance"]


def scipy_solve(pools, box, pgtol):
    n = len(box.lower)
    sweep = sc.oracle_sweep(pools, n)
    cache = {}

    def ev(x):
        key = x.tobytes()
        if key not in cache:
            cache[key] = sweep(x)
        return cache[key]

    fn = lambda x: float(box.lin @ x) + ev(x)[1]
    jac = lambda x: box.lin + ev(x)[0]
    bounds = [(lo, None) for lo in box.lower]
    res = minimize(fn, np.maximum(np.full(n, 1.0 / n), box.lower), jac=jac, method="L-BFGS-B", bounds=bounds,
                   options=dict(maxcor=5, ftol=0.0, gtol=pgtol, maxiter=2000))
    return res


@pytest.mark.parametrize("n,m,seed,kinds", CASES[1:])
def test_scipy_on_the_exact_dual_certifies(n, m, seed, kinds):
    pools, c = market(n, m, seed, kinds)
    box = sc.linear_nonnegative(c)
    res = scipy_solve(pools, box, PGTOL)
    assert "PGTOL" in str(res.message), res.message
    D, L = sc.oracle_trades(pools, res.x)
    cert = sc.certify(pools, box, res.x, D, L, pgtol=PGTOL, rule="lbfgsb")
    # the restatement's optimum and scipy's agree within the sum of their certified gaps
    x, info, _ = sr.solve(sc.oracle_sweep(pools, n), **box.solve_args(), pgtol=PGTOL)
    mine = sc.certify(pools, box, x, *sc.oracle_trades(pools, x), info=info, pgtol=PGTOL)
    slack = cert["bound"] + cert["allowance"] + mine["bound"] + mine["allowance"]
    assert abs(cert["g50"] - mine["g50"]) <= slack, (cert, mine)


@pytest.fixture(scope="module")
def solved():
    n, m, seed, kinds = CASES[1]
    pools, c = market(n, m, seed, kinds)
    box = sc.linear_nonnegative(c)
    x, info, _ = sr.solve(sc.oracle_sweep(pools, n), **box.solve_args(), pgtol=PGTOL)
    assert info["status"] == 0
    D, L = sc.oracle_trades(pools, x)
    return pools, box, x, info, D, L


def test_certificate_rejects_a_trade_off_by_1e9(solved):
    pools, box, x, info, D, L = solved
    k = int(np.argmax(np.max(L, axis=1)))
    s = int(np.argmax(L[k]))
    L2 = L.copy()
    L2[k, s] *= 1.0 + 1e-9
    with pytest.raises(AssertionError, match="optimal response"):
        sc.certify(pools, box, x, D, L2, info=info, pgtol=PGTOL)


def test_certificate_rejects_a_moved_coordinate(solved):
    pools, box, x, info, D, L = solved
    # move the free coordinate whose gradient is steepest: |pg| > pgtol there afterwards
    free = np.flatnonzero(x > box.lower)
    j = int(free[0])
    x2 = x.copy()
    for f in (1e-4, 1e-3, 1e-2, 1e-1):
        x2[j] = x[j] * (1.0 + f)
        psi, _ = sc.oracle_sweep(pools, len(x))(x2)
        if abs(psi[j]) > 2 * PGTOL:
            break
    assert abs(psi[j]) > 2 * PGTOL
    D2, L2 = sc.oracle_trades(pools, x2)
    with pytest.raises(AssertionError, match="pgtol"):
        sc.certify(pools, box, x2, D2, L2, pgtol=PGTOL)


def test_certificate_rejects_an_early_status0():
    n, m, seed, kinds = CASES[1]
    pools, c = market(n, m, seed, kinds)
    box = sc.linear_nonnegative(c)
    x, info, _ = sr.solve(sc.oracle_sweep(pools, n), **box.solve_args(), pgtol=10 * PGTOL)
    assert info["status"] == 0
    D, L = sc.oracle_trades(pools, x)
    res = sc.certify(pools, box, x, D, L, info=info, pgtol=10 * PGTOL)
    assert res["pg50"] > 2 * PGTOL, res       # a stop at ≈ 10·pgtol
    with pytest.raises(AssertionError, match="pgtol"):
        sc.certify(pools, box, x, D, L, info=info, pgtol=PGTOL)
