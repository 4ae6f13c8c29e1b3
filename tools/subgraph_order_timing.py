"""Times cfmm_quote_subgraph_orders on one GPU; prints one JSON line per measurement.

  hub       routed_order_timing.py's hub set: 2k tokens, hubs 1..7 each paired with every other token
            by three pools (ProductTwoCoin, GeometricMeanTwoCoin, UniV3), 20k sparse direct pools.
  headline  10M ProductTwoCoin pools, 50k tokens (bench.py's headline set).
B is tokens 1..|B| (the hubs first on the hub set), |B| in {8, 64, 256}.  Rows sell one token outside
B for another at 1e-3 of a pool's depth (exact-in), default options.  Per quote call: the wall time
of the synchronous call (host clock), the kernel time (CUDA events, option "profile", slot 4: the
B-subgraph, plan and solve kernels), the filled / unreachable / not-converged rows, the mean and
largest iterations and evaluations of the solved rows, the largest m_r of the filled rows and the
smallest of the not-converged ones (the floor the default rtol meets or misses), and the mean pools
per row.  The same rows are then quoted as auto-routed orders (cfmm_choose_order_hubs with the mask,
then cfmm_quote_routed_orders) and as best paths (cfmm_find_order_paths, H = 4): the fraction of rows
where the subgraph's received is at least theirs (within 3·rtol) and the median ratio.  Each
configuration runs on 1k rows first; the 100k-row call runs when the 1k-row kernel time predicts at
most --budget-s seconds for it, and is reported as not run (with the estimate) otherwise.

--kind out quotes exact-out rows (cfmm_quote_subgraph_swap_orders): the same rows are first quoted
exact-in (untimed), and each row that filled asks for what it received; --kind mixed alternates
exact-in rows (even) and such exact-out rows (odd) in one call.  The records then also report, for
the exact-out rows, paid against the exact-in tender δ (the median paid/δ and the fraction within
(|T| + 1)·rtol·δ + (|T| + 2)·rtol·y·ν_i, the round-trip bound of the tests) and against auto-routed
and best-path exact-out (the fraction where the subgraph pays at most theirs within 3·rtol, and the
median ratio).  --B restricts the mask sizes.

    python tools/subgraph_order_timing.py [--only hub|headline] [--budget-s 20] [--kind in|out|mixed]
                                          [--B 8,64]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402
from routed_order_timing import hub_set, timed  # noqa: E402
from split_order_timing import card  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def stats(o):
    solved = o.solver_status >= 0
    filled = o.status == 0
    nc = o.status == cr._lib.ORDER_NOT_CONVERGED
    pools = np.diff(o.leg_off)
    return dict(filled=int(np.sum(filled)), unreachable=int(np.sum(o.status == 2)), not_converged=int(np.sum(nc)),
                iter_mean=round(float(np.mean(o.iterations[solved])), 1) if np.any(solved) else 0.0,
                iter_max=int(np.max(o.iterations[solved])) if np.any(solved) else 0,
                fev_mean=round(float(np.mean(o.fun_evals[solved])), 1) if np.any(solved) else 0.0,
                fev_max=int(np.max(o.fun_evals[solved])) if np.any(solved) else 0,
                merit_filled_max=float(np.max(o.merit[filled & solved])) if np.any(filled & solved) else 0.0,
                merit_nc_min=float(np.min(o.merit[nc])) if np.any(nc) else None,
                pools_mean=round(float(np.mean(pools)), 1))


def compare(p, tin, tout, amt, allowed, o):
    q = len(tin)
    kind = np.zeros(q, np.uint8)
    off, flat, _, _ = p.choose_order_hubs(tin, tout, kind, amt, 7, allowed)
    _, recv_r, _, st_r = p.quote_routed_orders(tin, tout, kind, amt, off, flat)[:4]
    value, st_p = p.find_order_paths(tin, tout, kind, amt, 4, allowed)[6:]
    out = {}
    for name, recv, st in (("auto_routed", recv_r, st_r), ("best_path", value, st_p)):
        both = (o.status == 0) & (st == 0) & (recv > 0)
        if np.any(both):
            ratio = o.received[both] / recv[both]
            out[name] = dict(rows=int(np.sum(both)), at_least=float(np.mean(ratio >= 1 - 3e-4)),
                             median_ratio=round(float(np.median(ratio)), 6))
    return out


def compare_out(p, tin, tout, y, delta, allowed, o, rtol=1e-4):
    """Paid by the exact-out rows o against the exact-in tender and auto-routed / best-path exact-out."""
    q = len(tin)
    kind = np.ones(q, np.uint8)
    filled = o.status == 0
    out = {}
    if np.any(filled):
        nt = np.diff(o.tok_off)
        nu_i = o.nu[o.tok_off[:-1]]
        bound = (nt + 1) * rtol * delta + (nt + 2) * rtol * y * nu_i
        out["vs_exact_in"] = dict(rows=int(np.sum(filled)),
                                  median_ratio=round(float(np.median(o.paid[filled] / delta[filled])), 6),
                                  within_bound=float(np.mean(np.abs(o.paid - delta)[filled] <= bound[filled])))
    off, flat, _, _ = p.choose_order_hubs(tin, tout, kind, y, 7, allowed)
    paid_r, _, _, st_r = p.quote_routed_orders(tin, tout, kind, y, off, flat)[:4]
    value, st_p = p.find_order_paths(tin, tout, kind, y, 4, allowed)[6:]
    for name, paid, st in (("auto_routed", paid_r, st_r), ("best_path", value, st_p)):
        both = filled & (st == 0) & (paid > 0)
        if np.any(both):
            ratio = o.paid[both] / paid[both]
            out[name] = dict(rows=int(np.sum(both)), at_most=float(np.mean(ratio <= 1 + 3 * rtol)),
                             median_ratio=round(float(np.median(ratio)), 6))
    return out


def run(p, name, n, pick, amt_of, budget_s, kind="in", sizes=(8, 64, 256)):
    tin, tout = pick(1, 8)  # the first call builds the pair index and the token adjacency
    p.quote_subgraph_orders(tin, tout, amt_of(tin, tout), np.arange(n) < 8)
    if kind != "in":
        return run_out(p, name, n, pick, amt_of, budget_s, kind, sizes)
    for nb in sizes:
        allowed = np.arange(n) < nb
        est = None
        for q in (1_000, 100_000):
            if q > 1_000 and est > budget_s * 1e3:
                emit(set=name, B=nb, rows=q, run=False, estimated_kernel_ms=round(est, 1))
                continue
            tin, tout = pick(q, nb)
            amt = amt_of(tin, tout)
            o, wall, ms, launches = timed(p, lambda: p._subgraph(False, tin, tout, amt, allowed, None, None))
            rec = dict(set=name, B=nb, rows=q, wall_ms=round(wall, 3), kernel_ms=round(ms, 3),
                       profile_entries=launches, **stats(o))
            if q == 1_000:
                rec.update(compare(p, tin, tout, amt, allowed, o))
            emit(**rec)
            est = ms * 100_000 / q


def run_out(p, name, n, pick, amt_of, budget_s, kind, sizes):
    for nb in sizes:
        allowed = np.arange(n) < nb
        est = None
        for q in (1_000, 100_000):
            if q > 1_000 and est > budget_s * 1e3:
                emit(set=name, B=nb, rows=q, kind=kind, run=False, estimated_kernel_ms=round(est, 1))
                continue
            tin, tout = pick(q, nb)
            delta = amt_of(tin, tout)
            qi = p.quote_subgraph_orders(tin, tout, delta, allowed)
            keep = qi.status == 0  # exact-out rows ask for what the exact-in row received
            k = np.zeros(q, np.uint8) if kind == "mixed" else np.ones(q, np.uint8)
            if kind == "mixed":
                k[1::2] = 1
                keep |= k == 0
            tin, tout, delta, k = tin[keep], tout[keep], delta[keep], k[keep]
            amt = np.where(k == 1, qi.received[keep], delta)
            o, wall, ms, launches = timed(p, lambda: p._subgraph(False, tin, tout, amt, allowed, None, None, k))
            rec = dict(set=name, B=nb, rows=int(len(tin)), kind=kind, out_rows=int(np.sum(k == 1)),
                       wall_ms=round(wall, 3), kernel_ms=round(ms, 3), profile_entries=launches)
            sel = np.flatnonzero(k == 1)
            rec["exact_out"] = stats(pick_rows(o, sel))
            if kind == "mixed":
                rec["exact_in"] = stats(pick_rows(o, np.flatnonzero(k == 0)))
            if q == 1_000:
                rec.update(compare_out(p, tin[sel], tout[sel], amt[sel], delta[sel], allowed, pick_rows(o, sel)))
            emit(**rec)
            est = ms * 100_000 / q


def pick_rows(o, sel):
    """The per-row outputs of rows sel (with their token and leg offsets), as a namespace."""
    from types import SimpleNamespace
    tok = [np.arange(o.tok_off[r], o.tok_off[r + 1]) for r in sel]
    leg_off = np.concatenate([[0], np.cumsum(np.diff(o.leg_off)[sel])]).astype(np.int64)
    tok_off = np.concatenate([[0], np.cumsum([len(t) for t in tok])]).astype(np.int64)
    ti = np.concatenate(tok + [np.zeros(0, np.int64)]).astype(np.int64)
    return SimpleNamespace(paid=o.paid[sel], received=o.received[sel], status=o.status[sel],
                           solver_status=o.solver_status[sel], iterations=o.iterations[sel],
                           fun_evals=o.fun_evals[sel], merit=o.merit[sel], leg_off=leg_off, tok_off=tok_off,
                           token=o.token[ti], nu=o.nu[ti])


def hub(rng, budget_s, kind="in", sizes=(8, 64, 256)):
    p, n, others, nu, _ = hub_set(rng)

    def pick(q, nb):
        out = others[others > nb]
        tin = rng.choice(out, size=q)
        tout = out[(np.searchsorted(out, tin) + rng.integers(1, len(out), size=q)) % len(out)]
        return tin.astype(np.int64), tout.astype(np.int64)

    run(p, "hub", n, pick, lambda tin, tout: 1e-3 * 1e4 / nu[tin], budget_s, kind, sizes)
    p.close()


def headline(rng, budget_s, kind="in", sizes=(8, 64, 256)):
    m, n = 10_000_000, 50_000
    R, g, Ai = synth.product_pools(m, n, seed=1234)
    p = cr.DevicePools(n)
    p.add_product(R, g, Ai)
    p.finalize()
    emit(set="headline", pools=m, tokens=n)
    depth = np.zeros(n + 1)
    np.maximum.at(depth, Ai[:, 0], R[:, 0])
    np.maximum.at(depth, Ai[:, 1], R[:, 1])

    def pick(q, nb):
        ok = np.flatnonzero((Ai[:, 0] > nb) & (Ai[:, 1] > nb))
        sel = rng.choice(ok, size=q)
        side = rng.integers(0, 2, size=q)
        return Ai[sel, side].astype(np.int64), Ai[sel, 1 - side].astype(np.int64)

    run(p, "headline", n, pick, lambda tin, tout: 1e-3 * depth[tin], budget_s, kind, sizes)
    p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["hub", "headline"])
    ap.add_argument("--budget-s", type=float, default=20.0)
    ap.add_argument("--kind", choices=["in", "out", "mixed"], default="in")
    ap.add_argument("--B", default="8,64,256", help="mask sizes, comma-separated")
    args = ap.parse_args()
    sizes = tuple(int(x) for x in args.B.split(","))
    emit(card=card())
    rng = np.random.default_rng(2029)
    if args.only in (None, "hub"):
        hub(rng, args.budget_s, args.kind, sizes)
    if args.only in (None, "headline"):
        headline(rng, args.budget_s, args.kind, sizes)


if __name__ == "__main__":
    main()
