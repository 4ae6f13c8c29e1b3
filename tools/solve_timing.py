#!/usr/bin/env python
"""Device time of cfmm_solve on a ProductTwoCoin set per option set (measurement tool, not product
code): the projected L-BFGS-B solve of the box-constrained dual with its vector kernels between the
sweeps, a fixed number of function evaluations (pgtol = 0, so maxfun ends it), option sets
interleaved over the rounds.  Prints the GPU name, power limit and SM clock with the times.

    python tools/solve_timing.py [--m 10000000 --n 50000] [--maxfun 200] [--rounds 3] [--opt "k=v,k=v" ...]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cfmmrouter_b200 as cr  # noqa: E402
from cfmmrouter_b200 import synth  # noqa: E402


def gpu_facts():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        return out
    except (OSError, subprocess.CalledProcessError):
        return "not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=10_000_000)
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--maxfun", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--opt", action="append", default=[])
    a = ap.parse_args()
    R, g, Ai = synth.product_pools(a.m, a.n, seed=1234)
    lower = synth.dual_prices(a.n, "near")
    cfgs = []
    for o in a.opt or [""]:
        p = cr.DevicePools(a.n)
        p.add_product(R, g, Ai)
        p.finalize()
        for kv in (x for x in o.split(",") if x):
            k, v = kv.split("=")
            p.set_option(k, int(v))
        p.solve(lower, pgtol=0.0, maxfun=5)  # warm-up: stream packed, kernels loaded
        cfgs.append((o, p))
    res = {o: [] for o, _ in cfgs}
    for _ in range(a.rounds):
        for o, p in cfgs:
            x, info = p.solve(lower, pgtol=0.0, maxfun=a.maxfun)
            res[o].append((info["solve_ms"], info["fun_evals"], info["iterations"], x))
            print(json.dumps({"opt": o, "solve_ms": info["solve_ms"], "fun_evals": info["fun_evals"],
                              "iterations": info["iterations"], "gpu": gpu_facts()}), flush=True)
    x0 = res[cfgs[0][0]][0][3]
    for o, _ in cfgs:
        ms = [r[0] for r in res[o]]
        ev = [r[1] for r in res[o]]
        dx = max(float(np.max(np.abs(r[3] - x0) / np.abs(x0))) for r in res[o])
        print(json.dumps({"opt": o, "m": a.m, "n": a.n, "median_solve_ms": float(np.median(ms)), "solve_ms": ms,
                          "fun_evals": ev, "median_ms_per_eval": float(np.median(np.array(ms) / np.array(ev))),
                          "max_rel_diff_x_vs_first": dx}), flush=True)
    for _, p in cfgs:
        p.close()


if __name__ == "__main__":
    main()
