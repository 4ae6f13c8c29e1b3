#!/usr/bin/env python
"""A/B timing of gradient-only ProductTwoCoin sweeps (not product code): one or more
builds of libcfmm_b200.so x option sets, on the same inputs on the same box, interleaved.

    python tools/ab_kernel.py [--m 10000000 --n 50000] [--lib name=path ...] [--opt "k=v,k=v" ...]

Prints the median / min of CUDA-event-bracketed launches per (lib, option set) and checks that
all of them agree on Ψ to 1e-9 relative (a guard against timing a broken path)."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from cfmmrouter_b200 import synth  # noqa: E402

_dp, _ip = C.POINTER(C.c_double), C.POINTER(C.c_int64)


def bind(path):
    lib = C.CDLL(path)
    lib.cfmm_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int64]
    lib.cfmm_add_product.argtypes = [C.c_void_p, C.c_int64, _dp, _dp, _ip]
    lib.cfmm_add_geomean.argtypes = [C.c_void_p, C.c_int64, _dp, _dp, _ip, _dp]
    lib.cfmm_finalize.argtypes = [C.c_void_p]
    lib.cfmm_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    lib.cfmm_sweep_device_view.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]
    lib.cfmm_profile_read_times.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.c_int64, _ip]
    lib.cfmm_destroy.argtypes = [C.c_void_p]
    lib.cfmm_last_error.restype = C.c_char_p
    lib.cfmm_last_error.argtypes = [C.c_void_p]
    return lib


class Ctx:
    def __init__(self, lib, n, R, g, Ai, pre, w=None):
        self.lib, self.n = lib, n
        self.ptype = 0 if w is None else 1
        self.ctx = C.c_void_p()
        assert lib.cfmm_create(C.byref(self.ctx), 0, n) == 0
        for k, v in pre.items():
            self.opt(k, v)
        if w is None:
            assert lib.cfmm_add_product(self.ctx, len(g), R.ctypes.data_as(_dp), g.ctypes.data_as(_dp),
                                        Ai.ctypes.data_as(_ip)) == 0
        else:
            assert lib.cfmm_add_geomean(self.ctx, len(g), R.ctypes.data_as(_dp), g.ctypes.data_as(_dp),
                                        Ai.ctypes.data_as(_ip), w.ctypes.data_as(_dp)) == 0
        assert lib.cfmm_finalize(self.ctx) == 0, lib.cfmm_last_error(self.ctx)

    def opt(self, k, v):
        rc = self.lib.cfmm_set_option(self.ctx, k.encode(), int(v))
        assert rc == 0, (k, v, self.lib.cfmm_last_error(self.ctx))

    def sweep(self, d_nu, stream):
        out = C.c_void_p()
        rc = self.lib.cfmm_sweep_device_view(self.ctx, d_nu.data_ptr(), 0, stream, C.byref(out))
        assert rc == 0, self.lib.cfmm_last_error(self.ctx)
        return out.value

    def times(self):
        cnt = C.c_int64()
        self.lib.cfmm_profile_read_times(self.ctx, self.ptype, None, 0, C.byref(cnt))
        buf = np.zeros(cnt.value, dtype=np.float32)
        self.lib.cfmm_profile_read_times(self.ctx, self.ptype, buf.ctypes.data_as(C.POINTER(C.c_float)), cnt.value, C.byref(cnt))
        return buf.astype(np.float64) * 1e3

    def close(self):
        self.lib.cfmm_destroy(self.ctx)


def from_ptr(ptr, count):
    class H:
        pass
    h = H()
    h.__cuda_array_interface__ = {"shape": (count,), "typestr": "<f8", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device="cuda")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, default=10_000_000)
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--lib", action="append", default=[])
    ap.add_argument("--opt", action="append", default=[])
    ap.add_argument("--pre", default="")
    ap.add_argument("--nu", default="near")
    ap.add_argument("--out", default="")
    ap.add_argument("--type", default="product", choices=["product", "geomean"])
    ap.add_argument("--flush", action="store_true", help="write 256 MB (> L2) before every timed launch")
    a = ap.parse_args()
    libs = dict(x.split("=", 1) for x in a.lib) or {"new": os.path.join(ROOT, "cfmmrouter.jl_b200", "libcfmm_b200.so")}
    optsets = a.opt or [""]
    w = None
    if a.type == "geomean":
        R, g, Ai, w = synth.geomean_pools(a.m, a.n)
    else:
        R, g, Ai = synth.product_pools(a.m, a.n, seed=1234)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda") if a.flush else None
    flush_rd = torch.zeros(32 << 20, dtype=torch.int64, device="cuda") if a.flush else None  # read pass: no dirty lines left
    v = synth.dual_prices(a.n, a.nu)
    d_nu = torch.from_numpy(v).cuda()
    st = torch.cuda.current_stream().cuda_stream
    pre = dict((kv.split("=")[0], int(kv.split("=")[1])) for kv in a.pre.split(",") if kv)
    cfgs = []
    for lname, path in libs.items():
        lib = bind(path)
        for o in optsets:
            kv = dict((x.split("=")[0], int(x.split("=")[1])) for x in o.split(",") if x)
            try:
                c = Ctx(lib, a.n, R, g, Ai, pre, w)
                for k, val in kv.items():
                    c.opt(k, val)
                c.opt("sweep_events", 0)
            except AssertionError as e:
                print(json.dumps({"lib": lname, "opt": o, "error": str(e)}), flush=True)
                continue
            cfgs.append((f"{lname}[{o}]", c))
    ref = None
    res = {name: [] for name, _ in cfgs}
    for name, c in cfgs:
        for _ in range(5):
            ptr = c.sweep(d_nu, st)
        torch.cuda.synchronize()
        psi = from_ptr(ptr, a.n + 1).clone().cpu().numpy()
        if ref is None:
            ref = psi
        err = float(np.max(np.abs(psi - ref)) / max(np.max(np.abs(ref)), 1e-300))
        print(json.dumps({"cfg": name, "psi_rel_diff_vs_first": err}), flush=True)
    for r in range(a.rounds):  # interleave the configurations: clock / thermal drift hits all alike
        for name, c in cfgs:
            c.opt("profile", a.iters)
            for _ in range(a.iters):
                if flush_buf is not None:
                    flush_buf.zero_()
                    flush_rd.sum()
                c.sweep(d_nu, st)
            torch.cuda.synchronize()
            res[name].append(c.times())
            c.opt("profile", 0)
    out = []
    for name, _ in cfgs:
        t = np.concatenate(res[name])
        row = {"cfg": name, "type": a.type, "flushed": bool(a.flush), "m": a.m, "n": a.n, "median_us": float(np.median(t)), "mean_us": float(t.mean()),
               "min_us": float(t.min()), "p95_us": float(np.quantile(t, 0.95)), "launches": len(t),
               "round_medians_us": [round(float(np.median(x)), 3) for x in res[name]]}
        print(json.dumps(row), flush=True)
        out.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    for _, c in cfgs:
        c.close()


if __name__ == "__main__":
    main()
