"""Generate tests/golden/closed_forms.json: 50-digit (mpmath) evaluations of the
closed forms on the hot path, used to pin the CPU oracle independently of any
floating-point evaluation order.

Formulas restated from the reference (paths relative to the reference tree):
  ProductTwoCoin        src/cfmms.jl:125-126, 130-140
  GeometricMeanTwoCoin  src/cfmms.jl:180-181, 185-196
  UniV3                 src/cfmms.jl:251-259, 294-313, 321-337, 339-395
The reference itself (Julia) cannot run in this image; the known-answer cases of
its test-suite are included verbatim (test/cfmms.jl:74-86, 117-201).

Run:  python tests/golden/make_golden.py   (needs mpmath + numpy; deterministic)
"""
import json
import os

import mpmath as mp
import numpy as np

mp.mp.dps = 50
HERE = os.path.dirname(os.path.abspath(__file__))


def F(x):
    return mp.mpf(float(x))


def max0(x):
    return x if x > 0 else mp.mpf(0)


def product(R, g, v):
    R1, R2, g, v1, v2 = F(R[0]), F(R[1]), F(g), F(v[0]), F(v[1])
    k = R1 * R2
    d1 = max0(mp.sqrt(g * (v2 / v1) * k) - R1) / g
    d2 = max0(mp.sqrt(g * (v1 / v2) * k) - R2) / g
    l1 = max0(R1 - mp.sqrt(k / ((v1 / v2) * g)))
    l2 = max0(R2 - mp.sqrt(k / ((v2 / v1) * g)))
    return [d1, d2], [l1, l2]


def geomean(R, w, g, v):
    R1, R2, w1, w2, g, v1, v2 = (F(x) for x in (R[0], R[1], w[0], w[1], g, v[0], v[1]))
    eta = w1 / w2

    def gd(m, r1, r2, e):
        return max0((g * m * e * r1 * r2 ** e) ** (1 / (e + 1)) - r2) / g

    def gl(m, r1, r2, e):
        return max0(r1 - ((r2 * r1 ** (1 / e)) / (e * g * m)) ** (e / (1 + e)))

    return ([gd(v2 / v1, R2, R1, eta), gd(v1 / v2, R1, R2, 1 / eta)],
            [gl(v1 / v2, R1, R2, 1 / eta), gl(v2 / v1, R2, R1, eta)])


def univ3(cp, lt, lq, g, v):
    cp, g, v1, v2 = F(cp), F(g), F(v[0]), F(v[1])
    lt = [F(x) for x in lt]
    lq = [F(x) for x in lq]
    n = len(lt)
    cur = sum(1 for x in lt if x >= cp)

    def tick(idx):  # 1-based
        k = lq[idx - 1]
        pplus = lt[idx - 1]
        pminus = lt[idx] if idx < n else mp.mpf(0)
        a = mp.sqrt(k / pplus)
        b = mp.sqrt(k * pminus)
        p = pplus if idx > cur else (pminus if idx < cur else cp)
        return k, a, b, mp.sqrt(k / p) - a, mp.sqrt(k * p) - b

    def arb_pos(t, price):
        k, a, b, R1, R2 = t
        d = mp.sqrt(k / price) - (R1 + a)
        if d <= 0:
            return mp.mpf(0), mp.mpf(0)
        dmax = (k / b - (R1 + a)) if b > 0 else mp.inf
        if d >= dmax:
            return dmax, R2
        return d, (R2 + b) - mp.sqrt(price * k)

    D = [mp.mpf(0), mp.mpf(0)]
    L = [mp.mpf(0), mp.mpf(0)]
    p = v1 / v2
    if g * cp <= p <= cp / g:
        return D, L
    if p < g * cp:
        ids, price, di, li, flip = range(cur, n + 1), p / g, 0, 1, False
    else:
        ids, price, di, li, flip = range(cur, 0, -1), 1 / (g * p), 1, 0, True
    initial = True
    for idx in ids:
        t = tick(idx)
        if flip:
            t = (t[0], t[2], t[1], t[4], t[3])
        if t[0] == 0:
            initial = False
            continue
        d, l = arb_pos(t, price)
        if not initial and (d == 0 or l == 0):
            break
        D[di] += d
        L[li] += l
        initial = False
    D[di] /= g
    return D, L


def S(xs):
    return [mp.nstr(x, 40) for x in xs]


def main():
    rng = np.random.default_rng(20260923)
    out = {"meta": {"dps": 50, "generator": "tests/golden/make_golden.py"},
           "product": [], "geomean": [], "univ3": []}

    # reference known-answer cases, test/cfmms.jl:74-86
    kats = [([1.0, 1.0], 1.0, [1.0, 1.0]), ([1.0, 1.0], 1.0, [2.0, 2.0]),
            ([1.0, 1.0], 1.0, [2.0, 1.0]), ([1e3, 2e3], 0.997, [1.0, 1.0])]
    for R, g, v in kats:
        D, L = product(R, g, v)
        out["product"].append({"R": R, "gamma": g, "v": v, "Delta": S(D), "Lambda": S(L), "src": "kat"})
    for _ in range(96):
        R = (10.0 ** rng.uniform(-2, 4, size=2)).tolist()
        g = float(rng.choice([1.0, 0.997, float(rng.uniform(0.5, 1.0))]))
        v = rng.uniform(0.01, 1.0, size=2).tolist()
        D, L = product(R, g, v)
        out["product"].append({"R": R, "gamma": g, "v": v, "Delta": S(D), "Lambda": S(L), "src": "random"})

    gk = [([1e4, 2e4], [0.4, 0.6], 1.0, [1.0, 1.0]), ([1e4, 2e4], [0.5, 0.5], 0.997, [1.0, 1.0])]
    for R, w, g, v in gk:
        D, L = geomean(R, w, g, v)
        out["geomean"].append({"R": R, "w": w, "gamma": g, "v": v, "Delta": S(D), "Lambda": S(L), "src": "kat"})
    for _ in range(96):
        R = (10.0 ** rng.uniform(-1, 4, size=2)).tolist()
        w1 = float(rng.uniform(0.05, 0.95))
        w = [w1, 1.0 - w1]
        g = float(rng.choice([1.0, 0.997, float(rng.uniform(0.5, 1.0))]))
        v = rng.uniform(0.01, 1.0, size=2).tolist()
        D, L = geomean(R, w, g, v)
        out["geomean"].append({"R": R, "w": w, "gamma": g, "v": v, "Delta": S(D), "Lambda": S(L), "src": "random"})

    # reference scenarios, test/cfmms.jl:117-201
    cp, lt, lq = 15.0, [30.0, 20.0, 10.0, 5.0], [1.0, 2.0, 1.5, 0.0]
    for g in (1.0, 0.997):
        for v in ([15.0 if g == 1.0 else 15.0 * (1 + g) / 2, 1.0], [16.0, 1.0], [14.0, 1.0],
                  [25.0, 1.0], [7.5, 1.0], [4.0, 1.0], [35.0, 1.0]):
            D, L = univ3(cp, lt, lq, g, v)
            out["univ3"].append({"cp": cp, "lower_ticks": lt, "liquidity": lq, "gamma": g, "v": v,
                                 "Delta": S(D), "Lambda": S(L), "src": "test/cfmms.jl"})
    for _ in range(64):
        T = int(rng.integers(1, 9))
        c = float(np.exp(rng.uniform(np.log(0.1), np.log(10))))
        ladder = (c * 2.0 * np.cumprod(np.concatenate([[1.0], rng.uniform(0.5, 0.9, size=T - 1)]))).tolist()
        liq = (rng.uniform(0.0, 100.0, size=T) * (rng.random(T) > 0.2)).tolist()
        g = float(rng.choice([1.0, 0.997]))
        ratio = float(np.exp(rng.uniform(np.log(0.2), np.log(5.0))))
        v = [c * ratio, 1.0]
        D, L = univ3(c, ladder, liq, g, v)
        out["univ3"].append({"cp": c, "lower_ticks": ladder, "liquidity": liq, "gamma": g, "v": v,
                             "Delta": S(D), "Lambda": S(L), "src": "random"})

    with open(os.path.join(HERE, "closed_forms.json"), "w") as f:
        json.dump(out, f, indent=1)
    print({k: len(v) for k, v in out.items() if k != "meta"})


if __name__ == "__main__":
    main()
