"""Host mirror of cfmm_quote_token_values (include/cfmm_b200.h), for the tests.

A pool is (a, b, pool, active) as in best_path_oracle.py: its ingest tokens (1-based) and a
swap_order_oracle pool (f, exact_out).

  dp        the definition as the header states it, for one row: level by level over every reached
            token (unchanged ones included), strict improvement, the (amount, neighbour, position)
            ranking, the walks rebuilt from the per-level predecessors.  The quotes come from a
            callable, so the same DP runs on host pool objects or on the device's cfmm_quote_swaps /
            cfmm_quote_swaps_exact_out (the GPU tests' composed reference)
  brute     every walk of at most H hops from the root, one active pool per hop: the best amount per
            token, for cross-checks where the quotes are monotone
  product   the exact-in DP vectorised with numpy for ProductTwoCoin pools given as arrays (the
            device's quote in the same IEEE operations), for sets of millions of pools
"""
from __future__ import annotations

import numpy as np

import swap_order_oracle as oo

INF = float("inf")
EXACT_IN, EXACT_OUT = 0, 1
FILLED, UNREACHABLE, REPEATS_POOL = 0, 2, 4


class Result:
    """One row: value / hops / status per token (index t - 1), pred[h - 1] = {t: (neighbour, handle)}
    of the tokens that changed at level h, and walk(t) in path order."""

    def __init__(self, root, out, n, value, lvl, pred):
        self.root, self.out, self.n, self.value, self.lvl, self.pred = root, out, n, value, lvl, pred
        self.hops = np.zeros(n, np.uint8)
        self.status = np.full(n, UNREACHABLE, np.uint8)
        for t in range(1, n + 1):
            if lvl[t - 1] < 0:
                continue
            steps = self.steps(t)
            hs = [k for _, _, k in steps]
            self.hops[t - 1] = len(steps)
            self.status[t - 1] = REPEATS_POOL if len(set(hs)) < len(hs) else FILLED

    def steps(self, t):
        """DP order from t: (token, neighbour, handle) per step; each predecessor at the latest level
        below the step's at which it changed."""
        out, h, u = [], int(self.lvl[t - 1]), t
        while h > 0:
            v, k = self.pred[h - 1][u]
            out.append((u, v, k))
            u, h = v, h - 1
            while h > 0 and u not in self.pred[h - 1]:
                h -= 1
        return out

    def walk(self, t):
        """[(tendered, delivered, handle)] in path order: root → t exact-in, t → root exact-out."""
        st = self.steps(t)
        return [(u, v, k) for u, v, k in st] if self.out else [(v, u, k) for u, v, k in reversed(st)]


def dp(root, kind, amount, lists, n_tokens, allowed, H, quote):
    """lists: {(lo, hi): [(pool handle, its ingest token 1, active), ...]} in cfmm_pair_pools order;
    allowed: mask [n_tokens] or None.  quote(reqs): for reqs [(handle, tok1, a, out)] the exact-in
    output for tender a of the ingest token 1 side (tok1) or the exact-out tender for want a, one
    float each."""
    out = int(kind) == EXACT_OUT
    S = int(root)
    val = np.full(n_tokens, INF if out else 0.0)
    val[S - 1] = float(amount)
    lvl = np.full(n_tokens, -1)
    lvl[S - 1] = 0
    ok = lambda t: t != S and (allowed is None or bool(allowed[t - 1]))
    pred = []
    for h in range(1, H + 1):
        reqs, meta = [], []
        for (a, b), lst in lists.items():
            for src, dst in ((a, b), (b, a)):
                if lvl[src - 1] < 0 or not ok(dst):
                    continue
                tender = dst if out else src
                for pos, (hnd, t1, act) in enumerate(lst):
                    if act:
                        reqs.append((hnd, tender == t1, float(val[src - 1]), out))
                        meta.append((dst, src, pos, hnd))
        best = {}
        for (dst, src, pos, hnd), v in zip(meta, quote(reqs) if reqs else []):
            if not (v < INF if out else v > 0.0):  # NaNs fail both
                continue
            key = (v if out else -v, src, pos)
            if dst not in best or key < best[dst][0]:
                best[dst] = (key, src, hnd)
        nval, level = val.copy(), {}
        for t, (key, src, hnd) in best.items():
            amt = key[0] if out else -key[0]
            if amt < val[t - 1] if out else amt > val[t - 1]:
                nval[t - 1], lvl[t - 1], level[t] = amt, h, (src, hnd)
        val = nval
        pred.append(level)
    return Result(S, out, n_tokens, val, lvl, pred)


def pool_lists(pools):
    """dp's lists for pool objects: each unordered pair's pools in pool order."""
    lists = {}
    for k, (a, b, _, act) in enumerate(pools):
        lists.setdefault((min(a, b), max(a, b)), []).append((k, a, act))
    return lists


def pool_quote(pools):
    def quote(reqs):
        return [float(oo.exact_out(pools[k][2], a, t1)[0]) if out else (float(pools[k][2].f(a, t1)) if a > 0 else 0.0)
                for k, t1, a, out in reqs]
    return quote


def brute(pools, n_tokens, root, kind, amount, H, allowed=None):
    """The best amount per token over every walk root → … → t (exact-in) or t → … → root (exact-out)
    of at most H hops through allowed tokens, the root only at its end, one active pool per hop (pools
    may repeat; quotes on the unchanged state).  0 / inf where no walk carries the amount."""
    out = int(kind) == EXACT_OUT
    best = np.full(n_tokens, INF if out else 0.0)
    best[root - 1] = amount
    adj = {}
    for k, (a, b, _, act) in enumerate(pools):
        if act:
            adj.setdefault(a, []).append((b, k))
            adj.setdefault(b, []).append((a, k))

    def go(u, v, depth):
        for w, k in adj.get(u, []):
            if w == root or (allowed is not None and not allowed[w - 1]):
                continue
            pool, a = pools[k][2], pools[k][0]
            x = float(oo.exact_out(pool, v, w == a)[0]) if out else float(pool.f(v, u == a))
            if not (x < INF if out else x > 0.0):
                continue
            if x < best[w - 1] if out else x > best[w - 1]:
                best[w - 1] = x
            if depth + 1 < H:
                go(w, x, depth + 1)

    go(root, float(amount), 0)
    return best


def product_f(R_in, R_out, g, x):
    """ProductTwoCoin's exact-in quote in the device's operations (two_coin_out<0>)."""
    k = R_in * R_out
    lam = R_out - k / (R_in + g * x)
    return np.where(R_out < lam, R_out, lam)


def product(R, g, Ai, active, n_tokens, root, amount, H, allowed=None):
    """The exact-in DP on ProductTwoCoin pools given as arrays (R [m, 2] and Ai [m, 2] in ingest
    order, g [m], active [m]; the global insertion index is the row).  Returns (value [n], lvl [n]
    (-1 unreached), frontier [H]: tokens changed per level)."""
    Ai = np.asarray(Ai, np.int64) - 1
    n, S = n_tokens, int(root) - 1
    val = np.zeros(n)
    val[S] = float(amount)
    lvl = np.full(n, -1, np.int64)
    lvl[S] = 0
    ok = np.ones(n, bool) if allowed is None else np.asarray(allowed, bool).copy()
    ok[S] = False
    idx = np.flatnonzero(active)
    front = np.zeros(n, bool)
    front[S] = True
    frontier = np.zeros(H, np.int64)
    for h in range(1, H + 1):
        if not front.any():
            break
        dsts, cs, srcs, gis = [], [], [], []
        for side in (0, 1):
            src, dst = Ai[idx, side], Ai[idx, 1 - side]
            sel = front[src] & ok[dst]
            k = idx[sel]
            c = product_f(R[k, side], R[k, 1 - side], g[k], val[src[sel]])
            keep = c > val[dst[sel]]
            dsts.append(dst[sel][keep]), cs.append(c[keep]), srcs.append(src[sel][keep]), gis.append(k[keep])
        dst, c, src, gi = (np.concatenate(x) for x in (dsts, cs, srcs, gis))
        order = np.lexsort((gi, src, -c, dst))
        dst, c = dst[order], c[order]
        first = np.ones(len(dst), bool)
        first[1:] = dst[1:] != dst[:-1]
        won, amt = dst[first], c[first]
        val[won], lvl[won] = amt, h
        front = np.zeros(n, bool)
        front[won] = True
        frontier[h - 1] = len(won)
    return val, lvl, frontier
