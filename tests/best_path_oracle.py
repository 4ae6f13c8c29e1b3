"""Host mirror of cfmm_find_order_paths (include/cfmm_b200.h), for the tests.

A pool is (a, b, pool, active) as in hub_oracle.py: its ingest tokens (1-based) and a
swap_order_oracle pool (f, exact_out), so ProductTwoCoin and UniV3 amounts are the device's bits.

  dp      the definition as the header states it, level by level for a batch of rows: "at most h
          hops" over every reached predecessor, strict improvement, the (amount, hops, token,
          position) ranking, the walk rebuilt from the per-level predecessors.  The quotes come from
          a callable, so the same DP runs on host pool objects (find) or on the device's
          cfmm_quote_swaps / cfmm_quote_swaps_exact_out (the GPU tests' composed reference)
  find    dp on pool objects, each found walk priced by path_oracle.quote_path (the recursion of
          cfmm_quote_paths)
  brute   every walk of at most H hops through B, one active pool per hop, priced the same way: the
          best amount, for cross-checks where the quotes are monotone
"""
from __future__ import annotations

import itertools

import numpy as np

import hub_oracle as ho
import path_oracle as po
import swap_order_oracle as oo

INF = float("inf")
EXACT_IN, EXACT_OUT = 0, 1
FILLED, UNREACHABLE, REPEATS_POOL = 0, 2, 4


def _key(a, b):
    return (min(a, b), max(a, b))


def intermediates(n_tokens, allowed, j, i):
    return [t for t in range(1, n_tokens + 1) if allowed[t - 1] and t not in (j, i)]


def dp(rows, lists, n_tokens, allowed, H, quote):
    """rows: (j, i, kind, amount) each.  lists: {(lo, hi): [(pool handle, its ingest token 1,
    active), ...]} in cfmm_pair_pools order.  quote(reqs): for reqs [(handle, tok1, a, out)] the
    exact-in output for tender a (out False) or the exact-out tender for want a (out True), one float
    each.  Returns per row (walk [(tendered, delivered, handle)] in path order, status, amount): the
    amount is the DP's (received exact-in, paid exact-out), also for a REPEATS_POOL row."""
    st = []
    for j, i, kind, amount in rows:
        j, i, out = int(j), int(i), int(kind) == EXACT_OUT
        S, T = (i, j) if out else (j, i)
        st.append(dict(out=out, S=S, T=T, B=intermediates(n_tokens, allowed, j, i), a=float(amount),
                       val={S: float(amount)}, hops={S: 0}, preds=[]))
    live = [r for r, s in enumerate(st) if s["a"] > 0.0]

    def best_of(items):
        """items [(row, src, dst, a, hops)]: the best (key, src, handle) per item, or None; key =
        (−score, hops, src, position), score the amount (negated exact-out)."""
        reqs, where = [], []
        for n, (r, src, dst, a, _) in enumerate(items):
            tender = dst if st[r]["out"] else src
            for pos, (hnd, t1, act) in enumerate(lists.get(_key(src, dst), [])):
                if act:
                    reqs.append((hnd, tender == t1, a, st[r]["out"]))
                    where.append((n, pos, hnd))
        best = [None] * len(items)
        for (n, pos, hnd), (_, _, _, out), v in zip(where, reqs, quote(reqs) if reqs else []):
            if not (v < INF if out else v > 0.0):  # NaNs fail both
                continue
            r, src, _, _, hops = items[n]
            key = (v if out else -v, hops, src, pos)
            if best[n] is None or key < best[n][0]:
                best[n] = (key, src, hnd)
        return best

    for h in range(1, H):
        items = []
        for r in live:
            s = st[r]
            for u in s["B"]:
                items += [(r, u2, u, s["val"][u2], s["hops"][u2] + 1) for u2 in [s["S"]] + s["B"]
                          if u2 != u and u2 in s["val"]]
        cand = {}
        for it, b in zip(items, best_of(items)):
            if b is not None and ((it[0], it[2]) not in cand or b[0] < cand[(it[0], it[2])][0]):
                cand[(it[0], it[2])] = b
        for r in live:
            s = st[r]
            nval, nhops, pred = dict(s["val"]), dict(s["hops"]), {}
            for u in s["B"]:
                b = cand.get((r, u))
                if b is None:
                    continue
                amt = b[0][0] if s["out"] else -b[0][0]
                if u not in s["val"] or (amt < s["val"][u] if s["out"] else amt > s["val"][u]):
                    nval[u], nhops[u], pred[u] = amt, b[0][1], (b[1], b[2])
            s["val"], s["hops"] = nval, nhops
            s["preds"].append(pred)
    items = [(r, u, st[r]["T"], st[r]["val"][u], st[r]["hops"][u] + 1) for r in live
             for u in [st[r]["S"]] + st[r]["B"] if u in st[r]["val"]]
    final = {}
    for it, b in zip(items, best_of(items)):
        if b is not None and (it[0] not in final or b[0] < final[it[0]][0]):
            final[it[0]] = b
    res = []
    for r, s in enumerate(st):
        if not s["a"] > 0.0:
            res.append(([], FILLED, 0.0))
            continue
        if r not in final:
            res.append(([], UNREACHABLE, 0.0))
            continue
        key, u, hnd = final[r]
        amount = key[0] if s["out"] else -key[0]
        walk = [(u, s["T"], hnd)]  # DP order: (DP predecessor, token, handle)
        for h in range(H - 1, 0, -1):
            if u == s["S"]:
                break
            if u in s["preds"][h - 1]:
                u2, k = s["preds"][h - 1][u]
                walk.append((u2, u, k))
                u = u2
        path = [(b, a, k) for a, b, k in walk] if s["out"] else [(a, b, k) for a, b, k in reversed(walk)]
        ks = [k for _, _, k in path]
        res.append((path, REPEATS_POOL if len(set(ks)) < len(ks) else FILLED, amount))
    return res


def pool_quote(pools):
    """dp's quote over pool objects (handles are indices into pools)."""
    def quote(reqs):
        return [float(oo.exact_out(pools[k][2], a, t1)[0]) if out else (float(pools[k][2].f(a, t1)) if a > 0 else 0.0)
                for k, t1, a, out in reqs]
    return quote


def pool_lists(pools, pairs=None):
    """dp's lists for pool objects; pairs: each unordered pair's pool indices in cfmm_pair_pools
    order (default: ho.pair_lists, pool order)."""
    pairs = ho.pair_lists(pools) if pairs is None else pairs
    return {ab: [(k, pools[k][0], pools[k][3]) for k in ks] for ab, ks in pairs.items()}


def find(pools, n_tokens, token_in, token_out, kind, amount, max_hops, allowed, pairs=None):
    """cfmm_find_order_paths on the host: (hop_off [q + 1], hop_pool [Σ] indices into pools,
    hop_token [Σ], hop_tender [Σ], hop_received [Σ], value [q], status [q], dp [q]); dp is the DP's
    amount (also for REPEATS_POOL rows, which get no hops)."""
    rows = list(zip(token_in, token_out, kind, amount))
    out = []
    for (j, i, k, a), (path, status, amt) in zip(rows, dp(rows, pool_lists(pools, pairs), n_tokens, allowed,
                                                          int(max_hops), pool_quote(pools))):
        if status != FILLED or not path:
            out.append(([], [], [], [], 0.0, status, amt))
            continue
        ks = [h for _, _, h in path]
        x, lam, st = po.quote_path([pools[h][2] for h in ks], [t == pools[h][0] for t, _, h in path], k, a)
        out.append((ks, [b for _, b, _ in path], list(x), list(lam), float(x[0] if k == EXACT_OUT else lam[-1]), st,
                    amt))
    off = np.concatenate([[0], np.cumsum([len(r[0]) for r in out])]).astype(np.int64)
    cat = lambda c, dt: np.array([x for r in out for x in r[c]], dtype=dt)
    return (off, cat(0, np.int64), cat(1, np.int64), cat(2, np.float64), cat(3, np.float64),
            np.array([r[4] for r in out]), np.array([r[5] for r in out], dtype=np.uint8),
            np.array([r[6] for r in out]))


def brute(pools, n_tokens, j, i, kind, amount, max_hops, allowed):
    """The best amount over every walk j → … → i of at most max_hops hops through B, one active pool
    per hop (pools may repeat; quotes on the unchanged state), and one walk that reaches it (pool
    list), or (None, None) when no walk carries the amount: exact-in every hop's output > 0,
    exact-out every hop's tender finite."""
    pairs = ho.pair_lists(pools)
    B = intermediates(n_tokens, allowed, j, i)
    out = kind == EXACT_OUT
    best, arg = None, None
    for n in range(1, max_hops + 1):
        for mid in itertools.product(B, repeat=n - 1):
            toks = [j, *mid, i]
            choices = [[k for k in pairs.get(_key(a, b), []) if pools[k][3]] for a, b in zip(toks, toks[1:])]
            for ks in itertools.product(*choices):
                tok1 = [toks[h] == pools[k][0] for h, k in enumerate(ks)]
                objs = [pools[k][2] for k in ks]
                v = amount
                for h in (range(n - 1, -1, -1) if out else range(n)):
                    v = float(oo.exact_out(objs[h], v, tok1[h])[0]) if out else float(objs[h].f(v, tok1[h]))
                    if not (v < INF if out else v > 0.0):
                        break
                if not (v < INF if out else v > 0.0):
                    continue
                if best is None or (v < best if out else v > best):
                    best, arg = v, ks
    return best, arg
