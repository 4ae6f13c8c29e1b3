"""Host mirror of cfmm_choose_order_hubs (include/cfmm_b200.h), for the tests.

A pool is (a, b, pool, active): its ingest tokens (1-based) and a swap_order_oracle pool (f,
exact_out), so ProductTwoCoin and UniV3 scores are the device's bits.

  pair_lists   the pools of every token pair, retired ones included
  adjacency    each token's neighbours ascending (the token adjacency of the arbitrage scan)
  hub_score    out_h (exact-in) or in_h (exact-out) of one candidate, and whether it is eligible
  choose       the kernel's shape: a warp per row whose lanes walk the shorter adjacency list, keep
               their best max_hubs in a sorted insert, and merge the heads warp-wide
  brute        every token as a candidate, ranked with sorted(): the definition, for cross-checks
"""
from __future__ import annotations

import numpy as np

import swap_order_oracle as oo

INF = float("inf")
EXACT_IN, EXACT_OUT = 0, 1


def pair_lists(pools):
    """{(lo, hi): [pool index, ...]} over the pools' unordered token pairs."""
    out = {}
    for k, (a, b, _, _) in enumerate(pools):
        out.setdefault((min(a, b), max(a, b)), []).append(k)
    return out


def adjacency(pairs, n_tokens):
    nbr = [[] for _ in range(n_tokens + 1)]
    for a, b in pairs:
        nbr[a].append(b)
        nbr[b].append(a)
    return [sorted(x) for x in nbr]


def _f(pool, x, tok1):
    return float(pool.f(x, tok1)) if x > 0.0 else 0.0


def best_f(pools, ks, t, x):
    """The largest exact-in quote for x of token t over the active pools ks (NaNs ignored; 0 if none)."""
    best = 0.0
    for k in ks:
        a, _, p, active = pools[k]
        if active:
            v = _f(p, x, t == a)
            if v > best:
                best = v
    return best


def best_exact_out(pools, ks, t, y):
    """The smallest exact-out tender of token t for y over the active pools ks (+inf if none)."""
    best = INF
    for k in ks:
        a, _, p, active = pools[k]
        if active:
            v = float(oo.exact_out(p, y, t == a)[0])
            if v < best:
                best = v
    return best


def hub_score(pools, pairs, j, h, i, kind, amount):
    """(score, eligible) of hub h for the row j → i."""
    kjh, khi = pairs.get((min(j, h), max(j, h)), []), pairs.get((min(h, i), max(h, i)), [])
    if kind == EXACT_IN:
        o = best_f(pools, khi, h, best_f(pools, kjh, j, amount))
        return o, o > 0.0
    c = best_exact_out(pools, khi, h, amount)
    x = best_exact_out(pools, kjh, j, c) if c < INF else INF
    return x, x < INF


def _before(s1, y1, s2, y2):
    return s1 > s2 or (s1 == s2 and y1 < y2)


def _row(pools, pairs, nbr, j, i, kind, amount, max_hubs, allowed):
    if not (amount > 0.0):
        return [], [], 0
    wj, wi = nbr[j], nbr[i]
    walk, other = (wj, set(wi)) if len(wj) <= len(wi) else (wi, set(wj))
    lanes = [[] for _ in range(32)]
    count = 0
    for e, h in enumerate(walk):
        if h not in other or (allowed is not None and not allowed[h - 1]):
            continue
        s, ok = hub_score(pools, pairs, j, h, i, kind, amount)
        if not ok:
            continue
        count += 1
        key = s if kind == EXACT_IN else -s
        lst = lanes[e % 32]
        pos = 0
        while pos < len(lst) and _before(*lst[pos], key, h):
            pos += 1
        lst.insert(pos, (key, h))
        del lst[max_hubs:]
    hubs, scores = [], []
    for _ in range(max_hubs):
        heads = [l[0] for l in lanes if l]
        if not heads:
            break
        best = heads[0]
        for c in heads[1:]:
            if _before(*c, *best):
                best = c
        for l in lanes:
            if l and l[0] == best:
                l.pop(0)
        hubs.append(best[1])
        scores.append(best[0] if kind == EXACT_IN else -best[0])
    return hubs, scores, count


def _pack(per_row):
    hub_off = np.concatenate([[0], np.cumsum([len(h) for h, _, _ in per_row])]).astype(np.int64)
    hubs = np.array([x for h, _, _ in per_row for x in h], dtype=np.int64)
    score = np.array([x for _, s, _ in per_row for x in s], dtype=np.float64)
    n_elig = np.array([c for _, _, c in per_row], dtype=np.int64)
    return hub_off, hubs, score, n_elig


def choose(pools, n_tokens, token_in, token_out, kind, amount, max_hubs, allowed=None):
    """cfmm_choose_order_hubs: (hub_off [q + 1], hubs [Σ], score [Σ], n_eligible [q])."""
    pairs = pair_lists(pools)
    nbr = adjacency(pairs, n_tokens)
    return _pack([_row(pools, pairs, nbr, int(j), int(i), int(k), float(a), int(max_hubs), allowed)
                  for j, i, k, a in zip(token_in, token_out, kind, amount)])


def brute(pools, n_tokens, token_in, token_out, kind, amount, max_hubs, allowed=None):
    """The same output from the definition: every token h ∉ {j, i} holding pools with both, sorted."""
    pairs = pair_lists(pools)
    rows = []
    for j, i, k, a in zip(token_in, token_out, kind, amount):
        j, i, k, a = int(j), int(i), int(k), float(a)
        el = []
        for h in range(1, n_tokens + 1):
            if h in (j, i) or (allowed is not None and not allowed[h - 1]) or not (a > 0.0):
                continue
            if (min(j, h), max(j, h)) not in pairs or (min(h, i), max(h, i)) not in pairs:
                continue
            s, ok = hub_score(pools, pairs, j, h, i, k, a)
            if ok:
                el.append((s, h))
        el.sort(key=lambda t: ((-t[0] if k == EXACT_IN else t[0]), t[1]))
        top = el[:int(max_hubs)]
        rows.append(([h for _, h in top], [s for s, _ in top], len(el)))
    return _pack(rows)
