"""Host mirror of cfmm_find_order_paths_net / cfmm_quote_token_values_net (include/cfmm_b200.h).

The definition composes the existing calls: P_L is the result with max_hops = L.  Among the L whose
result is FILLED, the one with the best net (exact-in v − n·κ, larger; exact-out v + n·κ, smaller) is
taken, the larger L on a tie; with none, P_H as it is and net = value.

  net        one result's net, in the device's operations (one multiply, then one add or subtract)
  select     the selection over per-L (status, value, hops) triples
  paths      best_path_oracle.dp / find at L = 1 … H, selected per row
  values     token_value_oracle.dp at L = 1 … H, selected per token
  product    token_value_oracle.product at each L (exact-in, ProductTwoCoin arrays), selected per
             token, every reached level eligible: for sets without gaining cycles, where no walk
             repeats a pool
"""
from __future__ import annotations

import numpy as np

import best_path_oracle as bo
import token_value_oracle as tv

FILLED = 0


def net(value, hops, kappa, out):
    c = np.float64(hops) * np.float64(kappa)
    return float(np.float64(value) + c) if out else float(np.float64(value) - c)


def select(levels, kappa, out):
    """levels: (status, value, hops) for L = 1 … H.  Returns (L, net): the selected L (1-based), or H
    with net = value when no level filled."""
    sel, best = None, None
    for L, (st, v, n) in enumerate(levels, start=1):
        if st != FILLED:
            continue
        x = net(v, n, kappa, out)
        if sel is None or (x <= best if out else x >= best):
            sel, best = L, x
    if sel is None:
        return len(levels), float(levels[-1][1])
    return sel, best


def paths(rows, lists, n_tokens, allowed, H, quote, kappa):
    """best_path_oracle.dp at every L, selected: per row (walk, status, amount, net, L).  kappa [q]."""
    per_L = [bo.dp(rows, lists, n_tokens, allowed, L, quote) for L in range(1, H + 1)]
    out = []
    for r, (j, i, kind, amount) in enumerate(rows):
        res = [per_L[L][r] for L in range(H)]
        if not amount > 0.0:
            out.append(res[-1] + (0.0, H))
            continue
        L, x = select([(st, amt, len(w)) for w, st, amt in res], kappa[r], int(kind) == bo.EXACT_OUT)
        walk, st, amt = res[L - 1]
        out.append((walk, st, amt, x, L))
    return out


def find(pools, n_tokens, token_in, token_out, kind, amount, H, allowed, kappa, pairs=None):
    """best_path_oracle.find at every L, selected per row: find's tuple (hop_off, hop_pool, hop_token,
    hop_tender, hop_received, value, status) and net [q], L [q]."""
    per_L = [bo.find(pools, n_tokens, token_in, token_out, kind, amount, L, allowed, pairs) for L in range(1, H + 1)]
    rows = []
    for r in range(len(token_in)):
        def level(L):
            off, hp, ht, x, lam, value, status, _ = per_L[L - 1]
            a, b = off[r], off[r + 1]
            return (list(hp[a:b]), list(ht[a:b]), list(x[a:b]), list(lam[a:b]), float(value[r]), int(status[r]))
        levels = [level(L) for L in range(1, H + 1)]
        if not amount[r] > 0.0:
            rows.append(levels[-1] + (0.0, H))
            continue
        L, x = select([(lv[5], lv[4], len(lv[0])) for lv in levels], kappa[r], int(kind[r]) == bo.EXACT_OUT)
        rows.append(levels[L - 1] + (x, L))
    off = np.concatenate([[0], np.cumsum([len(x[0]) for x in rows])]).astype(np.int64)
    cat = lambda c, dt: np.array([v for x in rows for v in x[c]], dtype=dt)
    return (off, cat(0, np.int64), cat(1, np.int64), cat(2, np.float64), cat(3, np.float64),
            np.array([x[4] for x in rows]), np.array([x[5] for x in rows], np.uint8), np.array([x[6] for x in rows]),
            np.array([x[7] for x in rows]))


def values(root, kind, amount, lists, n_tokens, allowed, H, quote, kappa):
    """token_value_oracle.dp at every L, selected per token.  Returns (per_L results, value [n], hops
    [n], status [n], net [n], L [n], walk(t)) where walk(t) is the selected level's walk."""
    per_L = [tv.dp(root, kind, amount, lists, n_tokens, allowed, L, quote) for L in range(1, H + 1)]
    out = int(kind) == tv.EXACT_OUT
    value, hops = per_L[-1].value.copy(), per_L[-1].hops.copy()
    status, net_ = per_L[-1].status.copy(), per_L[-1].value.copy()
    sel = np.full(n_tokens, H)
    for t in range(n_tokens):
        if t == root - 1:
            continue
        L, x = select([(R.status[t], R.value[t], int(R.hops[t])) for R in per_L], kappa[t], out)
        R = per_L[L - 1]
        value[t], hops[t], status[t], net_[t], sel[t] = R.value[t], R.hops[t], R.status[t], x, L
    return per_L, value, hops, status, net_, sel, (lambda t: per_L[sel[t - 1] - 1].walk(t))


def product(R, g, Ai, active, n_tokens, root, amount, H, kappa, allowed=None):
    """The exact-in selection over token_value_oracle.product at L = 1 … H, every reached level
    eligible.  Returns (value [n], hops [n] (0 unreached), net [n])."""
    levels = [tv.product(R, g, Ai, active, n_tokens, root, amount, L, allowed)[:2] for L in range(1, H + 1)]
    kappa = np.broadcast_to(np.asarray(kappa, np.float64), (n_tokens,))
    val, lvl = levels[-1]
    value, hops = val.copy(), np.maximum(lvl, 0)
    net_ = val.copy()
    have = np.zeros(n_tokens, bool)
    for v, l in levels:
        ok = l > 0
        with np.errstate(invalid="ignore"):  # 0 · inf on unreached tokens, masked out below
            x = v - l * kappa  # float64 multiply, then subtract: the device's two roundings
        take = ok & (~have | (x >= net_))
        value[take], hops[take], net_[take] = v[take], l[take], x[take]
        have |= ok
    return value, hops, net_
