"""Host statements of the per-row mask calls' rules (include/cfmm_b200.h, "per-row masks"): a row's
list as the mask of the call without _rows, each row's own token set, and the levels an execute runs
its rows in."""
import numpy as np


def row_mask(tokens, n_tokens):
    """Row r's list (1-based tokens) as the mask [n_tokens] of the call without _rows."""
    m = np.zeros(n_tokens, bool)
    m[np.asarray(list(tokens), dtype=np.int64) - 1] = True
    return m


def own_subgraph(j, i, tokens):
    """A subgraph row's token set {j, i} ∪ B_r (its list may hold j and i)."""
    return {int(j), int(i)} | {int(t) for t in tokens}


def own_basket(i, entries, tokens):
    """A basket or limit row's token set {i} ∪ entries ∪ B_r."""
    return {int(i)} | {int(t) for t in entries} | {int(t) for t in tokens}


def levels(own):
    """cfmm_execute_paths' rule over one table of tokens: row r's level is 1 + the largest level of an
    earlier row sharing a token with it (1-based)."""
    last, lev = {}, []
    for s in own:
        L = 1 + max((last.get(t, 0) for t in s), default=0)
        for t in s:
            last[t] = L
        lev.append(L)
    return lev


def launches(lev, second):
    """The row-kernel launches of an execute: per level, one for its first-kernel rows and one for its
    second-kernel rows (exact-out or buy rows), each when the level has any."""
    n = 0
    for L in sorted(set(lev)):
        rows = [r for r, x in enumerate(lev) if x == L]
        n += any(not second[r] for r in rows) + any(second[r] for r in rows)
    return n
