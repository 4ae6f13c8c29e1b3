"""Host restatement of cfmm_modify_univ3_liquidity (include/cfmm_b200.h), for the tests: one row
at a time, boundary insertion by copy and the liquidity change as one IEEE double addition per
tick (numpy float64 adds round to nearest), so that ladders equal the device's bit for bit.

  insert_boundary   a ladder with one more boundary: the tick it falls in is split (both parts
                    keep its liquidity), above T₁ a new first tick with liquidity 0
  apply_row         one row (lo, hi, dL) on one ladder; False when a tick it adds to is left < 0
                    or not finite
  replay            rows in batch order on a CSR set of ladders; the first failing row or None
"""
from __future__ import annotations

import numpy as np

F = np.float64


def insert_boundary(lt, lq, b):
    """(lower_ticks, liquidity) with boundary b inserted; unchanged when some Tᵢ == b."""
    lt = np.asarray(lt, dtype=F)
    lq = np.asarray(lq, dtype=F)
    b = F(b)
    if np.any(lt == b):
        return lt.copy(), lq.copy()
    k = int(np.sum(lt > b))  # the ticks above b; b goes at position k
    inherit = lq[k - 1] if k > 0 else F(0.0)
    return np.insert(lt, k, b), np.insert(lq, k, inherit)


def apply_row(lt, lq, lo, hi, dL):
    """(lower_ticks, liquidity, ok) after one row: hi and lo inserted, then Lᵢ + dL on every tick
    whose upper bound Tᵢ has lo < Tᵢ <= hi."""
    lt, lq = insert_boundary(lt, lq, hi)
    lt, lq = insert_boundary(lt, lq, lo)
    on = (F(lo) < lt) & (lt <= F(hi))
    with np.errstate(all="ignore"):
        lq = lq.copy()
        lq[on] = lq[on] + F(dL)
        ok = bool(np.all((lq[on] >= 0.0) & np.isfinite(lq[on])))
    return lt, lq, ok


def replay(off, lt, lq, pools, lo, hi, dL):
    """Rows (pools[j], lo[j], hi[j], dL[j]) in order on the CSR set (off, lt, lq).  Returns
    (off, lt, lq, bad): the new CSR and None, or the unchanged inputs and the first failing row."""
    ladders = [(np.asarray(lt[off[i]:off[i + 1]], dtype=F), np.asarray(lq[off[i]:off[i + 1]], dtype=F))
               for i in range(len(off) - 1)]
    for j, i in enumerate(np.asarray(pools, dtype=np.int64)):
        a, b, ok = apply_row(*ladders[i], lo[j], hi[j], dL[j])
        if not ok:
            return off, lt, lq, j
        ladders[i] = (a, b)
    new_off = np.concatenate([[0], np.cumsum([len(a) for a, _ in ladders])]).astype(np.int64)
    return new_off, np.concatenate([a for a, _ in ladders]), np.concatenate([b for _, b in ladders]), None


def liquidity_at(lt, lq, price):
    """The liquidity of the tick holding `price` (Tᵢ₊₁ < price <= Tᵢ), 0 above T₁."""
    k = int(np.sum(np.asarray(lt) >= price))  # searchsortedlast, rev=true
    if k == 0:
        return F(0.0)
    return F(lq[k - 1])
