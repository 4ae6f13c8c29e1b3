"""Objectives of the routing problem -- host side, unchanged in spirit from the
reference (src/objectives.jl): the conjugate f(ν), its gradient and the box
bounds on ν.  O(n_tokens) numpy work per L-BFGS-B evaluation; stays on the host
by design (BASELINE north_star)."""
from __future__ import annotations

import numpy as np

__all__ = ["Objective", "LinearNonnegative", "LinearHoldings", "BasketLiquidation", "BasketSwap", "LimitBasket",
           "Swap"]


class Objective:
    """abstract type Objective (src/objectives.jl:3)"""

    def f(self, v):
        raise NotImplementedError

    def grad(self, g, v):
        raise NotImplementedError

    def lower_limit(self):
        raise NotImplementedError

    def upper_limit(self):
        raise NotImplementedError

    def linear_term(self):
        """lin such that f(ν) = linᵀν on the box [lower_limit, upper_limit] (None: the objective is
        not of that form and the device solver cannot be used)."""
        return None


class LinearNonnegative(Objective):
    """U(Ψ) = cᵀΨ − I(Ψ ≥ 0)  (src/objectives.jl:51-79)."""

    def __init__(self, c):
        c = np.array(c, dtype=np.float64)
        if c.ndim != 1 or not np.all(c > 0):
            # ArgumentError("all elements must be strictly positive"), objectives.jl:54
            raise ValueError("all elements must be strictly positive")
        self.c = c

    def f(self, v):  # objectives.jl:62-67
        return 0.0 if np.all(self.c <= v) else np.inf

    def grad(self, g, v):  # objectives.jl:69-76
        g[:] = 0.0 if np.all(self.c <= v) else np.inf

    def lower_limit(self):  # objectives.jl:78
        return self.c + 1e-8

    def linear_term(self):  # f = 0 on the box
        return np.zeros_like(self.c)

    def upper_limit(self):  # objectives.jl:79
        return np.full_like(self.c, np.inf)


class LinearHoldings(Objective):
    """U(Ψ) = cᵀΨ − I(Ψ + h ≥ 0): value the net trade at outside prices c ≥ 0, where the net may
    spend up to the holdings h ≥ 0.  The conjugate is finite only on ν ≥ c, where it is
    hᵀ(ν − c): the box is LinearNonnegative's, c + 1e-8, and f(ν) = linᵀν − hᵀc with lin = h, so
    that f(ν*) plus the pools' value bounds the profit cᵀΨ.  With h = 0 it is LinearNonnegative(c)
    (with prices of 0 allowed); c = e_i with h = Δin is BasketLiquidation(i, Δin) and c = (1 at i,
    limit_k at each sold k) is LimitBasket, each up to its box."""

    def __init__(self, c, h):
        c = np.array(c, dtype=np.float64)
        h = np.array(h, dtype=np.float64)
        if c.ndim != 1 or c.shape != h.shape:
            raise ValueError("c and h need one entry per token")
        if not np.all(np.isfinite(c) & (c >= 0.0)):
            raise ValueError("every price must be finite and >= 0")
        if not np.all(np.isfinite(h) & (h >= 0.0)):
            raise ValueError("every holding must be finite and >= 0")
        self.c = c
        self.h = h

    def _const(self):
        """Σ_t h_t·c_t, in token order."""
        s = 0.0
        for t in range(len(self.c)):
            s += self.h[t] * self.c[t]
        return s

    def linear_term(self):
        return self.h.copy()

    def f(self, v):
        if np.any(np.asarray(v) < self.c):
            return np.inf
        return float(np.dot(self.h, v)) - self._const()

    def grad(self, g, v):
        if np.any(np.asarray(v) < self.c):
            g[:] = np.inf
        else:
            g[:] = self.h

    def lower_limit(self):
        return self.c + 1e-8

    def upper_limit(self):
        return np.full_like(self.c, np.inf)


class BasketLiquidation(Objective):
    """Ψ_i − I(Ψ_{-i} + Δin_{-i} = 0, Ψ_i ≥ 0)  (src/objectives.jl:92-129).
    `i` is 1-based, as in the reference."""

    def __init__(self, i, delta_in):
        delta_in = np.array(delta_in, dtype=np.float64)
        if not (0 < i <= len(delta_in)):
            raise ValueError("Invalid index i")  # objectives.jl:97
        self.i = int(i)
        self.delta_in = delta_in

    def f(self, v):  # objectives.jl:106-111
        if v[self.i - 1] >= 1.0:
            s = 0.0
            for j in range(len(v)):
                s += 0.0 if j == self.i - 1 else self.delta_in[j] * v[j]
            return s
        return np.inf

    def grad(self, g, v):  # objectives.jl:113-121
        if v[self.i - 1] >= 1.0:
            g[:] = self.delta_in
            g[self.i - 1] = 0.0
        else:
            g[:] = np.inf

    def linear_term(self):  # f = Σ_{j≠i} Δin_j ν_j on the box (ν_i >= 1 there)
        lin = self.delta_in.copy()
        lin[self.i - 1] = 0.0
        return lin

    def lower_limit(self):  # objectives.jl:123-128
        eps = np.sqrt(np.finfo(np.float64).eps)
        ret = np.full(len(self.delta_in), eps)
        ret[self.i - 1] = 1.0 + eps
        return ret

    def upper_limit(self):  # objectives.jl:129
        return np.full(len(self.delta_in), np.inf)


class BasketSwap(Objective):
    """Ψ_i − I(Ψ_{-i} + Δin_{-i} − Δout_{-i} >= 0): sell up to Δin and buy at least Δout of the
    other tokens, maximising the net of token i, which may be negative (the order pays on net).
    `i` is 1-based.  With Δout all zero it is BasketLiquidation(i, Δin), box included.  Otherwise
    the conjugate is finite only at ν_i = 1 (Ψ_i is free), where it is (Δin − Δout)ᵀν over the other
    tokens: the box fixes ν_i = 1 (lower = upper = 1) and keeps ν_t >= √eps for every other t."""

    def __init__(self, i, delta_in, delta_out):
        delta_in = np.array(delta_in, dtype=np.float64)
        delta_out = np.array(delta_out, dtype=np.float64)
        if delta_in.shape != delta_out.shape or delta_in.ndim != 1:
            raise ValueError("delta_in and delta_out need one entry per token")
        if not (0 < i <= len(delta_in)):
            raise ValueError("Invalid index i")
        self.i = int(i)
        self.delta_in = delta_in
        self.delta_out = delta_out
        self.buys = bool(np.any(np.delete(delta_out, self.i - 1) != 0.0))
        self._basket = BasketLiquidation(i, delta_in)

    def linear_term(self):
        if not self.buys:
            return self._basket.linear_term()
        lin = self.delta_in - self.delta_out
        lin[self.i - 1] = 0.0
        return lin

    def f(self, v):
        if not self.buys:
            return self._basket.f(v)
        if v[self.i - 1] != 1.0:
            return np.inf
        return float(np.dot(self.linear_term(), v))

    def grad(self, g, v):
        if not self.buys:
            return self._basket.grad(g, v)
        if v[self.i - 1] != 1.0:
            g[:] = np.inf
        else:
            g[:] = self.linear_term()

    def lower_limit(self):
        ret = self._basket.lower_limit()
        if self.buys:
            ret[self.i - 1] = 1.0
        return ret

    def upper_limit(self):
        ret = self._basket.upper_limit()
        if self.buys:
            ret[self.i - 1] = 1.0
        return ret


class LimitBasket(Objective):
    """Ψ_i + Σ_k c_k·Ψ_k − I(Ψ_k + Δin_k >= 0 at the entries, Ψ_t >= 0 elsewhere, i included): sell
    up to Δin_k of each token k for as long as the margin pays at least limit_k of token i per unit
    (a limit order with partial fills, settled in i).  `i` is 1-based; limit is per token (its i
    entry and the entries of tokens not sold are ignored).  The conjugate is finite only on ν_i >= 1,
    ν_k >= limit_k and ν_t >= 0, where it is Σ_{k≠i} Δin_k·(ν_k − limit_k): the box is
    BasketLiquidation's with each sold token's bound raised to fmax(limit_k, √eps), and
    f(ν) = linᵀν − Σ Δin·limit, so that f(ν*) plus the pools' value is the optimal surplus
    Ψ_i + Σ_k limit_k·Ψ_k.  With every limit 0 it is BasketLiquidation(i, Δin)."""

    def __init__(self, i, delta_in, limit):
        delta_in = np.array(delta_in, dtype=np.float64)
        limit = np.array(limit, dtype=np.float64)
        if delta_in.shape != limit.shape or delta_in.ndim != 1:
            raise ValueError("delta_in and limit need one entry per token")
        if not (0 < i <= len(delta_in)):
            raise ValueError("Invalid index i")
        if not np.all(np.isfinite(limit) & (limit >= 0.0)):
            raise ValueError("every limit must be finite and >= 0")
        self.i = int(i)
        self.delta_in = delta_in
        self.limit = limit
        self._basket = BasketLiquidation(i, delta_in)

    def _const(self):
        """Σ_{k≠i} Δin_k·limit_k, in token order."""
        s = 0.0
        for k in range(len(self.delta_in)):
            if k != self.i - 1:
                s += self.delta_in[k] * self.limit[k]
        return s

    def linear_term(self):
        return self._basket.linear_term()

    def f(self, v):
        if np.any(np.asarray(v) < self.lower_limit()):
            return np.inf
        return float(np.dot(self.linear_term(), v)) - self._const()

    def grad(self, g, v):
        if np.any(np.asarray(v) < self.lower_limit()):
            g[:] = np.inf
        else:
            g[:] = self.linear_term()

    def lower_limit(self):
        ret = np.fmax(self.limit, np.sqrt(np.finfo(np.float64).eps))
        ret[self.i - 1] = 1.0 + np.sqrt(np.finfo(np.float64).eps)
        return ret

    def upper_limit(self):
        return self._basket.upper_limit()


def Swap(i, j, delta, n):
    """Swap(i, j, δ, n): one-hot BasketLiquidation (src/objectives.jl:142-146)."""
    delta_in = np.zeros(n)
    delta_in[j - 1] = delta
    return BasketLiquidation(i, delta_in)
