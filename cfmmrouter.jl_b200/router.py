"""Router / route! / find_arb! / netflows -- the host-side mirror of
src/router.jl, with the inner loop (the find_arb! sweep over every pool and the
two fold loops of the L-BFGS-B callback) replaced by libcfmm_b200.so.

What stays on the host, as in BASELINE's north_star: the Objective
(objectives.py) and the L-BFGS-B outer iteration (scipy's L-BFGS-B, the same
Nocedal/Zhu/Byrd algorithm LBFGSB.jl wraps; src/router.jl:60, 105).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
from types import SimpleNamespace

from . import _lib
from .cfmms import CFMM, GeometricMeanTwoCoin, ProductTwoCoin, UniV3
from .objectives import Objective

__all__ = ["DevicePools", "write_pool_file", "pool_file_info", "Router", "route", "find_arb", "netflows", "netflows_",
           "update_reserves", "shard_range"]


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int64))


def shard_range(m: int, world: int, rank: int):
    """Contiguous, balanced split of m pools over `world` ranks."""
    lo = (m * rank) // world
    hi = (m * (rank + 1)) // world
    return lo, hi


def write_pool_file(path, n_tokens: int, R, gamma, Ai, w=None):
    """Write ProductTwoCoin (w is None) or GeometricMeanTwoCoin pools as a flat pool file."""
    R = np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 2)
    gamma = np.ascontiguousarray(gamma, dtype=np.float64).reshape(-1)
    Ai = np.ascontiguousarray(Ai, dtype=np.int64).reshape(-1, 2)
    wp = None
    if w is not None:
        w = np.ascontiguousarray(w, dtype=np.float64).reshape(-1, 2)
        wp = _dp(w)
    rc = _lib.load().cfmm_pool_file_write(str(path).encode(), _lib.POOL_GEOMEAN if w is not None else _lib.POOL_PRODUCT,
                                          int(n_tokens), len(gamma), _dp(R), _dp(gamma), _ip(Ai), wp)
    if rc != _lib.CFMM_OK:
        raise OSError(f"cannot write pool file {path}")


def pool_file_info(path):
    """(pool type, n_tokens, m) of a flat pool file."""
    t, n, m = C.c_int(), C.c_int64(), C.c_int64()
    rc = _lib.load().cfmm_pool_file_info(str(path).encode(), C.byref(t), C.byref(n), C.byref(m))
    if rc != _lib.CFMM_OK:
        raise OSError(f"{path} is not a CFMM pool file")
    return t.value, n.value, m.value


def is_row_lists(allowed):
    """Whether `allowed` is one token list per row (a list or tuple of sequences, as Router.choose_hubs
    returns) rather than one mask over the tokens."""
    return isinstance(allowed, (list, tuple)) and all(isinstance(a, (list, tuple, np.ndarray)) for a in allowed)


def pack_row_lists(allowed, n_tokens, own, room, what):
    """(allow_off [q + 1], allow_token) int64 of the *_rows calls from one list of 1-based tokens per
    row, with their argument errors: q lists (q = len(own)); integer tokens in 1..n_tokens; none twice
    in a row; and at most room[r] tokens in row r's list outside own[r], the row's own tokens.  The
    checks run on the whole CSR at once (a batch holds many rows); an error names the first bad row."""
    q = len(own)
    if len(allowed) != q:
        raise ValueError(f"{what}: allowed needs one token list per row ({q})")
    rows = [np.asarray(lst).reshape(-1) for lst in allowed]
    for r, a in enumerate(rows):
        if len(a) and not np.issubdtype(a.dtype, np.integer):
            raise ValueError(f"{what}: row {r}: allowed tokens must be integers")
    lens = np.array([len(a) for a in rows], dtype=np.int64)
    off = np.zeros(q + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    tok = np.concatenate(rows).astype(np.int64) if off[-1] else np.zeros(0, dtype=np.int64)
    row = np.repeat(np.arange(q, dtype=np.int64), lens)
    bad = np.flatnonzero((tok < 1) | (tok > n_tokens))
    if len(bad):
        raise ValueError(f"{what}: row {row[bad[0]]}: an allowed token is outside 1..{n_tokens}")
    key = row * (n_tokens + 1) + tok
    ks = np.sort(key)
    dup = np.flatnonzero(ks[1:] == ks[:-1])
    if len(dup):
        raise ValueError(f"{what}: row {ks[dup[0]] // (n_tokens + 1)}: an allowed token is listed twice")
    own_len = np.array([len(o) for o in own], dtype=np.int64)
    own_key = np.repeat(np.arange(q, dtype=np.int64), own_len) * (n_tokens + 1) + \
        np.array([t for o in own for t in o], dtype=np.int64)
    extra = np.bincount(row[~np.isin(key, own_key)], minlength=q)
    over = np.flatnonzero(extra > np.asarray(room, dtype=np.int64))
    if len(over):
        r = over[0]
        raise ValueError(f"{what}: row {r}: {extra[r]} allowed tokens besides the row's own, more than {room[r]}")
    return off, np.ascontiguousarray(tok)


def _row_args(n_tokens, q, allowed, limit, opts, what, own=None, room=None):
    """(the allowed tokens as ctypes arguments, the limits, the options by reference or None) of a
    subgraph, basket or limit call, with the Python argument errors.  The allowed tokens: a namespace
    with rows (True for one token list per row, which selects the *_rows call: own and room give each
    row's own tokens and its room, as pack_row_lists takes them) and args (the mask, or allow_off and
    allow_token)."""
    if allowed is None:
        raise ValueError(f"{what}: allowed (a mask over the tokens, or one token list per row) is required")
    if own is not None and is_row_lists(allowed):
        off, tok = pack_row_lists(allowed, n_tokens, own, room, what)
        masks = SimpleNamespace(rows=True, args=(_ip(off), _ip(tok)))
    else:
        mask = np.ascontiguousarray(allowed, dtype=bool).reshape(-1).astype(np.uint8)
        if len(mask) != n_tokens:
            raise ValueError(f"{what}: allowed must have {n_tokens} entries, one per token")
        masks = SimpleNamespace(rows=False, args=(mask.ctypes.data_as(C.POINTER(C.c_uint8)),))
    if limit is not None:
        limit = np.ascontiguousarray(limit, dtype=np.float64).reshape(-1)
        if len(limit) != q:
            raise ValueError(f"limit must have {q} entries, one per row")
    o = None
    if opts is not None:
        d = {"max_iter": 1000, "max_fun": 4000, "rtol": 1e-4, "factr": 0.0}
        d.update(opts)
        o = _lib.SubgraphOpts(int(d["max_iter"]), int(d["max_fun"]), float(d["rtol"]), float(d["factr"]))
    return masks, limit, None if o is None else C.byref(o)


def _price_arb_opts(opts):
    """cfmm_price_arb_opts by reference from a dict of max_iter, max_fun, rtol, factr and atol (None:
    NULL, the defaults)."""
    if opts is None:
        return None
    d = {"max_iter": 1000, "max_fun": 4000, "rtol": 1e-4, "factr": 0.0, "atol": 0.0}
    d.update(opts)
    return C.byref(_lib.PriceArbOpts(int(d["max_iter"]), int(d["max_fun"]), float(d["rtol"]), float(d["factr"]),
                                     float(d["atol"])))


def _basket_room(token_out, basket_off, basket_token):
    """Each basket or limit row's own tokens (token_out and the entries) and its room for other allowed
    tokens: CFMM_SUBGRAPH_MAX_TOKENS + 1 tokens besides token_out, entries included."""
    own = [[int(token_out[r])] + [int(t) for t in basket_token[basket_off[r]:basket_off[r + 1]]]
           for r in range(len(token_out))]
    return own, [_lib.SUBGRAPH_MAX_TOKENS + 2 - len(o) for o in own]


def _entry_kind(kind, basket_off, limit, what):
    """The entry kinds of a basket call as a uint8 array (None: every entry sold, and the call is
    cfmm_quote/execute_basket_orders), with the Python argument errors: a scalar applies to every
    entry; a kind other than 0 (sold) or 1 (bought); a NaN limit, or a +inf limit on any row."""
    if kind is None:
        return None
    NE = int(basket_off[-1])
    k = np.asarray(kind)
    if k.ndim == 0:
        k = np.full(NE, k)
    k = k.reshape(-1)
    if len(k) != NE:
        raise ValueError(f"{what}: kind must have {NE} entries, one per basket entry (or be a scalar)")
    if not np.all(np.isin(k, (_lib.SWAP_EXACT_IN, _lib.SWAP_EXACT_OUT))):
        raise ValueError(f"{what}: kind must be 0 (sold) or 1 (bought)")
    if limit is not None and np.any(np.isnan(limit) | (limit == np.inf)):
        raise ValueError(f"{what}: a limit (the minimum received) is NaN or +inf")
    return np.ascontiguousarray(k, dtype=np.uint8)


def _row_kind(kind, q, limit, what):
    """The kinds of a subgraph call as a uint8 array (None: every row exact-in, passed as NULL), with
    the Python argument errors: a scalar applies to every row; a kind other than 0 (exact-in) or 1
    (exact-out); a limit that is NaN, or +inf on an exact-in row (the minimum received)."""
    if kind is None:
        return None
    k = np.asarray(kind)
    if k.ndim == 0:
        k = np.full(q, k)
    k = k.reshape(-1)
    if len(k) != q:
        raise ValueError(f"{what}: kind must have {q} entries, one per row (or be a scalar)")
    if not np.all(np.isin(k, (_lib.SWAP_EXACT_IN, _lib.SWAP_EXACT_OUT))):
        raise ValueError(f"{what}: kind must be 0 (exact-in) or 1 (exact-out)")
    k = np.ascontiguousarray(k, dtype=np.uint8)
    if limit is not None:
        if np.any(np.isnan(limit)):
            raise ValueError(f"{what}: a limit is NaN")
        if np.any(np.isinf(limit) & (k == _lib.SWAP_EXACT_IN)):
            raise ValueError(f"{what}: an exact-in limit (the minimum received) is +inf")
    return k


def _order_paths(pools, token_in, token_out, kind, amount, max_hops, allowed, hop_cost):
    """DevicePools.find_order_paths (hop_cost None) and find_order_paths_net."""
    tin = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
    tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
    kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
    amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
    q = len(tin)
    if not (len(tout) == len(kind) == len(amount) == q):
        raise ValueError("find_order_paths: token_in, token_out, kind and amount need one entry per row")
    mask = np.ascontiguousarray(allowed, dtype=bool).reshape(-1).astype(np.uint8)
    if len(mask) != pools.n_tokens:
        raise ValueError(f"find_order_paths: allowed must have {pools.n_tokens} entries, one per token")
    u8, i32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int)
    cap = max(q * max(int(max_hops), 0), 1)
    hop_off = np.zeros(q + 1, dtype=np.int64)
    typ, pool, tok = np.zeros(cap, dtype=np.int32), np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.int64)
    tender, received = np.zeros(cap), np.zeros(cap)
    value, status = np.zeros(q), np.zeros(q, dtype=np.uint8)
    outs = (_ip(hop_off), typ.ctypes.data_as(i32), _ip(pool), _ip(tok), _dp(tender), _dp(received), _dp(value),
            status.ctypes.data_as(u8))
    if hop_cost is None:
        pools._chk(pools._lib.cfmm_find_order_paths(pools._ctx, q, _ip(tin), _ip(tout), kind.ctypes.data_as(u8),
                                                  _dp(amount), int(max_hops), mask.ctypes.data_as(u8), *outs))
    else:
        cost = np.ascontiguousarray(hop_cost, dtype=np.float64).reshape(-1)
        if len(cost) != q:
            raise ValueError("find_order_paths_net: hop_cost needs one entry per row")
        net = np.zeros(q)
        pools._chk(pools._lib.cfmm_find_order_paths_net(pools._ctx, q, _ip(tin), _ip(tout), kind.ctypes.data_as(u8),
                                                      _dp(amount), int(max_hops), mask.ctypes.data_as(u8),
                                                      _dp(cost), *outs, _dp(net)))
    n = int(hop_off[-1])
    found = (hop_off, typ[:n].copy(), pool[:n].copy(), tok[:n].copy(), tender[:n].copy(), received[:n].copy(),
             value, status)
    return found if hop_cost is None else found + (net,)


def _token_values(pools, root, kind, amount, max_hops, allowed, requests, hop_cost):
    """DevicePools.quote_token_values (hop_cost None) and quote_token_values_net."""
    root = np.ascontiguousarray(root, dtype=np.int64).reshape(-1)
    kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
    amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
    q, n, H = len(root), pools.n_tokens, int(max_hops)
    if not (len(kind) == len(amount) == q):
        raise ValueError("quote_token_values: root, kind and amount need one entry per row")
    u8, i32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int)
    mask = None
    if allowed is not None:
        mask = np.ascontiguousarray(allowed, dtype=bool).reshape(-1).astype(np.uint8)
        if len(mask) != n:
            raise ValueError(f"quote_token_values: allowed must have {n} entries, one per token")
    rows = toks = np.zeros(0, dtype=np.int64)
    if requests is not None:
        rows = np.ascontiguousarray(requests[0], dtype=np.int64).reshape(-1)
        toks = np.ascontiguousarray(requests[1], dtype=np.int64).reshape(-1)
        if len(rows) != len(toks):
            raise ValueError("quote_token_values: requests need one row per token")
    k = len(rows)
    value = np.zeros((q, n))
    hops, status = np.zeros((q, n), dtype=np.uint8), np.zeros((q, n), dtype=np.uint8)
    frontier = np.zeros((q, max(H, 0)), dtype=np.int64)
    cap = max(k * max(H, 0), 1)
    hop_off = np.zeros(k + 1, dtype=np.int64)
    typ, pool, tok = np.zeros(cap, dtype=np.int32), np.zeros(cap, dtype=np.int64), np.zeros(cap, dtype=np.int64)
    tender, received, rstatus = np.zeros(cap), np.zeros(cap), np.zeros(max(k, 1), dtype=np.uint8)
    ins = (pools._ctx, q, _ip(root), kind.ctypes.data_as(u8), _dp(amount), H,
           None if mask is None else mask.ctypes.data_as(u8))
    reqs = (_ip(frontier), k, _ip(rows), _ip(toks), _ip(hop_off), typ.ctypes.data_as(i32), _ip(pool), _ip(tok),
            _dp(tender), _dp(received), rstatus.ctypes.data_as(u8))
    if hop_cost is None:
        pools._chk(pools._lib.cfmm_quote_token_values(*ins, _dp(value), hops.ctypes.data_as(u8),
                                                    status.ctypes.data_as(u8), *reqs))
        head = (value, hops, status, frontier)
    else:
        cost = np.ascontiguousarray(hop_cost, dtype=np.float64).reshape(-1)
        if len(cost) != n:
            raise ValueError(f"quote_token_values_net: hop_cost must have {n} entries, one per token")
        net = np.zeros((q, n))
        pools._chk(pools._lib.cfmm_quote_token_values_net(*ins, _dp(cost), _dp(value), hops.ctypes.data_as(u8),
                                                        status.ctypes.data_as(u8), _dp(net), *reqs))
        head = (value, hops, status, net, frontier)
    if requests is None:
        return head
    m = int(hop_off[-1])
    return head + (hop_off, typ[:m].copy(), pool[:m].copy(), tok[:m].copy(), tender[:m].copy(),
                   received[:m].copy(), rstatus[:k].copy())


class DevicePools:
    """One GPU's shard of the pool set: a thin object wrapper over cfmm_ctx."""

    def __init__(self, n_tokens: int, device: int = 0):
        self._lib = _lib.load()
        self._ctx = C.c_void_p()
        self._ptr_args = {}
        rc = self._lib.cfmm_create(C.byref(self._ctx), int(device), int(n_tokens))
        if rc != _lib.CFMM_OK:
            msg = self._lib.cfmm_last_error(None)
            raise _lib.CFMMError(rc, msg.decode() if msg else "")
        self.n_tokens = int(n_tokens)
        self.device = int(device)
        self.peer_attached = False
        self._univ3_ticks = np.zeros(0, dtype=np.int64)  # tick count per UniV3 pool (update_univ3 checks)
        self._psi = np.zeros(self.n_tokens)
        self._acc = C.c_double(0.0)
        # pinned staging for sweep(): ν in, [Ψ; acc] out (contiguous) -- the buffers the library
        # replays its {H2D, sweep, D2H} graph on (cfmm_b200.h, option "sweep_graphs")
        nbytes = 8 * (2 * self.n_tokens + 1)
        self._pin = self._lib.cfmm_host_alloc(nbytes)
        if not self._pin:
            self._lib.cfmm_destroy(self._ctx)
            raise MemoryError("cfmm_host_alloc failed")
        buf = (C.c_double * (2 * self.n_tokens + 1)).from_address(self._pin)
        arr = np.frombuffer(buf, dtype=np.float64)
        self._pin_nu, self._pin_out = arr[:self.n_tokens], arr[self.n_tokens:]

    # -- ingest -------------------------------------------------------------
    def _chk(self, rc):
        _lib.check(self._lib, self._ctx, rc)

    def add_product(self, R, gamma, Ai):
        self._product(self._lib.cfmm_add_product, R, gamma, Ai)

    def add_geomean(self, R, gamma, Ai, w):
        self._geomean(self._lib.cfmm_add_geomean, R, gamma, Ai, w)

    def add_univ3(self, current_price, gamma, Ai, tick_off, lower_ticks, liquidity):
        self._univ3(self._lib.cfmm_add_univ3, current_price, gamma, Ai, tick_off, lower_ticks, liquidity)

    def _product(self, fn, R, gamma, Ai):
        R = np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 2)
        gamma = np.ascontiguousarray(gamma, dtype=np.float64).reshape(-1)
        Ai = np.ascontiguousarray(Ai, dtype=np.int64).reshape(-1, 2)
        if not (len(R) == len(gamma) == len(Ai)):
            raise ValueError("R, gamma, Ai must describe the same number of pools")
        self._chk(fn(self._ctx, len(gamma), _dp(R), _dp(gamma), _ip(Ai)))

    def _geomean(self, fn, R, gamma, Ai, w):
        R = np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 2)
        w = np.ascontiguousarray(w, dtype=np.float64).reshape(-1, 2)
        gamma = np.ascontiguousarray(gamma, dtype=np.float64).reshape(-1)
        Ai = np.ascontiguousarray(Ai, dtype=np.int64).reshape(-1, 2)
        if not (len(R) == len(gamma) == len(Ai) == len(w)):
            raise ValueError("R, gamma, Ai, w must describe the same number of pools")
        self._chk(fn(self._ctx, len(gamma), _dp(R), _dp(gamma), _ip(Ai), _dp(w)))

    def _univ3(self, fn, current_price, gamma, Ai, tick_off, lower_ticks, liquidity):
        cp = np.ascontiguousarray(current_price, dtype=np.float64).reshape(-1)
        gamma = np.ascontiguousarray(gamma, dtype=np.float64).reshape(-1)
        Ai = np.ascontiguousarray(Ai, dtype=np.int64).reshape(-1, 2)
        off = np.ascontiguousarray(tick_off, dtype=np.int64).reshape(-1)
        lt = np.ascontiguousarray(lower_ticks, dtype=np.float64).reshape(-1)
        lq = np.ascontiguousarray(liquidity, dtype=np.float64).reshape(-1)
        if not (len(cp) == len(gamma) == len(Ai) == len(off) - 1) or len(lt) != len(lq) \
                or (len(off) and off[-1] != len(lt)):
            raise ValueError("inconsistent UniV3 CSR arrays")
        self._chk(fn(self._ctx, len(cp), _dp(cp), _dp(gamma), _ip(Ai), _ip(off), _dp(lt), _dp(lq)))
        self._univ3_ticks = np.concatenate([self._univ3_ticks, np.diff(off)])

    def add_file(self, path: str):
        """Add the pools of a flat pool file (write_pool_file / cfmm_pool_file_write)."""
        self._chk(self._lib.cfmm_add_pool_file(self._ctx, str(path).encode()))

    def finalize(self):
        self._chk(self._lib.cfmm_finalize(self._ctx))

    @property
    def num_pools(self) -> int:
        return int(self._lib.cfmm_num_pools(self._ctx))

    def set_option(self, key: str, value: int):
        self._chk(self._lib.cfmm_set_option(self._ctx, key.encode(), int(value)))

    # -- the hot path ---------------------------------------------------------
    def sweep(self, v, materialize: bool = False):
        """find_arb!(r, v) + both folds; returns (psi [n_tokens], acc)."""
        v = np.ascontiguousarray(v, dtype=np.float64)
        if v.shape != (self.n_tokens,):
            raise ValueError(f"v must have length {self.n_tokens}")
        np.copyto(self._pin_nu, v)
        base = self._pin
        n8 = 8 * self.n_tokens
        dp = C.POINTER(C.c_double)
        self._chk(self._lib.cfmm_sweep(self._ctx, C.cast(base, dp), C.cast(base + n8, dp),
                                       C.cast(base + 2 * n8, dp), 1 if materialize else 0))
        return self._pin_out[:self.n_tokens].copy(), float(self._pin_out[self.n_tokens])

    def sweep_into(self, v_ptr: int, psi_ptr: int, acc_ptr: int, materialize: bool = False):
        """Raw-pointer form of sweep (host pointers, e.g. pinned buffers)."""
        key = (v_ptr, psi_ptr, acc_ptr)
        args = self._ptr_args.get(key)
        if args is None:  # ctypes casts cost microseconds each: keep them for buffers that come back every sweep
            if len(self._ptr_args) > 64:
                self._ptr_args.clear()
            args = self._ptr_args[key] = tuple(C.cast(q, C.POINTER(C.c_double)) for q in key)
        rc = self._lib.cfmm_sweep(self._ctx, args[0], args[1], args[2], 1 if materialize else 0)
        if rc != 0:
            self._chk(rc)

    def sweep_device(self, d_v_ptr: int, d_psi_acc_ptr: int, materialize: bool = False,
                     stream_ptr: int = 0):
        self._chk(self._lib.cfmm_sweep_device(self._ctx, d_v_ptr, d_psi_acc_ptr,
                                              1 if materialize else 0, stream_ptr or None))

    def sweep_device_view(self, d_v_ptr: int, materialize: bool = False, stream_ptr: int = 0) -> int:
        """Zero-copy device sweep: returns the device address of [psi; acc]
        (valid until the next sweep on this context)."""
        out = C.c_void_p()
        self._chk(self._lib.cfmm_sweep_device_view(self._ctx, d_v_ptr, 1 if materialize else 0,
                                                   stream_ptr or None, C.byref(out)))
        return int(out.value)

    def last_sweep_ms(self) -> float:
        ms = C.c_float(0.0)
        self._chk(self._lib.cfmm_last_sweep_ms(self._ctx, C.byref(ms)))
        return float(ms.value)

    @property
    def launch_count(self) -> int:
        return int(self._lib.cfmm_launch_count(self._ctx))

    def profile_read(self, pool_type: int):
        """(total_ms, launches) of the event-timed kernels of one pool type."""
        ms, cnt = C.c_double(0.0), C.c_int64(0)
        self._chk(self._lib.cfmm_profile_read(self._ctx, int(pool_type), C.byref(ms), C.byref(cnt)))
        return float(ms.value), int(cnt.value)

    def profile_times(self, pool_type: int):
        """Per-launch durations (ms, launch order) of the event-timed kernels of one pool type."""
        cnt = C.c_int64(0)
        self._chk(self._lib.cfmm_profile_read_times(self._ctx, int(pool_type), None, 0, C.byref(cnt)))
        out = np.zeros(int(cnt.value), dtype=np.float32)
        if len(out):
            self._chk(self._lib.cfmm_profile_read_times(self._ctx, int(pool_type),
                                                        out.ctypes.data_as(C.POINTER(C.c_float)),
                                                        len(out), C.byref(cnt)))
        return out

    def profile_reset(self):
        self._chk(self._lib.cfmm_profile_reset(self._ctx))

    def trades(self):
        m = self.num_pools
        D = np.zeros((m, 2))
        L = np.zeros((m, 2))
        self._chk(self._lib.cfmm_get_trades(self._ctx, _dp(D), _dp(L)))
        return D, L

    def solve(self, lower, lin=None, upper=None, v0=None, pgtol=1e-5, factr=1e1, maxfun=15_000, maxiter=15_000):
        """cfmm_solve: minimise linᵀν + Σ arb_i(ν) over the box on the device.  Returns (ν, info dict);
        the trades at ν are materialised (trades())."""
        n = self.n_tokens
        lower = np.ascontiguousarray(lower, dtype=np.float64)
        arrs = [lower]
        def opt(a):
            if a is None:
                return None
            a = np.ascontiguousarray(a, dtype=np.float64)
            if a.shape != (n,):
                raise ValueError(f"vector arguments must have length {n}")
            arrs.append(a)
            return _dp(a)
        if lower.shape != (n,):
            raise ValueError(f"lower must have length {n}")
        opts = _lib.SolveOpts(int(maxiter), int(maxfun), float(pgtol), float(factr))
        info = _lib.SolveInfo()
        out = np.empty(n)
        self._chk(self._lib.cfmm_solve(self._ctx, opt(lin), _dp(lower), opt(upper), opt(v0), C.byref(opts),
                                       _dp(out), C.byref(info)))
        return out, {k: getattr(info, k) for k, _ in _lib.SolveInfo._fields_}

    def apply_trades(self):
        """Apply the trades of the last materialising sweep on the device: R <- R + γΔ − Λ for the
        two-coin pools, UniV3 pools move to the price their walk traded them to (univ3_moved_price)."""
        self._chk(self._lib.cfmm_apply_trades(self._ctx))

    def update_reserves(self, pool_type: int, first: int, R):
        R = np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 2)
        self._chk(self._lib.cfmm_update_reserves(self._ctx, int(pool_type), int(first), len(R), _dp(R)))

    def update_univ3(self, first: int, current_price=None, liquidity=None, count: int = None):
        """cfmm_update_univ3: new current prices and/or tick liquidities of the UniV3 pools
        [first, first + count) (UniV3 insertion order).  current_price: [count]; liquidity: the
        concatenated ticks of the same pools in ingest CSR order.  count defaults to
        len(current_price); a liquidity-only push must give it."""
        first = int(first)
        cp = None if current_price is None else np.ascontiguousarray(current_price, dtype=np.float64).reshape(-1)
        lq = None if liquidity is None else np.ascontiguousarray(liquidity, dtype=np.float64).reshape(-1)
        if count is None:
            if cp is None:
                raise ValueError("update_univ3: count is required when no prices are given")
            count = len(cp)
        count = int(count)
        if cp is not None and len(cp) != count:
            raise ValueError(f"update_univ3: {len(cp)} prices for {count} pools")
        if lq is not None:
            nt = self._univ3_ticks[first:first + count] if 0 <= first <= len(self._univ3_ticks) else []
            if len(nt) == count and len(lq) != int(np.sum(nt)):
                raise ValueError(f"update_univ3: {len(lq)} liquidities for {int(np.sum(nt))} ticks")
        self._chk(self._lib.cfmm_update_univ3(self._ctx, first, count, None if cp is None else _dp(cp),
                                              None if lq is None else _dp(lq)))

    # -- changing the pool set after finalize (include/cfmm_b200.h) ---------------
    def append_product(self, R, gamma, Ai):
        """cfmm_append_product: ProductTwoCoin pools added after finalize (next insertion indices)."""
        self._product(self._lib.cfmm_append_product, R, gamma, Ai)

    def append_geomean(self, R, gamma, Ai, w):
        self._geomean(self._lib.cfmm_append_geomean, R, gamma, Ai, w)

    def append_univ3(self, current_price, gamma, Ai, tick_off, lower_ticks, liquidity):
        self._univ3(self._lib.cfmm_append_univ3, current_price, gamma, Ai, tick_off, lower_ticks, liquidity)

    def set_active(self, pool_type: int, first: int, active):
        """cfmm_set_active: retire (False) or restore (True) the pools [first, first + len(active))
        of one type, counted in that type's insertion order."""
        a = np.ascontiguousarray(np.asarray(active).reshape(-1) != 0, dtype=np.uint8)
        self._chk(self._lib.cfmm_set_active(self._ctx, int(pool_type), int(first), len(a),
                                            a.ctypes.data_as(C.POINTER(C.c_uint8))))

    def pool_state(self, pool_type: int, first: int = 0, count: int = None):
        """cfmm_get_pool_state: (state, active) of the pools [first, first + count) of one type.
        state: reserves (count, 2) for the two-coin types, current prices (count,) for UniV3;
        active: bool (count,).  count defaults to the rest of the type's pools."""
        if count is None:
            info = self.pool_set_info(pool_type)
            count = info["main"] + info["tail"] - int(first)
        count = int(count)
        width = 1 if pool_type == _lib.POOL_UNIV3 else 2
        state = np.zeros(max(count, 0) * width)
        active = np.zeros(max(count, 0), dtype=np.uint8)
        self._chk(self._lib.cfmm_get_pool_state(self._ctx, int(pool_type), int(first), count, _dp(state),
                                                active.ctypes.data_as(C.POINTER(C.c_uint8))))
        return (state if width == 1 else state.reshape(-1, 2)), active.astype(bool)

    def compact(self):
        """cfmm_compact: fold the appended pools into the main layout (finalize's layout path)."""
        self._chk(self._lib.cfmm_compact(self._ctx))

    # -- swaps (include/cfmm_b200.h, cfmm_quote_swaps / cfmm_execute_swaps) ---------------
    @staticmethod
    def _swap_args(pools, tender):
        pools = np.ascontiguousarray(pools, dtype=np.int64).reshape(-1)
        tender = np.ascontiguousarray(tender, dtype=np.float64)
        if tender.ndim != 2 or tender.shape[1] != 2 or len(tender) != len(pools):
            raise ValueError(f"tender must have shape ({len(pools)}, 2), one row per pool index")
        return pools, tender

    def quote_swaps(self, pool_type: int, pools, tender):
        """cfmm_quote_swaps: what each row (pools[j], tender[j]) would receive, every row priced on
        the current state on its own; no state changes.  pools: indices in the type's insertion
        order; tender: (q, 2) in each pool's token order.  Returns received (q, 2)."""
        pools, tender = self._swap_args(pools, tender)
        out = np.zeros((len(pools), 2))
        self._chk(self._lib.cfmm_quote_swaps(self._ctx, int(pool_type), len(pools), _ip(pools), _dp(tender),
                                             _dp(out)))
        return out

    def execute_swaps(self, pool_type: int, pools, tender):
        """cfmm_execute_swaps: apply the rows in batch order (a row sees every earlier row on the same
        pool) and return what each row received, (q, 2)."""
        pools, tender = self._swap_args(pools, tender)
        out = np.zeros((len(pools), 2))
        self._chk(self._lib.cfmm_execute_swaps(self._ctx, int(pool_type), len(pools), _ip(pools), _dp(tender),
                                               _dp(out)))
        return out

    def quote_swaps_exact_out(self, pool_type: int, pools, want):
        """cfmm_quote_swaps_exact_out: the tender x* each row needs to receive want[j] ((0, y):
        receive token 2 for token 1; (y, 0) the reverse), every row on the current state on its own;
        no state changes.  Returns tender (q, 2); +inf where y cannot be reached."""
        pools, want = self._swap_args(pools, want)
        out = np.zeros((len(pools), 2))
        self._chk(self._lib.cfmm_quote_swaps_exact_out(self._ctx, int(pool_type), len(pools), _ip(pools),
                                                       _dp(want), _dp(out)))
        return out

    def execute_swap_orders(self, pool_type: int, pools, kind, amount, limit=None):
        """cfmm_execute_swap_orders: rows of kind 0 (exact-in: amount is the tender, limit the
        minimum received) or 1 (exact-out: amount the wanted output, limit the maximum tender), in
        batch order; a row whose limit fails reverts.  limit=None: no limits.  Returns
        (paid (q, 2), received (q, 2), status (q,) uint8; 0 filled, 1 limit, 2 unreachable,
        3 retired)."""
        pools, amount = self._swap_args(pools, amount)
        kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
        if len(kind) != len(pools):
            raise ValueError(f"kind must have {len(pools)} entries, one per row")
        if limit is not None:
            limit = np.ascontiguousarray(limit, dtype=np.float64).reshape(-1)
            if len(limit) != len(pools):
                raise ValueError(f"limit must have {len(pools)} entries, one per row")
        paid, received = np.zeros((len(pools), 2)), np.zeros((len(pools), 2))
        status = np.zeros(len(pools), dtype=np.uint8)
        u8 = C.POINTER(C.c_uint8)
        self._chk(self._lib.cfmm_execute_swap_orders(
            self._ctx, int(pool_type), len(pools), _ip(pools), kind.ctypes.data_as(u8), _dp(amount),
            None if limit is None else _dp(limit), _dp(paid), _dp(received), status.ctypes.data_as(u8)))
        return paid, received, status

    # -- multi-hop paths (include/cfmm_b200.h, cfmm_quote_paths / cfmm_execute_paths) ------------
    @staticmethod
    def _path_args(hop_off, hop_type, hop_pool, token_in, kind, amount):
        hop_off = np.ascontiguousarray(hop_off, dtype=np.int64).reshape(-1)
        hop_type = np.ascontiguousarray(hop_type, dtype=np.int32).reshape(-1)
        hop_pool = np.ascontiguousarray(hop_pool, dtype=np.int64).reshape(-1)
        token_in = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
        kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
        amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
        q = len(hop_off) - 1
        if q < 0 or not (len(token_in) == len(kind) == len(amount) == q):
            raise ValueError("paths: hop_off needs q + 1 entries and token_in, kind, amount q each")
        H = int(hop_off[-1])
        if not (len(hop_type) == len(hop_pool) == H):
            raise ValueError(f"paths: hop_type and hop_pool need hop_off[-1] = {H} entries")
        return q, H, hop_off, hop_type, hop_pool, token_in, kind, amount

    def quote_paths(self, hop_off, hop_type, hop_pool, token_in, kind, amount):
        """cfmm_quote_paths: path j is the hops hop_off[j] .. hop_off[j+1] (pool hop_pool[h] of type
        hop_type[h]), starting with token token_in[j] (1-based); kind 0 tenders amount[j] to the first
        hop, kind 1 wants amount[j] out of the last.  Every path on the current state on its own; no
        state changes.  Returns (hop_tender [H], hop_received [H], status [q] uint8)."""
        q, H, off, typ, pool, tok, kind, amount = self._path_args(hop_off, hop_type, hop_pool, token_in, kind, amount)
        tender, received, status = np.zeros(H), np.zeros(H), np.zeros(q, dtype=np.uint8)
        u8, i32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int)
        self._chk(self._lib.cfmm_quote_paths(self._ctx, q, _ip(off), typ.ctypes.data_as(i32), _ip(pool), _ip(tok),
                                             kind.ctypes.data_as(u8), _dp(amount), _dp(tender), _dp(received),
                                             status.ctypes.data_as(u8)))
        return tender, received, status

    def execute_paths(self, hop_off, hop_type, hop_pool, token_in, kind, amount, limit=None):
        """cfmm_execute_paths: the paths of quote_paths in batch order, each with its limit (kind 0:
        the minimum final output; kind 1: the maximum first tender; None: no limits).  A path whose
        limit fails reverts every hop, and later paths see the state without it.  Returns
        (hop_tender [H], hop_received [H], status [q] uint8)."""
        q, H, off, typ, pool, tok, kind, amount = self._path_args(hop_off, hop_type, hop_pool, token_in, kind, amount)
        if limit is not None:
            limit = np.ascontiguousarray(limit, dtype=np.float64).reshape(-1)
            if len(limit) != q:
                raise ValueError(f"limit must have {q} entries, one per path")
        tender, received, status = np.zeros(H), np.zeros(H), np.zeros(q, dtype=np.uint8)
        u8, i32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int)
        self._chk(self._lib.cfmm_execute_paths(self._ctx, q, _ip(off), typ.ctypes.data_as(i32), _ip(pool), _ip(tok),
                                               kind.ctypes.data_as(u8), _dp(amount),
                                               None if limit is None else _dp(limit), _dp(tender), _dp(received),
                                               status.ctypes.data_as(u8)))
        return tender, received, status

    # -- orders split across the pools of their pair (include/cfmm_b200.h, cfmm_pair_pools /
    #    cfmm_quote_split_orders / cfmm_execute_split_orders) ------------------------------------
    def pair_pools(self, token_a, token_b):
        """cfmm_pair_pools: the pools holding each unordered pair {token_a[j], token_b[j]} (1-based),
        in global insertion order.  Returns (off [q + 1], type [L], index [L] in the type's insertion
        order, active [L] bool); row j's pools are off[j] .. off[j + 1]."""
        a = np.ascontiguousarray(token_a, dtype=np.int64).reshape(-1)
        b = np.ascontiguousarray(token_b, dtype=np.int64).reshape(-1)
        if len(a) != len(b):
            raise ValueError("pair_pools: token_a and token_b need one entry per row")
        count = np.zeros(len(a), dtype=np.int64)
        self._chk(self._lib.cfmm_pair_pools(self._ctx, len(a), _ip(a), _ip(b), _ip(count), 0, None, None, None))
        off = np.concatenate([[0], np.cumsum(count)]).astype(np.int64)
        L = int(off[-1])
        typ, idx, act = np.zeros(L, dtype=np.int32), np.zeros(L, dtype=np.int64), np.zeros(L, dtype=np.uint8)
        if L:
            self._chk(self._lib.cfmm_pair_pools(self._ctx, len(a), _ip(a), _ip(b), _ip(count), L,
                                                typ.ctypes.data_as(C.POINTER(C.c_int)), _ip(idx),
                                                act.ctypes.data_as(C.POINTER(C.c_uint8))))
        return off, typ, idx, act.astype(bool)

    def _split(self, execute, token_in, token_out, kind, amount, limit, legs):
        tin = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
        amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
        q = len(tin)
        if not (len(tout) == len(kind) == len(amount) == q):
            raise ValueError("split orders: token_in, token_out, kind and amount need one entry per row")
        if limit is not None:
            limit = np.ascontiguousarray(limit, dtype=np.float64).reshape(-1)
            if len(limit) != q:
                raise ValueError(f"limit must have {q} entries, one per row")
        paid, received, price = np.zeros(q), np.zeros(q), np.zeros(q)
        status = np.zeros(q, dtype=np.uint8)
        off = ld = ll = None
        if legs:
            off = self.pair_pools(tin, tout)[0] if q else np.zeros(1, dtype=np.int64)
            ld, ll = np.zeros((int(off[-1]), 2)), np.zeros((int(off[-1]), 2))
        u8 = C.POINTER(C.c_uint8)
        args = [self._ctx, q, _ip(tin), _ip(tout), kind.ctypes.data_as(u8), _dp(amount)]
        if execute:
            args.append(None if limit is None else _dp(limit))
        args += [_dp(paid), _dp(received), _dp(price), status.ctypes.data_as(u8),
                 _dp(ld) if legs else None, _dp(ll) if legs else None]
        fn = self._lib.cfmm_execute_split_orders if execute else self._lib.cfmm_quote_split_orders
        self._chk(fn(*args))
        out = (paid, received, price, status)
        return out + ((off, ld, ll),) if legs else out

    def quote_split_orders(self, token_in, token_out, kind, amount, legs: bool = False):
        """cfmm_quote_split_orders: row j sells token_in[j] for token_out[j] (1-based) over every pool
        of the pair, split where the pools' marginal prices meet; kind 0 tenders amount[j], kind 1
        wants amount[j].  Every row on the current state on its own; no state changes.  Returns
        (paid [q], received [q], price [q] = s*, status [q] uint8) and, with legs=True, also
        (off [q + 1], leg_delta [L, 2], leg_lambda [L, 2]) in pair_pools order."""
        return self._split(False, token_in, token_out, kind, amount, None, legs)

    def execute_split_orders(self, token_in, token_out, kind, amount, limit=None, legs: bool = False):
        """cfmm_execute_split_orders: the rows of quote_split_orders in batch order, each on the state
        the earlier filled rows left, with optional limits (kind 0: minimum received; kind 1: maximum
        paid); a row whose limit fails reverts.  Returns what quote_split_orders returns."""
        return self._split(True, token_in, token_out, kind, amount, limit, legs)

    # -- orders routed over their pair and two-hop routes through hubs (include/cfmm_b200.h,
    #    cfmm_quote_routed_orders / cfmm_execute_routed_orders) -----------------------------------
    @staticmethod
    def route_pairs(token_in, token_out, hub_off, hubs):
        """The pair lists of routed rows, as cfmm_pair_pools rows: per row (j, i), then (j, h), (h, i)
        for each of its hubs.  Returns (token_a, token_b, first list of each row [q + 1])."""
        a, b, first = [], [], [0]
        for r in range(len(token_in)):
            j, i = int(token_in[r]), int(token_out[r])
            a.append(j)
            b.append(i)
            for h in hubs[int(hub_off[r]):int(hub_off[r + 1])]:
                a += [j, int(h)]
                b += [int(h), i]
            first.append(len(a))
        return np.array(a, dtype=np.int64), np.array(b, dtype=np.int64), np.array(first, dtype=np.int64)

    def _routed(self, execute, token_in, token_out, kind, amount, hub_off, hubs, limit, legs):
        tin = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
        amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
        hub_off = np.ascontiguousarray(hub_off, dtype=np.int64).reshape(-1)
        hubs = np.ascontiguousarray(hubs, dtype=np.int64).reshape(-1)
        q = len(tin)
        if not (len(tout) == len(kind) == len(amount) == q) or len(hub_off) != q + 1:
            raise ValueError("routed orders: token_in, token_out, kind and amount need one entry per row, "
                             "hub_off q + 1")
        if limit is not None:
            limit = np.ascontiguousarray(limit, dtype=np.float64).reshape(-1)
            if len(limit) != q:
                raise ValueError(f"limit must have {q} entries, one per row")
        nh = int(hub_off[-1]) if q else 0
        if q and (hub_off[0] != 0 or np.any(np.diff(hub_off) < 0) or len(hubs) != nh):
            raise ValueError("routed orders: hub_off must rise from 0 to len(hubs)")
        paid, received, price = np.zeros(q), np.zeros(q), np.zeros(q)
        status = np.zeros(q, dtype=np.uint8)
        hp, hs = np.zeros(nh), np.zeros(nh)
        off = ld = ll = None
        if legs:
            off = np.zeros(1, dtype=np.int64)
            if q:
                a, b, first = self.route_pairs(tin, tout, hub_off, hubs)
                off = self.pair_pools(a, b)[0][first]
            ld, ll = np.zeros((int(off[-1]), 2)), np.zeros((int(off[-1]), 2))
        u8 = C.POINTER(C.c_uint8)
        args = [self._ctx, q, _ip(tin), _ip(tout), kind.ctypes.data_as(u8), _dp(amount)]
        if execute:
            args.append(None if limit is None else _dp(limit))
        args += [_ip(hub_off) if q else None, _ip(hubs) if nh else None, _dp(paid), _dp(received), _dp(price),
                 status.ctypes.data_as(u8), _dp(hp) if nh else None, _dp(hs) if nh else None,
                 _dp(ld) if legs else None, _dp(ll) if legs else None]
        fn = self._lib.cfmm_execute_routed_orders if execute else self._lib.cfmm_quote_routed_orders
        self._chk(fn(*args))
        out = (paid, received, price, status, hp, hs)
        return out + ((off, ld, ll),) if legs else out

    def quote_routed_orders(self, token_in, token_out, kind, amount, hub_off, hubs, legs: bool = False):
        """cfmm_quote_routed_orders: row j sells token_in[j] for token_out[j] (1-based) over the pools of
        the pair and, for each hub h of hubs[hub_off[j] .. hub_off[j+1]] (at most ROUTE_MAX_HUBS), the
        pools of (token_in, h) and (h, token_out), split optimally; kind 0 tenders amount[j], kind 1
        wants amount[j].  Every row on the current state on its own; no state changes.  Returns (paid
        [q], received [q], price [q] = s*, status [q] uint8, hub_price [Σ] = t_h*, hub_surplus [Σ]) and,
        with legs=True, also (off [q + 1], leg_delta [L, 2], leg_lambda [L, 2]), each row's legs in the
        pair_pools order of route_pairs."""
        return self._routed(False, token_in, token_out, kind, amount, hub_off, hubs, None, legs)

    def execute_routed_orders(self, token_in, token_out, kind, amount, hub_off, hubs, limit=None,
                              legs: bool = False):
        """cfmm_execute_routed_orders: the rows of quote_routed_orders in batch order, each on the state
        the earlier filled rows left, with optional limits (kind 0: minimum received; kind 1: maximum
        paid); a row whose limit fails reverts.  Returns what quote_routed_orders returns."""
        return self._routed(True, token_in, token_out, kind, amount, hub_off, hubs, limit, legs)

    # -- arbitrage cycles through base tokens (include/cfmm_b200.h, cfmm_quote_arbitrage /
    #    cfmm_execute_arbitrage / cfmm_scan_arbitrage) -------------------------------------------
    def _arbitrage(self, execute, base, other, hub_off, hubs, min_profit, legs):
        base = np.ascontiguousarray(base, dtype=np.int64).reshape(-1)
        other = np.ascontiguousarray(other, dtype=np.int64).reshape(-1)
        hub_off = np.ascontiguousarray(hub_off, dtype=np.int64).reshape(-1)
        hubs = np.ascontiguousarray(hubs, dtype=np.int64).reshape(-1)
        q = len(base)
        if len(other) != q or len(hub_off) != q + 1:
            raise ValueError("arbitrage rows: base and other need one entry per row, hub_off q + 1")
        if min_profit is not None:
            min_profit = np.ascontiguousarray(min_profit, dtype=np.float64).reshape(-1)
            if len(min_profit) != q:
                raise ValueError(f"min_profit must have {q} entries, one per row")
        nh = int(hub_off[-1]) if q else 0
        if q and (hub_off[0] != 0 or np.any(np.diff(hub_off) < 0) or len(hubs) != nh):
            raise ValueError("arbitrage rows: hub_off must rise from 0 to len(hubs)")
        profit, surplus, price = np.zeros(q), np.zeros(q), np.zeros(q)
        status = np.zeros(q, dtype=np.uint8)
        hp, hs = np.zeros(nh), np.zeros(nh)
        off = ld = ll = None
        if legs:
            off = np.zeros(1, dtype=np.int64)
            if q:
                a, b, first = self.route_pairs(other, base, hub_off, hubs)
                off = self.pair_pools(a, b)[0][first]
            ld, ll = np.zeros((int(off[-1]), 2)), np.zeros((int(off[-1]), 2))
        u8 = C.POINTER(C.c_uint8)
        args = [self._ctx, q, _ip(base), _ip(other)]
        if execute:
            args.append(None if min_profit is None else _dp(min_profit))
        args += [_ip(hub_off) if q else None, _ip(hubs) if nh else None, _dp(profit), _dp(surplus), _dp(price),
                 status.ctypes.data_as(u8), _dp(hp) if nh else None, _dp(hs) if nh else None,
                 _dp(ld) if legs else None, _dp(ll) if legs else None]
        fn = self._lib.cfmm_execute_arbitrage if execute else self._lib.cfmm_quote_arbitrage
        self._chk(fn(*args))
        out = (profit, surplus, price, status, hp, hs)
        return out + ((off, ld, ll),) if legs else out

    def quote_arbitrage(self, base, other, hub_off, hubs, legs: bool = False):
        """cfmm_quote_arbitrage: row j runs the cycles from base[j] (1-based) through other[j] and back,
        directly and through each hub of hubs[hub_off[j] .. hub_off[j+1]] (at most ROUTE_MAX_HUBS),
        sized optimally (route! with BasketLiquidation(base, 0) over the row's pools).  Every row on
        the current state on its own; no state changes.  Returns (profit [q] in the base token,
        surplus_in [q] of other, price [q] = s*, status [q] uint8, hub_price [Σ], hub_surplus [Σ]) and,
        with legs=True, also (off [q + 1], leg_delta [L, 2], leg_lambda [L, 2]) in the pair_pools order
        of route_pairs(other, base, hub_off, hubs)."""
        return self._arbitrage(False, base, other, hub_off, hubs, None, legs)

    def execute_arbitrage(self, base, other, hub_off, hubs, min_profit=None, legs: bool = False):
        """cfmm_execute_arbitrage: the rows of quote_arbitrage in batch order, each re-solved on the state
        the earlier filled rows left; a row whose profit is below min_profit[j] (None: 0) reverts.
        Returns what quote_arbitrage returns."""
        return self._arbitrage(True, base, other, hub_off, hubs, min_profit, legs)

    def scan_arbitrage(self, base, min_profit, max_hubs: int = _lib.ROUTE_MAX_HUBS, cap: int = None):
        """cfmm_scan_arbitrage: the pair cycles and triangles through the distinct base tokens `base`
        (1-based) that yield at least min_profit[b] (> 0, in base b's token) on the current state,
        with up to max_hubs hubs per row, ordered by (base index, profit descending, other
        ascending).  No state changes.  cap (None: every row found) bounds the rows returned.
        Returns (found, row_base [n], row_other [n], hub_off [n + 1], hubs [Σ], profit [n],
        price [n]) with n = min(found, cap); the rows go to execute_arbitrage as they are.  With
        cap=None the scan runs twice: once to count, once to fetch."""
        base = np.ascontiguousarray(base, dtype=np.int64).reshape(-1)
        min_profit = np.ascontiguousarray(np.broadcast_to(np.asarray(min_profit, dtype=np.float64), base.shape))
        found = np.zeros(1, dtype=np.int64)

        def call(c):
            rb, ro, hc = np.zeros(c, dtype=np.int64), np.zeros(c, dtype=np.int64), np.zeros(c, dtype=np.int64)
            hb, pr, px = np.zeros((c, _lib.ROUTE_MAX_HUBS), dtype=np.int64), np.zeros(c), np.zeros(c)
            self._chk(self._lib.cfmm_scan_arbitrage(self._ctx, len(base), _ip(base), _dp(min_profit), int(max_hubs), c,
                                                    _ip(found), _ip(rb), _ip(ro), _ip(hc), _ip(hb), _dp(pr), _dp(px)))
            return rb, ro, hc, hb, pr, px

        out = call(max(0, int(cap)) if cap is not None else 0)
        if cap is None and found[0] > 0:
            out = call(int(found[0]))
        n = min(int(found[0]), len(out[0]))
        rb, ro, hc, hb, pr, px = (x[:n] for x in out)
        hub_off = np.concatenate([[0], np.cumsum(hc)]).astype(np.int64)
        hubs = np.concatenate([hb[r, :hc[r]] for r in range(n)]).astype(np.int64) if n else np.zeros(0, np.int64)
        return int(found[0]), rb, ro, hub_off, hubs, pr, px

    # -- hub tokens chosen for order rows (include/cfmm_b200.h, cfmm_choose_order_hubs) ------------
    def choose_order_hubs(self, token_in, token_out, kind, amount, max_hubs: int = _lib.ROUTE_MAX_HUBS,
                          allowed=None):
        """cfmm_choose_order_hubs: for row j (sell token_in[j] for token_out[j], 1-based; kind 0
        tenders amount[j], kind 1 wants amount[j]) the common neighbours h of the two tokens (with
        allowed[h - 1] when a mask [n_tokens] is given), ranked by their best single two-hop route: the
        most received (kind 0) or the least paid (kind 1) through the best pool of each hop.  No state
        changes.  Returns (hub_off [q + 1], hubs [Σ] best first, score [Σ], n_eligible [q]); hub_off
        and hubs go to quote_routed_orders / execute_routed_orders as they are."""
        tin = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        kind = np.ascontiguousarray(kind, dtype=np.uint8).reshape(-1)
        amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
        q = len(tin)
        if not (len(tout) == len(kind) == len(amount) == q):
            raise ValueError("choose_order_hubs: token_in, token_out, kind and amount need one entry per row")
        u8 = C.POINTER(C.c_uint8)
        mask = None
        if allowed is not None:
            mask = np.ascontiguousarray(allowed, dtype=bool).reshape(-1).astype(np.uint8)
            if len(mask) != self.n_tokens:
                raise ValueError(f"choose_order_hubs: allowed must have {self.n_tokens} entries, one per token")
        cap = q * max(int(max_hubs), 0)
        hub_off, hubs = np.zeros(q + 1, dtype=np.int64), np.zeros(max(cap, 1), dtype=np.int64)
        score, n_elig = np.zeros(max(cap, 1)), np.zeros(q, dtype=np.int64)
        self._chk(self._lib.cfmm_choose_order_hubs(self._ctx, q, _ip(tin), _ip(tout), kind.ctypes.data_as(u8),
                                                   _dp(amount), int(max_hubs),
                                                   None if mask is None else mask.ctypes.data_as(u8), _ip(hub_off),
                                                   _ip(hubs), _dp(score), _ip(n_elig)))
        n = int(hub_off[-1])
        return hub_off, hubs[:n].copy(), score[:n].copy(), n_elig

    # -- best paths through allowed tokens (include/cfmm_b200.h, cfmm_find_order_paths) ----------
    def find_order_paths(self, token_in, token_out, kind, amount, max_hops: int, allowed):
        """cfmm_find_order_paths: for row j (sell token_in[j] for token_out[j], 1-based; kind 0
        tenders amount[j], kind 1 wants amount[j]) the best single path of at most max_hops (1..8)
        hops, one pool per hop, whose intermediate tokens t have allowed[t - 1] (a mask [n_tokens],
        at most 1024 such tokens per row besides the row's two).  No state changes.  Returns (hop_off
        [q + 1], hop_type [Σ], hop_pool [Σ], hop_token [Σ] delivered, hop_tender [Σ], hop_received
        [Σ], value [q], status [q] uint8); the first three go to quote_paths / execute_paths as they
        are.  Status 0 filled, 2 no path, 4 (PATH_REPEATS_POOL) the best walk uses a pool twice."""
        return _order_paths(self, token_in, token_out, kind, amount, max_hops, allowed, None)

    def find_order_paths_net(self, token_in, token_out, kind, amount, max_hops: int, allowed, hop_cost):
        """cfmm_find_order_paths_net: find_order_paths at the max_hops = L (1..max_hops) whose filled
        result is best net of hop_cost[j] per hop (row j's cost in the token it settles in: token_out
        kind 0, token_in kind 1; the larger L on a tie).  Returns find_order_paths' tuple and net [q]."""
        return _order_paths(self, token_in, token_out, kind, amount, max_hops, allowed, hop_cost)

    # -- token values against one root (include/cfmm_b200.h, cfmm_quote_token_values) -------------
    def quote_token_values(self, root, kind, amount, max_hops: int, allowed=None, requests=None):
        """cfmm_quote_token_values: for row r (root[r] 1-based; kind 0 spends amount[r] of the root,
        kind 1 receives amount[r] of it) the best walk of at most max_hops (1..8) hops between the root
        and every token, through tokens t with allowed[t - 1] (a mask [n_tokens]; None: every token).
        No state changes.  Returns (value [q, n_tokens], hops [q, n_tokens] uint8, status [q, n_tokens]
        uint8, frontier [q, max_hops]: the tokens changed per level); with requests = (rows [k] 0-based,
        tokens [k] 1-based) also (hop_off [k + 1], hop_type, hop_pool, hop_token, hop_tender,
        hop_received, req_status [k]), the walks as quote_paths / execute_paths take them (exact-in
        from the root, exact-out into it)."""
        return _token_values(self, root, kind, amount, max_hops, allowed, requests, None)

    def quote_token_values_net(self, root, kind, amount, max_hops: int, hop_cost, allowed=None, requests=None):
        """cfmm_quote_token_values_net: per (row, token) quote_token_values at the max_hops = L
        (1..max_hops) whose filled result is best net of hop_cost[t - 1] per hop (the cost of a hop in
        units of token t, [n_tokens]; the larger L on a tie).  Returns quote_token_values' tuple with
        net [q, n_tokens] after status; the requested walks are the selected levels'."""
        return _token_values(self, root, kind, amount, max_hops, allowed, requests, hop_cost)

    # -- orders over every pool among allowed tokens (include/cfmm_b200.h,
    #    cfmm_quote_subgraph_swap_orders / cfmm_execute_subgraph_swap_orders) ------------------------
    def _subgraph(self, execute, token_in, token_out, amount, allowed, limit, opts, kind=None):
        tin = np.ascontiguousarray(token_in, dtype=np.int64).reshape(-1)
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        amount = np.ascontiguousarray(amount, dtype=np.float64).reshape(-1)
        q = len(tin)
        if not (len(tout) == len(amount) == q):
            raise ValueError("subgraph orders: token_in, token_out and amount need one entry per row")
        own = [(int(a), int(b)) for a, b in zip(tin, tout)]
        mk, limit, po = _row_args(self.n_tokens, q, allowed, limit, opts, "subgraph orders", own,
                                  [_lib.SUBGRAPH_MAX_TOKENS] * q)
        kind = _row_kind(kind, q, limit, "subgraph orders")
        ti, to, am = _ip(tin), _ip(tout), _dp(amount)
        kd = None if kind is None else kind.ctypes.data_as(C.POINTER(C.c_uint8))
        lim = None if limit is None else _dp(limit)
        sfx = "_rows" if mk.rows else ""

        def call(size, out):
            if execute and not size:
                return getattr(self._lib, "cfmm_execute_subgraph_swap_orders" + sfx)(self._ctx, q, ti, to, kd, am, lim,
                                                                                     *mk.args, po, C.byref(out))
            return getattr(self._lib, "cfmm_quote_subgraph_swap_orders" + sfx)(self._ctx, q, ti, to, kd, am, *mk.args,
                                                                               po, C.byref(out))
        return self._order_solve(q, q, _lib.SubgraphOut, call)

    def _order_solve(self, q, n_paid, out_type, call):
        """The outputs of a subgraph or basket call: call(True, out) with tok_cap = leg_cap = 0 for the
        sizes (a row's token set and pool list do not depend on the reserves, so an execute's are the
        same), then call(False, out) with every output.  Returns them as a namespace."""
        u8, i32, i64, f64 = C.POINTER(C.c_uint8), C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_double)
        tok_off, leg_off = np.zeros(q + 1, dtype=np.int64), np.zeros(q + 1, dtype=np.int64)
        size = out_type()
        size.tok_off, size.leg_off = tok_off.ctypes.data_as(i64), leg_off.ctypes.data_as(i64)
        self._chk(call(True, size))
        NT, L = int(tok_off[-1]), int(leg_off[-1])
        paid, received, merit = np.zeros(max(n_paid, 1)), np.zeros(q), np.zeros(q)
        status = np.zeros(q, dtype=np.uint8)
        sst, iters, fev = (np.zeros(q, dtype=np.int32) for _ in range(3))
        token, nu, psi = np.zeros(max(NT, 1), dtype=np.int64), np.zeros(max(NT, 1)), np.zeros(max(NT, 1))
        ltype, lpool = np.zeros(max(L, 1), dtype=np.int32), np.zeros(max(L, 1), dtype=np.int64)
        ld, ll = np.zeros((max(L, 1), 2)), np.zeros((max(L, 1), 2))
        head = ((received.ctypes.data_as(f64),) if out_type is _lib.PriceArbOut else
                (paid.ctypes.data_as(f64), received.ctypes.data_as(f64)))  # price rows: the profit
        out = out_type(*head, status.ctypes.data_as(u8),
                       sst.ctypes.data_as(i32), iters.ctypes.data_as(i32), fev.ctypes.data_as(i32),
                       merit.ctypes.data_as(f64), tok_off.ctypes.data_as(i64), NT, token.ctypes.data_as(i64),
                       nu.ctypes.data_as(f64), psi.ctypes.data_as(f64), leg_off.ctypes.data_as(i64), L,
                       ltype.ctypes.data_as(i32), lpool.ctypes.data_as(i64), ld.ctypes.data_as(f64),
                       ll.ctypes.data_as(f64))
        self._chk(call(False, out))
        return SimpleNamespace(paid=paid[:n_paid], received=received, status=status, solver_status=sst,
                               iterations=iters, fun_evals=fev, merit=merit, tok_off=tok_off, token=token[:NT],
                               nu=nu[:NT], psi=psi[:NT], leg_off=leg_off, leg_type=ltype[:L], leg_pool=lpool[:L],
                               leg_delta=ld[:L], leg_lambda=ll[:L])

    def quote_subgraph_orders(self, token_in, token_out, amount, allowed, opts=None, kind=None):
        """cfmm_quote_subgraph_swap_orders: row j sells amount[j] of token_in[j] for token_out[j]
        (1-based; kind 0, exact-in) or buys amount[j] of token_out[j] paying in token_in[j] (kind 1,
        exact-out) over every pool among the two and the tokens t with allowed[t - 1] (at most 256
        besides the row's two), split optimally: route! over the row's pools, solved per row on the
        device.  kind: None (every row exact-in), a scalar, or one entry per row.  opts: dict of
        max_iter, max_fun, rtol, factr (None: the defaults).  No state changes.  Returns a namespace:
        paid, received, status (uint8), solver_status, iterations, fun_evals, merit [q]; tok_off
        [q + 1], token, nu, psi [Σ]; leg_off [q + 1], leg_type, leg_pool [L], leg_delta, leg_lambda
        [L, 2].  allowed may instead be one list of 1-based tokens per row (choose_hubs' output as it is):
        each row then runs over its own list, as the call with that list as its mask (the *_rows calls)."""
        return self._subgraph(False, token_in, token_out, amount, allowed, None, opts, kind)

    def execute_subgraph_orders(self, token_in, token_out, amount, allowed, limit=None, opts=None, kind=None):
        """cfmm_execute_subgraph_swap_orders: the rows of quote_subgraph_orders in batch order, each
        re-solved on the state the earlier filled rows left; limit[j] (None: none) is the minimum
        received of an exact-in row and the maximum paid of an exact-out row (+inf allowed), and a row
        that misses it reverts.  Returns what quote_subgraph_orders returns."""
        return self._subgraph(True, token_in, token_out, amount, allowed, limit, opts, kind)

    # -- token baskets over every pool among allowed tokens (include/cfmm_b200.h,
    #    cfmm_quote_basket_(swap_)orders / cfmm_execute_basket_(swap_)orders) -------------------------
    def _basket(self, execute, token_out, basket_off, basket_token, basket_amount, allowed, limit, opts, kind=None):
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        boff = np.ascontiguousarray(basket_off, dtype=np.int64).reshape(-1)
        btok = np.ascontiguousarray(basket_token, dtype=np.int64).reshape(-1)
        bamt = np.ascontiguousarray(basket_amount, dtype=np.float64).reshape(-1)
        q = len(tout)
        if len(boff) != q + 1:
            raise ValueError(f"basket orders: basket_off must have {q + 1} entries, one per row plus one")
        NE = int(boff[-1])
        if not (len(btok) == len(bamt) == NE):
            raise ValueError(f"basket orders: basket_token and basket_amount need basket_off[-1] = {NE} entries")
        own, room = _basket_room(tout, boff, btok)
        mk, limit, po = _row_args(self.n_tokens, q, allowed, limit, opts, "basket orders", own, room)
        kind = _entry_kind(kind, boff, limit, "basket orders")
        to, bo, bt, ba = _ip(tout), _ip(boff), _ip(btok), _dp(bamt)
        lim = None if limit is None else _dp(limit)

        def call(size, out):
            if mk.rows:  # every row kind through the swap calls' _rows form
                kd = None if kind is None else kind.ctypes.data_as(C.POINTER(C.c_uint8))
                if execute and not size:
                    return self._lib.cfmm_execute_basket_swap_orders_rows(self._ctx, q, to, bo, bt, kd, ba, lim,
                                                                          *mk.args, po, C.byref(out))
                return self._lib.cfmm_quote_basket_swap_orders_rows(self._ctx, q, to, bo, bt, kd, ba, *mk.args, po,
                                                                    C.byref(out))
            u8m = mk.args[0]
            if kind is not None:
                kd = kind.ctypes.data_as(C.POINTER(C.c_uint8))
                if execute and not size:
                    return self._lib.cfmm_execute_basket_swap_orders(self._ctx, q, to, bo, bt, kd, ba, lim, u8m, po,
                                                                     C.byref(out))
                return self._lib.cfmm_quote_basket_swap_orders(self._ctx, q, to, bo, bt, kd, ba, u8m, po,
                                                               C.byref(out))
            if execute and not size:
                return self._lib.cfmm_execute_basket_orders(self._ctx, q, to, bo, bt, ba, lim, u8m, po, C.byref(out))
            return self._lib.cfmm_quote_basket_orders(self._ctx, q, to, bo, bt, ba, u8m, po, C.byref(out))
        out = self._order_solve(q, NE, _lib.BasketOut, call)
        out.basket_off = boff
        return out

    def quote_basket_orders(self, token_out, basket_off, basket_token, basket_amount, allowed, opts=None,
                            kind=None):
        """cfmm_quote_basket_orders: row r sells basket_amount[k] of basket_token[k] for k in
        basket_off[r] .. basket_off[r + 1] - 1 (1 to 16 distinct tokens, 1-based, none token_out[r])
        for token_out[r] over every pool among them and the tokens t with allowed[t - 1], split
        optimally: route! with BasketLiquidation over the row's pools, solved per row on the device.
        kind (cfmm_quote_basket_swap_orders): None (every entry sold), a scalar, or one entry per basket
        entry, 0 sold or 1 bought (buy basket_amount[k] of basket_token[k]); a row with a bought entry
        settles in token_out[r], and its received may be negative.  opts as quote_subgraph_orders.  No
        state changes.  Returns quote_subgraph_orders' namespace, with paid per basket entry (−Ψ: a
        bought entry reads at most −amount) and basket_off added.  allowed may instead be one list of
        1-based tokens per row (choose_hubs' output as it is): each row then runs over its own list, as the
        call with that list as its mask (the *_rows calls)."""
        return self._basket(False, token_out, basket_off, basket_token, basket_amount, allowed, None, opts, kind)

    def execute_basket_orders(self, token_out, basket_off, basket_token, basket_amount, allowed, limit=None,
                              opts=None, kind=None):
        """cfmm_execute_basket_(swap_)orders: the rows of quote_basket_orders in batch order, each
        re-solved on the state the earlier filled rows left; limit[r] (None: none) is the minimum
        received of token_out[r] (for a row with a bought entry it may be negative or -inf), and a row
        below it reverts.  Returns what quote_basket_orders returns."""
        return self._basket(True, token_out, basket_off, basket_token, basket_amount, allowed, limit, opts, kind)

    # -- limit orders over every pool among allowed tokens (include/cfmm_b200.h,
    #    cfmm_quote_limit_orders / cfmm_execute_limit_orders) ----------------------------------------------
    def _limit(self, execute, token_out, basket_off, basket_token, basket_amount, limit_price, allowed,
               min_received, opts):
        tout = np.ascontiguousarray(token_out, dtype=np.int64).reshape(-1)
        boff = np.ascontiguousarray(basket_off, dtype=np.int64).reshape(-1)
        btok = np.ascontiguousarray(basket_token, dtype=np.int64).reshape(-1)
        bamt = np.ascontiguousarray(basket_amount, dtype=np.float64).reshape(-1)
        lp = np.ascontiguousarray(limit_price, dtype=np.float64).reshape(-1)
        q = len(tout)
        if len(boff) != q + 1:
            raise ValueError(f"limit orders: basket_off must have {q + 1} entries, one per row plus one")
        NE = int(boff[-1])
        if not (len(btok) == len(bamt) == len(lp) == NE):
            raise ValueError(f"limit orders: basket_token, basket_amount and limit_price need basket_off[-1] = {NE} "
                             "entries")
        if not np.all(np.isfinite(lp) & (lp >= 0.0)):
            raise ValueError("limit orders: a limit price is negative, NaN or Inf")
        own, room = _basket_room(tout, boff, btok)
        mk, min_received, po = _row_args(self.n_tokens, q, allowed, min_received, opts, "limit orders", own, room)
        to, bo, bt, ba, lpp = _ip(tout), _ip(boff), _ip(btok), _dp(bamt), _dp(lp)
        lim = None if min_received is None else _dp(min_received)
        surplus = np.zeros(q)
        quote = getattr(self._lib, "cfmm_quote_limit_orders" + ("_rows" if mk.rows else ""))
        execute_ = getattr(self._lib, "cfmm_execute_limit_orders" + ("_rows" if mk.rows else ""))

        def call(size, out):
            if size:
                return quote(self._ctx, q, to, bo, bt, ba, lpp, *mk.args, po, C.byref(out))
            out.surplus = surplus.ctypes.data_as(C.POINTER(C.c_double))
            if execute:
                return execute_(self._ctx, q, to, bo, bt, ba, lpp, lim, *mk.args, po, C.byref(out))
            return quote(self._ctx, q, to, bo, bt, ba, lpp, *mk.args, po, C.byref(out))
        out = self._order_solve(q, NE, _lib.LimitOut, call)
        out.surplus = surplus
        out.basket_off = boff
        return out

    def quote_limit_orders(self, token_out, basket_off, basket_token, basket_amount, limit_price, allowed,
                           opts=None):
        """cfmm_quote_limit_orders: row r sells up to basket_amount[k] of basket_token[k] for k in
        basket_off[r] .. basket_off[r + 1] - 1 (1 to 16 distinct tokens, 1-based, none token_out[r]) for
        token_out[r], each for as long as the margin pays at least limit_price[k] of token_out[r] per unit
        (finite, >= 0), over every pool among them and the tokens t with allowed[t - 1]: a basket row
        with each entry's dual bound raised to its limit, solved per row on the device; rows fill
        partially.  opts as quote_subgraph_orders.  No state changes.  Returns quote_basket_orders'
        namespace, with surplus [q] (received - Σ limit·paid) added.  allowed may instead be one list of
        1-based tokens per row (choose_hubs' output as it is): each row then runs over its own list, as the
        call with that list as its mask (the *_rows calls)."""
        return self._limit(False, token_out, basket_off, basket_token, basket_amount, limit_price, allowed, None,
                           opts)

    def execute_limit_orders(self, token_out, basket_off, basket_token, basket_amount, limit_price, allowed,
                             min_received=None, opts=None):
        """cfmm_execute_limit_orders: the rows of quote_limit_orders in batch order, each re-solved on the
        state the earlier filled rows left; min_received[r] (None: none) is the minimum received of
        token_out[r], and a row below it reverts.  Returns what quote_limit_orders returns."""
        return self._limit(True, token_out, basket_off, basket_token, basket_amount, limit_price, allowed,
                           min_received, opts)

    # -- arbitrage against external prices over every pool among allowed tokens (include/cfmm_b200.h,
    #    cfmm_quote_price_arbitrage / cfmm_execute_price_arbitrage) --------------------------------------
    def _price_arb(self, execute, price, allowed, min_profit, opts):
        mk, _, po = _row_args(self.n_tokens, None, allowed, None, opts, "price arbitrage")
        u8m = mk.args[0]
        nA = int(np.count_nonzero(np.asarray(allowed, dtype=bool)))
        if nA > _lib.PRICE_ARB_MAX_TOKENS:
            raise ValueError(f"price arbitrage: {nA} allowed tokens, more than {_lib.PRICE_ARB_MAX_TOKENS}")
        price = np.ascontiguousarray(price, dtype=np.float64)
        if price.ndim != 2 or price.shape[1] != nA:
            raise ValueError(f"price arbitrage: price must be [q, {nA}], one column per allowed token")
        q = price.shape[0]
        if not np.all(np.isfinite(price) & (price >= 0.0)):
            raise ValueError("price arbitrage: a price is negative, NaN or Inf")
        if q and not np.all(np.any(price > 0.0, axis=1)):
            raise ValueError("price arbitrage: a row has no positive price")
        lim = None
        if min_profit is not None:
            min_profit = np.ascontiguousarray(np.broadcast_to(np.asarray(min_profit, dtype=np.float64), (q,)))
            if not np.all(np.isfinite(min_profit) & (min_profit >= 0.0)):
                raise ValueError("price arbitrage: a min_profit is negative, NaN or Inf")
            lim = _dp(min_profit)
        pr = _dp(price)

        def call(size, out):
            if execute and not size:
                return self._lib.cfmm_execute_price_arbitrage(self._ctx, q, pr, lim, u8m, po, C.byref(out))
            return self._lib.cfmm_quote_price_arbitrage(self._ctx, q, pr, u8m, po, C.byref(out))
        out = self._order_solve(q, 0, _lib.PriceArbOut, call)
        out.profit = out.received
        del out.paid, out.received
        return out

    def quote_price_arbitrage(self, price, allowed, opts=None):
        """cfmm_quote_price_arbitrage: row r values the tokens t with allowed[t - 1] (ascending, at most
        258) at price[r] (0: the token is not in the row, else finite and > 0) and trades over every pool
        among its priced tokens to maximise Σ price·Ψ with no token's net negative: route! with
        LinearNonnegative over the row's pools, solved per row on the device.  opts as
        quote_subgraph_orders.  No state changes.  Returns a namespace: profit, status (uint8),
        solver_status, iterations, fun_evals, merit [q]; tok_off [q + 1], token, nu, psi [Σ]; leg_off
        [q + 1], leg_type, leg_pool [L], leg_delta, leg_lambda [L, 2]."""
        return self._price_arb(False, price, allowed, None, opts)

    def execute_price_arbitrage(self, price, allowed, min_profit=None, opts=None):
        """cfmm_execute_price_arbitrage: the rows of quote_price_arbitrage in batch order, each re-solved
        on the state the earlier filled rows left; min_profit (None, a scalar or one per row; finite and
        >= 0) is the minimum profit, and a row below it reverts.  Returns what quote_price_arbitrage
        returns."""
        return self._price_arb(True, price, allowed, min_profit, opts)

    # -- arbitrage from inventory, one token list per row (include/cfmm_b200.h,
    #    cfmm_quote_price_arbitrage_rows / cfmm_execute_price_arbitrage_rows) ----------------------------
    def _price_arb_rows(self, execute, allow_off, allow_token, price, holding, min_profit, opts):
        what = "inventory arbitrage"
        off = np.ascontiguousarray(allow_off, dtype=np.int64).reshape(-1)
        tok = np.ascontiguousarray(allow_token, dtype=np.int64).reshape(-1)
        q = len(off) - 1
        if q < 0 or off[0] != 0 or np.any(np.diff(off) < 0) or off[-1] != len(tok):
            raise ValueError(f"{what}: allow_off must start at 0, not decrease and end at len(allow_token)")
        n = np.diff(off)
        if np.any((n < 1) | (n > _lib.PRICE_ARB_MAX_TOKENS)):
            raise ValueError(f"{what}: every row lists 1 to {_lib.PRICE_ARB_MAX_TOKENS} tokens")
        price = np.ascontiguousarray(price, dtype=np.float64).reshape(-1)
        if len(price) != len(tok):
            raise ValueError(f"{what}: price needs one entry per listed token ({len(tok)})")
        if not np.all(np.isfinite(price) & (price >= 0.0)):
            raise ValueError(f"{what}: a price is negative, NaN or Inf")
        if q and not np.all(np.maximum.reduceat(price, off[:-1]) > 0.0):
            raise ValueError(f"{what}: a row has no positive price")
        hp = None
        if holding is not None:
            holding = np.ascontiguousarray(holding, dtype=np.float64).reshape(-1)
            if len(holding) != len(tok):
                raise ValueError(f"{what}: holding needs one entry per listed token ({len(tok)})")
            if not np.all(np.isfinite(holding) & (holding >= 0.0)):
                raise ValueError(f"{what}: a holding is negative, NaN or Inf")
            hp = _dp(holding)
        lim = None
        if min_profit is not None:
            min_profit = np.ascontiguousarray(np.broadcast_to(np.asarray(min_profit, dtype=np.float64), (q,)))
            if not np.all(np.isfinite(min_profit) & (min_profit >= 0.0)):
                raise ValueError(f"{what}: a min_profit is negative, NaN or Inf")
            lim = _dp(min_profit)
        if opts is not None and not (np.isfinite(opts.get("atol", 0.0)) and opts.get("atol", 0.0) >= 0.0):
            raise ValueError(f"{what}: atol must be finite and >= 0")
        po, ao, at, pr = _price_arb_opts(opts), _ip(off), _ip(tok), _dp(price)

        def call(size, out):
            if execute and not size:
                return self._lib.cfmm_execute_price_arbitrage_rows(self._ctx, q, ao, at, pr, hp, lim, po, C.byref(out))
            return self._lib.cfmm_quote_price_arbitrage_rows(self._ctx, q, ao, at, pr, hp, po, C.byref(out))
        out = self._order_solve(q, 0, _lib.PriceArbOut, call)
        out.profit = out.received
        del out.paid, out.received
        return out

    def quote_price_arbitrage_rows(self, allow_off, allow_token, price, holding=None, opts=None):
        """cfmm_quote_price_arbitrage_rows: row r lists the tokens allow_token[allow_off[r] ..
        allow_off[r + 1]) (1-based, distinct, 1 to 258, any order), with price and holding aligned with
        allow_token (price finite and >= 0, a positive one per row; holding None: all 0, else finite and
        >= 0).  Each row trades over every pool among its tokens that have an active pool to another
        listed token, maximising Σ price·Ψ with Ψ + holding >= 0 (a price of 0 keeps the token as an
        intermediate), one dual solve per row on the device.  opts: dict of max_iter, max_fun, rtol,
        factr and atol (the absolute stop on max ν·|pg|, default 0).  No state changes.  Returns
        quote_price_arbitrage's namespace."""
        return self._price_arb_rows(False, allow_off, allow_token, price, holding, None, opts)

    def execute_price_arbitrage_rows(self, allow_off, allow_token, price, holding=None, min_profit=None,
                                     opts=None):
        """cfmm_execute_price_arbitrage_rows: the rows of quote_price_arbitrage_rows in batch order, each
        re-solved on the state the earlier filled rows left (rows on disjoint lists share a launch);
        min_profit (None, a scalar or one per row; finite and >= 0) reverts a row below it.  Returns
        what quote_price_arbitrage_rows returns."""
        return self._price_arb_rows(True, allow_off, allow_token, price, holding, min_profit, opts)

    # -- UniV3 liquidity changes (include/cfmm_b200.h, cfmm_modify_univ3_liquidity) ---------------
    def modify_univ3_liquidity(self, pools, lo, hi, dL):
        """cfmm_modify_univ3_liquidity: row j adds dL[j] (> 0 mints, < 0 burns) to the ticks of UniV3
        pool pools[j] (insertion order) on the price range (lo[j], hi[j]], inserting lo and hi into its
        ladder when they are not boundaries yet.  Rows apply in batch order; a row that would leave a
        tick below zero rejects the whole call and changes nothing."""
        pools = np.ascontiguousarray(pools, dtype=np.int64).reshape(-1)
        rng = np.ascontiguousarray(np.stack([np.asarray(lo, dtype=np.float64).reshape(-1),
                                             np.asarray(hi, dtype=np.float64).reshape(-1)], axis=1))
        dL = np.ascontiguousarray(dL, dtype=np.float64).reshape(-1)
        if not (len(pools) == len(rng) == len(dL)):
            raise ValueError("modify_univ3_liquidity: pools, lo, hi, dL must have one entry per row")
        self._chk(self._lib.cfmm_modify_univ3_liquidity(self._ctx, len(pools), _ip(pools), _dp(rng), _dp(dL)))
        if len(pools):
            first = int(pools.min())
            self.univ3_ticks(first, int(pools.max()) + 1 - first, ladders=False)

    def univ3_ticks(self, first: int = 0, count: int = None, ladders: bool = True):
        """cfmm_get_univ3_ticks: (tick_off [count + 1], lower_ticks, liquidity) of the UniV3 pools
        [first, first + count), the current ladders in CSR form (lower_ticks / liquidity are None
        with ladders=False).  count defaults to the rest of the UniV3 pools."""
        first = int(first)
        if count is None:
            info = self.pool_set_info(_lib.POOL_UNIV3)
            count = info["main"] + info["tail"] - first
        count = int(count)
        off = np.zeros(max(count, 0) + 1, dtype=np.int64)
        self._chk(self._lib.cfmm_get_univ3_ticks(self._ctx, first, count, _ip(off), None, None))
        lt = lq = None
        if ladders:
            lt, lq = np.zeros(int(off[-1])), np.zeros(int(off[-1]))
            self._chk(self._lib.cfmm_get_univ3_ticks(self._ctx, first, count, _ip(off), _dp(lt), _dp(lq)))
        if len(self._univ3_ticks) >= first + count:
            self._univ3_ticks[first:first + count] = np.diff(off)
        return off, lt, lq

    def pool_set_info(self, pool_type: int) -> dict:
        """Layout facts of one pool type (cfmm_debug_pool_set_info; read-only)."""
        info = np.zeros(8, dtype=np.int64)
        self._chk(self._lib.cfmm_debug_pool_set_info(self._ctx, int(pool_type), _ip(info)))
        keys = ("main", "tail", "padded", "tma", "fixed_point", "compact_stream", "fast_range", "retired")
        return {k: int(x) for k, x in zip(keys, info)}

    def compact_record(self, pool_type: int) -> int:
        """Pools per compact record the next gradient-only sweep of the main set streams: 192
        (18-byte pool records), 96 (20-byte pool records) or 0 (cfmm_debug_compact_record; read-only)."""
        out = np.zeros(1, dtype=np.int64)
        self._chk(self._lib.cfmm_debug_compact_record(self._ctx, int(pool_type), _ip(out)))
        return int(out[0])

    def l2_keep(self, pool_type: int) -> int:
        """L2 keep rule of the next gradient-only sweep of the main set: h > 0 = the first h records
        of every CTA's range stay in the L2 across sweeps, 0 = no L2 hints (cfmm_debug_l2_keep; read-only)."""
        out = np.zeros(1, dtype=np.int64)
        self._chk(self._lib.cfmm_debug_l2_keep(self._ctx, int(pool_type), _ip(out)))
        return int(out[0])

    # -- multi-GPU --------------------------------------------------------------
    def detach_group(self):
        self._chk(self._lib.cfmm_comm_detach(self._ctx))
        self.peer_attached = False

    def comm_check(self):
        """After sweep_device* calls: wait for them and raise CFMMError (CFMM_ERR_COMM) if an
        exchange gave up on a peer (cfmm_comm_check)."""
        self._chk(self._lib.cfmm_comm_check(self._ctx))

    def attach_group(self, group=None, barrier=True):
        """Join the NVLink peer exchange of a torch.distributed group (one
        process per GPU): export this rank's handle, all-gather the handles
        (torch.distributed is only the transport for 128 bytes per rank),
        attach.  After this, sweep() returns the sum over all ranks."""
        import torch
        import torch.distributed as dist

        world = dist.get_world_size(group)
        rank = dist.get_rank(group)
        if world == 1:
            return
        buf = (C.c_ubyte * _lib.COMM_HANDLE_BYTES)()
        self._chk(self._lib.cfmm_comm_export(self._ctx, buf))
        dev = torch.device("cuda", self.device) if dist.get_backend(group) == "nccl" else torch.device("cpu")
        mine = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device=dev)
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine, group=group)
        allh = bytes(torch.cat(gathered).cpu().numpy().tobytes())
        self._chk(self._lib.cfmm_comm_attach(self._ctx, world, rank, allh))
        self.peer_attached = True
        if barrier:
            dist.barrier(group)

    def close(self):
        if self._ctx:
            self._lib.cfmm_destroy(self._ctx)
            self._ctx = C.c_void_p()
            self._pin_nu = self._pin_out = None
            if self._pin:
                self._lib.cfmm_host_free(self._pin)
                self._pin = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def pack_hop_cost(hop_cost, n_tokens, settle, what):
    """A Router call's hop_cost as the _net calls take it: a scalar (every entry), or one cost per token
    ([n_tokens], e.g. Router.hop_costs), each >= 0 (inf allowed: no walk pays for itself).  settle:
    each row's settlement token (1-based), which picks a per-token cost for the row; None: the costs
    per token, as they are."""
    c = np.asarray(hop_cost, dtype=np.float64)
    size = n_tokens if settle is None else len(settle)
    if c.ndim == 0:
        c = np.full(size, float(c))
    else:
        c = c.reshape(-1)
        if len(c) != n_tokens:
            raise ValueError(f"{what}: hop_cost must be a scalar or have {n_tokens} entries, one per token")
        if settle is not None:
            c = c[np.asarray(settle, dtype=np.int64) - 1]
    if not np.all(c >= 0.0):
        raise ValueError(f"{what}: hop_cost must be >= 0 (inf allowed), not NaN or negative")
    return np.ascontiguousarray(c)


def _pack(cfmms):
    """Vector{CFMM} (AoS of Python objects) -> per-type SoA + the map from the
    library's global insertion order back to list positions."""
    idx = {0: [], 1: [], 2: []}
    for i, c in enumerate(cfmms):
        if isinstance(c, ProductTwoCoin):
            idx[0].append(i)
        elif isinstance(c, GeometricMeanTwoCoin):
            idx[1].append(i)
        elif isinstance(c, UniV3):
            idx[2].append(i)
        else:
            # the reference would hit a MethodError in find_arb! for these
            raise TypeError(f"no find_arb! method for {type(c).__name__}")
    return idx


class Router:
    """Router(objective, cfmms, n_tokens) (src/router.jl:4-36).

    Fields as in the reference: objective, cfmms, Δs, Λs, v.  Δs / Λs are
    (m, 2) arrays; Δs[i] / Λs[i] are the trade vectors of cfmms[i].  As in the
    reference (router.jl:39, loop bound length(r.Δs)), pools appended to
    r.cfmms after construction are ignored; add_cfmms adds pools to a built
    router, and set_active retires and restores pools (single GPU).

    Multi-GPU: with `group` (a torch.distributed process group, one process per
    GPU) every rank holds the full Python pool list but uploads only its
    contiguous shard; Ψ/acc are summed across ranks after each sweep and every
    rank runs the same L-BFGS-B iteration on the identical reduced vector.
    """

    def __init__(self, objective: Objective, cfmms=None, n_tokens: int = None, *,
                 device: int = 0, group=None, exchange: str = "peer", _pools_factory=None):
        if n_tokens is None and isinstance(cfmms, (int, np.integer)):
            cfmms, n_tokens = None, int(cfmms)  # Router(objective, n_tokens): empty pool list, router.jl:36
        if n_tokens is None:
            raise TypeError("n_tokens is required")
        self.objective = objective
        self.cfmms = list(cfmms) if cfmms is not None else []
        m = len(self.cfmms)
        self.Δs = np.zeros((m, 2))  # zerotrade(c), router.jl:23-26
        self.Λs = np.zeros((m, 2))
        self.v = np.zeros(int(n_tokens))
        self._group = group
        self._world, self._rank = 1, 0
        if group is not None:
            import torch.distributed as dist
            self._world, self._rank = dist.get_world_size(group), dist.get_rank(group)
        self._lo, self._hi = shard_range(m, self._world, self._rank)
        self._exchange = exchange
        factory = _pools_factory or DevicePools
        self._pools = factory(int(n_tokens), device)
        self._retired = np.zeros(m, dtype=bool)
        self._upload()
        if self._world > 1 and exchange == "peer":
            self._attach_with_agreement(group)
        self._psi = np.zeros(int(n_tokens))
        self._acc = 0.0

    def _attach_with_agreement(self, group):
        """Join the NVLink peer exchange, or -- if ANY rank cannot (no P2P / IPC) -- fall back to
        torch.distributed on every rank: a rank that raised alone would leave the others blocked in
        their first exchange."""
        import torch
        import torch.distributed as dist
        ok = 1
        try:
            self._pools.attach_group(group, barrier=False)
        except _lib.CFMMError:
            ok = 0
        dev = torch.device("cuda", self._pools.device) if dist.get_backend(group) == "nccl" else torch.device("cpu")
        flag = torch.tensor([ok], dtype=torch.int32, device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if int(flag.item()) == 0:
            if ok:
                self._pools.detach_group()
            self._exchange = "dist"
        dist.barrier(group)

    # ascii aliases
    @property
    def Ds(self):
        return self.Δs

    @property
    def Ls(self):
        return self.Λs

    def _upload(self):
        shard = self.cfmms[self._lo:self._hi]
        idx = _pack(shard)
        order = self._add(shard, idx, append=False)  # library global order -> shard-local list position
        self._pools.finalize()
        self._order = np.asarray(order, dtype=np.int64)
        self._type_lists = idx

    def _add(self, cs_all, idx, append):
        """Hand the pools cs_all[idx[t]] to the library type by type (cfmm_add_* before finalize,
        cfmm_append_* after); returns the positions in cs_all in the library's global order."""
        p = self._pools
        order = []
        if idx[0]:
            cs = [cs_all[i] for i in idx[0]]
            (p.append_product if append else p.add_product)(
                np.array([c.R for c in cs]), np.array([c.gamma for c in cs]), np.array([c.Ai for c in cs]))
            order += idx[0]
        if idx[1]:
            cs = [cs_all[i] for i in idx[1]]
            (p.append_geomean if append else p.add_geomean)(
                np.array([c.R for c in cs]), np.array([c.gamma for c in cs]),
                np.array([c.Ai for c in cs]), np.array([c.w for c in cs]))
            order += idx[1]
        if idx[2]:
            cs = [cs_all[i] for i in idx[2]]
            off = np.concatenate([[0], np.cumsum([len(c.lower_ticks) for c in cs])]).astype(np.int64)
            (p.append_univ3 if append else p.add_univ3)(
                np.array([c.current_price for c in cs]), np.array([c.gamma for c in cs]),
                np.array([c.Ai for c in cs]), off, np.concatenate([c.lower_ticks for c in cs]),
                np.concatenate([c.liquidity for c in cs]))
            order += idx[2]
        return order

    def add_cfmms(self, cfmms):
        """Add pools to a built router without rebuilding it (cfmm_append_*): they extend r.cfmms,
        r.Δs and r.Λs, and trade from the next route on.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("add_cfmms drives one GPU")
        new = list(cfmms)
        if not new:
            return
        idx = _pack(new)
        base = len(self.cfmms)
        order = self._add(new, idx, append=True)
        self.cfmms += new
        self.Δs = np.concatenate([self.Δs, np.zeros((len(new), 2))])
        self.Λs = np.concatenate([self.Λs, np.zeros((len(new), 2))])
        self._retired = np.concatenate([self._retired, np.zeros(len(new), dtype=bool)])
        self._order = np.concatenate([self._order, base + np.asarray(order, dtype=np.int64)])
        self._hi = len(self.cfmms)
        for t in (0, 1, 2):
            self._type_lists[t] = self._type_lists[t] + [base + i for i in idx[t]]

    def set_active(self, list_indices, flag: bool):
        """Retire (flag False) or restore (True) the pools r.cfmms[i] for i in list_indices
        (cfmm_set_active).  A retired pool trades nothing and update_reserves(r) leaves it as it
        is; its trades read back as zero.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("set_active drives one GPU")
        ids = np.unique(np.asarray(list_indices, dtype=np.int64).reshape(-1))
        if len(ids) and (ids[0] < 0 or ids[-1] >= len(self.cfmms)):
            raise IndexError("set_active: pool index out of range")
        for t in (0, 1, 2):
            local = {i: k for k, i in enumerate(self._type_lists[t])}
            ks = sorted(local[i] for i in ids if i in local)
            if not ks:
                continue
            span = np.array(self._type_lists[t][ks[0]:ks[-1] + 1])
            active = ~self._retired[span]
            active[np.asarray(ks) - ks[0]] = bool(flag)
            self._pools.set_active(t, ks[0], active)
            self._retired[span] = ~active

    def _locate(self):
        """Per list position: the pool's type and its index in the type's insertion order."""
        kind = np.full(len(self.cfmms), -1, dtype=np.int64)
        local = np.zeros(len(self.cfmms), dtype=np.int64)
        for t in (0, 1, 2):
            lst = np.asarray(self._type_lists[t], dtype=np.int64)
            kind[lst] = t
            local[lst] = np.arange(len(lst))
        return kind, local

    def _swap_rows(self, list_indices, tenders, what):
        """Per pool type: (rows of the call, type-local pool indices) of the pools r.cfmms[i]."""
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        ids = np.asarray(list_indices, dtype=np.int64).reshape(-1)
        tenders = np.ascontiguousarray(tenders, dtype=np.float64)
        if tenders.shape != (len(ids), 2):
            raise ValueError(f"{what}: tenders must have shape ({len(ids)}, 2)")
        if len(ids) and (ids.min() < 0 or ids.max() >= len(self.cfmms)):
            raise IndexError(f"{what}: pool index out of range")
        kind, local = self._locate()
        groups = []
        for t in (0, 1, 2):
            rows = np.flatnonzero(kind[ids] == t)
            if len(rows):
                groups.append((t, rows, local[ids[rows]]))
        return ids, tenders, groups

    def quote_swaps(self, list_indices, tenders):
        """What tendering tenders[j] (in the pool's token order) to r.cfmms[list_indices[j]] pays
        out, every row on the current state on its own (cfmm_quote_swaps); no state changes.
        Returns received (q, 2) in the caller's order.  Single GPU."""
        ids, tenders, groups = self._swap_rows(list_indices, tenders, "quote_swaps")
        out = np.zeros((len(ids), 2))
        for t, rows, loc in groups:
            out[rows] = self._pools.quote_swaps(t, loc, tenders[rows])
        return out

    def execute_swaps(self, list_indices, tenders):
        """Execute the swaps in order (cfmm_execute_swaps): each row sees every earlier row on the
        same pool.  Returns received (q, 2) in the caller's order and refreshes the touched pool
        objects (R, or current_price / current_tick) from the device state.  Single GPU."""
        ids, tenders, groups = self._swap_rows(list_indices, tenders, "execute_swaps")
        out = np.zeros((len(ids), 2))
        for t, rows, loc in groups:
            out[rows] = self._pools.execute_swaps(t, loc, tenders[rows])
        self._refresh_swapped(groups)
        return out

    def quote_swaps_exact_out(self, list_indices, wants):
        """The tender each row needs to receive wants[j] ((0, y): y of the pool's token 2 for its
        token 1; (y, 0) the reverse) from r.cfmms[list_indices[j]], every row on the current state on
        its own (cfmm_quote_swaps_exact_out); no state changes.  Returns tender (q, 2) in the
        caller's order, +inf where y cannot be reached.  Single GPU."""
        ids, wants, groups = self._swap_rows(list_indices, wants, "quote_swaps_exact_out")
        out = np.zeros((len(ids), 2))
        for t, rows, loc in groups:
            out[rows] = self._pools.quote_swaps_exact_out(t, loc, wants[rows])
        return out

    def execute_swap_orders(self, list_indices, kinds, amounts, limits=None):
        """Execute exact-in (kind 0) and exact-out (kind 1) rows in order with optional limits
        (cfmm_execute_swap_orders): a row whose limit fails reverts and later rows see the state
        without it.  Returns (paid, received, status) in the caller's order and refreshes the
        touched pool objects from the device state, as execute_swaps does.  Single GPU."""
        ids, amounts, groups = self._swap_rows(list_indices, amounts, "execute_swap_orders")
        kinds = np.asarray(kinds, dtype=np.uint8).reshape(-1)
        if len(kinds) != len(ids):
            raise ValueError(f"execute_swap_orders: kinds must have {len(ids)} entries")
        if limits is not None:
            limits = np.asarray(limits, dtype=np.float64).reshape(-1)
            if len(limits) != len(ids):
                raise ValueError(f"execute_swap_orders: limits must have {len(ids)} entries")
        paid, received = np.zeros((len(ids), 2)), np.zeros((len(ids), 2))
        status = np.zeros(len(ids), dtype=np.uint8)
        for t, rows, loc in groups:
            paid[rows], received[rows], status[rows] = self._pools.execute_swap_orders(
                t, loc, kinds[rows], amounts[rows], None if limits is None else limits[rows])
        self._refresh_swapped(groups)
        return paid, received, status

    def _path_args(self, paths, token_in, kinds, amounts, what):
        """The CSR form of cfmm_quote_paths of paths (lists of r.cfmms positions), and the per-type
        groups of the hops' pools (for _refresh_swapped)."""
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        paths = [np.asarray(p, dtype=np.int64).reshape(-1) for p in paths]
        q = len(paths)
        token_in, kinds, amounts = (np.asarray(a).reshape(-1) for a in (token_in, kinds, amounts))
        if not (len(token_in) == len(kinds) == len(amounts) == q):
            raise ValueError(f"{what}: token_in, kinds and amounts need one entry per path ({q})")
        off = np.zeros(q + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in paths])
        ids = np.concatenate(paths) if q else np.zeros(0, dtype=np.int64)
        if len(ids) and (ids.min() < 0 or ids.max() >= len(self.cfmms)):
            raise IndexError(f"{what}: pool index out of range")
        kind, local = self._locate()
        hop_type, hop_pool = kind[ids], local[ids]
        groups = [(t, None, hop_pool[hop_type == t]) for t in (0, 1, 2) if np.any(hop_type == t)]
        return off, hop_type, hop_pool, token_in, kinds, amounts, groups

    def quote_paths(self, paths, token_in, kinds, amounts):
        """Price multi-hop paths (cfmm_quote_paths): paths[j] lists r.cfmms positions, token_in[j]
        (1-based, as Ai) is tendered to the first pool, and each pool's output goes to the next.  Kind
        0 tenders amounts[j]; kind 1 wants amounts[j] out of the last pool.  Every path on the current
        state on its own; no state changes.  Returns (paid [q], received [q], status [q], hop_tender
        [H], hop_received [H]) with the hops flattened in path order.  Single GPU."""
        off, ht, hp, tok, kinds, amounts, _ = self._path_args(paths, token_in, kinds, amounts, "quote_paths")
        tender, received, status = self._pools.quote_paths(off, ht, hp, tok, kinds, amounts)
        return self._path_result(off, tender, received, status)

    def execute_paths(self, paths, token_in, kinds, amounts, limits=None):
        """Execute multi-hop paths in order (cfmm_execute_paths), each with an optional limit (kind 0:
        the minimum final output; kind 1: the maximum tender): a path whose limit fails reverts every
        hop and later paths see the state without it.  Returns what quote_paths returns and refreshes
        the touched pool objects from the device state, as execute_swaps does.  Single GPU."""
        off, ht, hp, tok, kinds, amounts, groups = self._path_args(paths, token_in, kinds, amounts, "execute_paths")
        if limits is not None:
            limits = np.asarray(limits, dtype=np.float64).reshape(-1)
            if len(limits) != len(off) - 1:
                raise ValueError(f"execute_paths: limits must have {len(off) - 1} entries")
        tender, received, status = self._pools.execute_paths(off, ht, hp, tok, kinds, amounts, limits)
        self._refresh_swapped(groups)
        return self._path_result(off, tender, received, status)

    @staticmethod
    def _path_result(off, tender, received, status):
        q = len(off) - 1
        paid = tender[off[:-1]] if q else np.zeros(0)
        got = received[off[1:] - 1] if q else np.zeros(0)
        return paid, got, status, tender, received

    def pair_pools(self, a, b):
        """The r.cfmms positions of the pools that hold the token pair {a, b} (1-based), in the
        library's global insertion order, retired ones included (cfmm_pair_pools).  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("pair_pools drives one GPU")
        _, typ, idx, _ = self._pools.pair_pools([int(a)], [int(b)])
        return np.array([self._type_lists[int(t)][int(i)] for t, i in zip(typ, idx)], dtype=np.int64)

    def _split_args(self, token_in, token_out, kinds, amounts, limits, what):
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        tin, tout, kinds, amounts = (np.asarray(x).reshape(-1) for x in (token_in, token_out, kinds, amounts))
        if not (len(tin) == len(tout) == len(kinds) == len(amounts)):
            raise ValueError(f"{what}: token_in, token_out, kinds and amounts need one entry per row")
        if limits is not None:
            limits = np.asarray(limits, dtype=np.float64).reshape(-1)
            if len(limits) != len(tin):
                raise ValueError(f"{what}: limits must have {len(tin)} entries")
        return tin, tout, kinds, amounts, limits

    def quote_split_orders(self, token_in, token_out, kinds, amounts):
        """Sell token_in[j] for token_out[j] (1-based) over every pool of the pair, split so that the
        pools' marginal prices meet (cfmm_quote_split_orders): kind 0 tenders amounts[j], kind 1 wants
        amounts[j] out.  Every row on the current state on its own; no state changes.  Returns
        (paid [q], received [q], price [q], status [q]); price is s* = ν_in/ν_out.  Single GPU."""
        tin, tout, kinds, amounts, _ = self._split_args(token_in, token_out, kinds, amounts, None,
                                                        "quote_split_orders")
        return self._pools.quote_split_orders(tin, tout, kinds, amounts)

    def execute_split_orders(self, token_in, token_out, kinds, amounts, limits=None):
        """Execute split orders in order (cfmm_execute_split_orders), each with an optional limit (kind
        0: the minimum received; kind 1: the maximum paid): a row whose limit fails reverts and later
        rows see the state without it.  Returns what quote_split_orders returns and refreshes the pool
        objects of the filled rows' pairs from the device state, as execute_swaps does.  Single GPU."""
        tin, tout, kinds, amounts, limits = self._split_args(token_in, token_out, kinds, amounts, limits,
                                                             "execute_split_orders")
        out = self._pools.execute_split_orders(tin, tout, kinds, amounts, limits)
        filled = out[3] == _lib.ORDER_FILLED
        if np.any(filled):
            _, typ, idx, _ = self._pools.pair_pools(tin[filled], tout[filled])
            self._refresh_swapped([(t, None, idx[typ == t]) for t in (0, 1, 2) if np.any(typ == t)])
        return out

    def _routed_args(self, token_in, token_out, kinds, amounts, hubs, limits, what):
        tin, tout, kinds, amounts, limits = self._split_args(token_in, token_out, kinds, amounts, limits, what)
        q = len(tin)
        if all(np.ndim(h) == 0 for h in hubs):  # one list shared by every row
            per_row = [list(hubs)] * q
        else:
            per_row = [list(h) for h in hubs]
            if len(per_row) != q:
                raise ValueError(f"{what}: hubs must be one list, or one list per row ({q})")
        hub_off = np.concatenate([[0], np.cumsum([len(h) for h in per_row])]).astype(np.int64)
        flat = np.array([int(x) for h in per_row for x in h], dtype=np.int64)
        return tin, tout, kinds, amounts, hub_off, flat, limits

    def quote_routed_orders(self, token_in, token_out, kinds, amounts, hubs):
        """Sell token_in[j] for token_out[j] (1-based) over the pools of the pair and the two-hop routes
        through the hub tokens `hubs` (one list for every row, or one list per row; at most
        ROUTE_MAX_HUBS each), split optimally (cfmm_quote_routed_orders): kind 0 tenders amounts[j],
        kind 1 wants amounts[j] out.  Pools between two hubs are not used.  Every row on the current
        state on its own; no state changes.  Returns (paid [q], received [q], price [q], status [q]);
        price is s* = ν_in/ν_out.  Single GPU."""
        tin, tout, kinds, amounts, off, flat, _ = self._routed_args(token_in, token_out, kinds, amounts, hubs, None,
                                                                    "quote_routed_orders")
        return self._pools.quote_routed_orders(tin, tout, kinds, amounts, off, flat)[:4]

    def execute_routed_orders(self, token_in, token_out, kinds, amounts, hubs, limits=None):
        """Execute routed orders in order (cfmm_execute_routed_orders), each with an optional limit (kind
        0: the minimum received; kind 1: the maximum paid): a row whose limit fails reverts and later
        rows see the state without it.  Returns what quote_routed_orders returns and refreshes the pool
        objects of the filled rows' pairs from the device state, as execute_swaps does.  Single GPU."""
        tin, tout, kinds, amounts, off, flat, limits = self._routed_args(token_in, token_out, kinds, amounts, hubs,
                                                                         limits, "execute_routed_orders")
        out = self._pools.execute_routed_orders(tin, tout, kinds, amounts, off, flat, limits)[:4]
        filled = np.flatnonzero(out[3] == _lib.ORDER_FILLED)
        if len(filled):
            sub = np.concatenate([[0], np.cumsum(np.diff(off)[filled])]).astype(np.int64)
            fh = np.concatenate([flat[off[r]:off[r + 1]] for r in filled]).astype(np.int64)
            a, b, _ = DevicePools.route_pairs(tin[filled], tout[filled], sub, fh)
            _, typ, idx, _ = self._pools.pair_pools(a, b)
            self._refresh_swapped([(t, None, idx[typ == t]) for t in (0, 1, 2) if np.any(typ == t)])
        return out

    def _choose(self, token_in, token_out, kinds, amounts, max_hubs, allowed, what):
        tin, tout, kinds, amounts, _ = self._split_args(token_in, token_out, kinds, amounts, None, what)
        if not 0 <= int(max_hubs) <= _lib.ROUTE_MAX_HUBS:
            raise ValueError(f"{what}: max_hubs must be 0..{_lib.ROUTE_MAX_HUBS}")
        off, flat, _, _ = self._pools.choose_order_hubs(tin, tout, kinds, amounts, int(max_hubs), allowed)
        return tin, tout, kinds, amounts, off, flat

    def choose_hubs(self, token_in, token_out, kinds, amounts, max_hubs: int = _lib.ROUTE_MAX_HUBS, allowed=None):
        """Choose each order row's hub tokens on the device (cfmm_choose_order_hubs): the common
        neighbours h of token_in[j] and token_out[j] (1-based; with allowed[h - 1] when a mask over the
        tokens is given) that carry a two-hop route on active pools, ranked by that route's best single
        quote (kind 0: most received for amounts[j]; kind 1: least paid for amounts[j] out), at most
        max_hubs per row.  No state changes.  Returns one list of hubs per row, best first, ready for
        quote_routed_orders / execute_routed_orders.  Single GPU."""
        _, _, _, _, off, flat = self._choose(token_in, token_out, kinds, amounts, max_hubs, allowed, "choose_hubs")
        return [flat[off[r]:off[r + 1]].tolist() for r in range(len(off) - 1)]

    def quote_auto_routed_orders(self, token_in, token_out, kinds, amounts, max_hubs: int = _lib.ROUTE_MAX_HUBS,
                                 allowed=None):
        """choose_hubs, then quote_routed_orders with the chosen hubs: each row split optimally over its
        pair's pools and the two-hop routes through its chosen hubs.  No state changes.  Returns
        (paid [q], received [q], price [q], status [q], hubs), hubs one list per row.  Single GPU."""
        tin, tout, kinds, amounts, off, flat = self._choose(token_in, token_out, kinds, amounts, max_hubs, allowed,
                                                            "quote_auto_routed_orders")
        out = self._pools.quote_routed_orders(tin, tout, kinds, amounts, off, flat)[:4]
        return out + ([flat[off[r]:off[r + 1]].tolist() for r in range(len(tin))],)

    def execute_auto_routed_orders(self, token_in, token_out, kinds, amounts, limits=None,
                                   max_hubs: int = _lib.ROUTE_MAX_HUBS, allowed=None):
        """choose_hubs, then execute_routed_orders with the chosen hubs and the optional limits (kind 0:
        the minimum received; kind 1: the maximum paid).  Every row's hubs are chosen once, on the state
        at entry; the execute then re-solves each row, over those hubs, on the state the earlier rows
        left.  Returns what quote_auto_routed_orders returns and refreshes the touched pool objects, as
        execute_routed_orders does.  Single GPU."""
        tin, tout, kinds, amounts, off, flat = self._choose(token_in, token_out, kinds, amounts, max_hubs, allowed,
                                                            "execute_auto_routed_orders")
        hubs = [flat[off[r]:off[r + 1]].tolist() for r in range(len(tin))]
        return self.execute_routed_orders(tin, tout, kinds, amounts, hubs, limits) + (hubs,)

    def _find(self, token_in, token_out, kinds, amounts, allowed, max_hops, limits, what, hop_cost=None):
        tin, tout, kinds, amounts, limits = self._split_args(token_in, token_out, kinds, amounts, limits, what)
        if not 1 <= int(max_hops) <= _lib.PATH_MAX_HOPS:
            raise ValueError(f"{what}: max_hops must be 1..{_lib.PATH_MAX_HOPS}")
        if allowed is None:
            raise ValueError(f"{what}: allowed (a mask over the tokens) is required")
        if hop_cost is None:
            found = self._pools.find_order_paths(tin, tout, kinds, amounts, int(max_hops), allowed)
        else:
            settle = np.where(np.asarray(kinds).astype(np.int64) == 1, tin, tout)
            found = self._pools.find_order_paths_net(tin, tout, kinds, amounts, int(max_hops), allowed,
                                                     pack_hop_cost(hop_cost, len(self.v), settle, what))
        off, typ, pool = found[:3]
        paths = [[self._type_lists[int(typ[h])][int(pool[h])] for h in range(off[r], off[r + 1])]
                 for r in range(len(tin))]
        return tin, tout, kinds, amounts, limits, found, paths

    def find_paths(self, token_in, token_out, kinds, amounts, allowed, max_hops: int = _lib.PATH_MAX_HOPS,
                   hop_cost=None):
        """Find each order row's best single path on the device (cfmm_find_order_paths): at most
        max_hops hops from token_in[j] to token_out[j] (1-based), one pool per hop, every intermediate
        token t with allowed[t - 1] (a mask over the tokens), ranked by the amount out (kind 0, for
        amounts[j] in) or in (kind 1, for amounts[j] out).  No state changes.  Returns (paths, value
        [q], status [q]): paths[j] lists r.cfmms positions in hop order (empty without a path), ready
        for quote_paths / execute_paths with token_in.  hop_cost (a scalar, or per token as hop_costs
        returns it; row j pays its settlement token's, token_out kind 0 and token_in kind 1): the path
        whose amount net of hop_cost per hop is best (cfmm_find_order_paths_net), and net [q] is
        returned last.  Single GPU."""
        *_, found, paths = self._find(token_in, token_out, kinds, amounts, allowed, max_hops, None, "find_paths",
                                      hop_cost)
        return (paths, found[6], found[7]) + tuple(found[8:])

    def quote_best_paths(self, token_in, token_out, kinds, amounts, allowed, max_hops: int = _lib.PATH_MAX_HOPS,
                         hop_cost=None):
        """find_paths, priced: what quote_paths returns for the found paths, bit for bit (the find's
        amounts are that recursion).  Returns (paid [q], received [q], status [q], paths); a row
        without a path has paid = received = 0 and the find's status.  hop_cost: as find_paths, with
        net [q] returned last.  No state changes.  Single GPU."""
        *_, found, paths = self._find(token_in, token_out, kinds, amounts, allowed, max_hops, None,
                                      "quote_best_paths", hop_cost)
        off, tender, received, status = found[0], found[4], found[5], found[7]
        has = np.diff(off) > 0
        paid, got = np.zeros(len(paths)), np.zeros(len(paths))
        paid[has], got[has] = tender[off[:-1][has]], received[off[1:][has] - 1]
        return (paid, got, status, paths) + tuple(found[8:])

    def execute_best_paths(self, token_in, token_out, kinds, amounts, allowed, max_hops: int = _lib.PATH_MAX_HOPS,
                           limits=None, hop_cost=None):
        """find_paths, then execute_paths over the rows that have a path, with the optional limits
        (kind 0: the minimum received; kind 1: the maximum paid).  Every row's path is found once, on
        the state at entry; the execute re-prices each path on the state the earlier paths left.
        Returns what quote_best_paths returns (rows without a path: zeros and the find's status) and
        refreshes the touched pool objects, as execute_paths does.  hop_cost: as find_paths, with the
        find's net [q] returned last.  Single GPU."""
        tin, _, kinds, amounts, limits, found, paths = self._find(token_in, token_out, kinds, amounts, allowed,
                                                                  max_hops, limits, "execute_best_paths", hop_cost)
        status = found[7].copy()
        paid, got = np.zeros(len(paths)), np.zeros(len(paths))
        rows = np.array([r for r in range(len(paths)) if paths[r]], dtype=np.int64)
        if len(rows):
            p, g, s, _, _ = self.execute_paths([paths[r] for r in rows], tin[rows], kinds[rows], amounts[rows],
                                               None if limits is None else limits[rows])
            paid[rows], got[rows], status[rows] = p, g, s
        return (paid, got, status, paths) + tuple(found[8:])

    def quote_token_values(self, roots, kinds, amounts, max_hops: int = _lib.PATH_MAX_HOPS, allowed=None,
                           hop_cost=None):
        """Value every token against each row's root on the device (cfmm_quote_token_values): kind 0
        rows spend amounts[r] of roots[r] (1-based) and get, per token, the most of it that a walk of at
        most max_hops hops delivers; kind 1 rows receive amounts[r] of the root and get, per token, the
        least of it that such a walk must be paid.  Walks pass through tokens t with allowed[t - 1] (a
        mask over the tokens; None: every token), one pool per hop.  No state changes.  Returns (value,
        hops, status), each [q, n_tokens]: value 0 (kind 0) or inf (kind 1) where no walk reaches.
        hop_cost (a scalar, or the cost of one hop in each token, as hop_costs returns it): per token
        the walk whose amount net of the token's hop_cost per hop is best
        (cfmm_quote_token_values_net), and net [q, n_tokens] is returned last.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("quote_token_values drives one GPU")
        if not 1 <= int(max_hops) <= _lib.PATH_MAX_HOPS:
            raise ValueError(f"quote_token_values: max_hops must be 1..{_lib.PATH_MAX_HOPS}")
        if hop_cost is None:
            return self._pools.quote_token_values(roots, kinds, amounts, int(max_hops), allowed)[:3]
        cost = pack_hop_cost(hop_cost, len(self.v), None, "quote_token_values")
        value, hops, status, net, _ = self._pools.quote_token_values_net(roots, kinds, amounts, int(max_hops), cost,
                                                                         allowed)
        return value, hops, status, net

    def hop_costs(self, gas_token, gas_per_hop, max_hops: int = _lib.PATH_MAX_HOPS, allowed=None):
        """What gas_per_hop of gas_token (1-based) buys of each token: the exact-in token values rooted
        at the gas token, [n_tokens].  The gas token gets gas_per_hop and unreached tokens inf (no walk
        into them pays for itself).  Ready as the hop_cost of find_paths, quote_token_values and the
        other path calls.  No state changes.  Single GPU."""
        value, _, status = self.quote_token_values([gas_token], [0], [gas_per_hop], max_hops, allowed)
        cost = value[0].copy()
        cost[status[0] == _lib.ORDER_UNREACHABLE] = np.inf
        return cost

    def token_paths(self, root, kind, amount, tokens, max_hops: int = _lib.PATH_MAX_HOPS, allowed=None,
                    hop_cost=None):
        """The walks behind quote_token_values for one root and the given tokens (1-based): kind 0
        from the root to each token, kind 1 from each token into the root.  Returns (paths, token_in,
        value, status): paths[j] lists r.cfmms positions in hop order (empty for the root, an unreached
        token or a walk that repeats a pool), ready for quote_paths / execute_paths with token_in[j]
        and the same kind and amount; value[j] the token's value.  hop_cost: as quote_token_values,
        the walks net of it, with net [len(tokens)] returned last.  No state changes.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("token_paths drives one GPU")
        if not 1 <= int(max_hops) <= _lib.PATH_MAX_HOPS:
            raise ValueError(f"token_paths: max_hops must be 1..{_lib.PATH_MAX_HOPS}")
        tokens = np.asarray(tokens, dtype=np.int64).reshape(-1)
        req = (np.zeros(len(tokens), dtype=np.int64), tokens)
        if hop_cost is None:
            got = self._pools.quote_token_values([root], [kind], [amount], int(max_hops), allowed, req)
        else:
            cost = pack_hop_cost(hop_cost, len(self.v), None, "token_paths")
            got = self._pools.quote_token_values_net([root], [kind], [amount], int(max_hops), cost, allowed, req)
            net = got[3]
            got = got[:3] + got[4:]
        value, off, typ, pool, st = got[0], got[4], got[5], got[6], got[10]
        paths = [[self._type_lists[int(typ[h])][int(pool[h])] for h in range(off[j], off[j + 1])]
                 for j in range(len(tokens))]
        token_in = tokens.copy() if int(kind) == 1 else np.full(len(tokens), int(root), dtype=np.int64)
        out = (paths, token_in, value[0, tokens - 1], st)
        return out if hop_cost is None else out + (net[0, tokens - 1],)

    def _subgraph_args(self, token_in, token_out, amounts, allowed, limits, what):
        tin, tout, _, amounts, limits = self._split_args(token_in, token_out, np.zeros(len(np.atleast_1d(token_in))),
                                                         amounts, limits, what)
        if allowed is None:
            raise ValueError(f"{what}: allowed (a mask over the tokens) is required")
        return tin, tout, amounts, limits

    def quote_subgraph_orders(self, token_in, token_out, amounts, allowed, opts=None, kind=None):
        """Sell amounts[j] of token_in[j] for token_out[j] (1-based; kind 0, exact-in), or buy
        amounts[j] of token_out[j] paying in token_in[j] (kind 1, exact-out), over every pool among the
        two and the tokens t with allowed[t - 1] (a mask over the tokens, at most 256 such tokens per
        row besides its two), split optimally: route! over those pools, one dual solve per row on the
        device (cfmm_quote_subgraph_swap_orders).  kind: None (every row exact-in), a scalar, or one
        entry per row.  No state changes.  Returns (paid [q], received [q], status [q], detail):
        detail is DevicePools.quote_subgraph_orders' namespace (solver status, iterations, ν, Ψ,
        legs).  Single GPU.  allowed may instead be one list of 1-based tokens per row (choose_hubs' output
        as it is): each row then runs over its own list, as the call with that list as its mask (the *_rows
        calls)."""
        tin, tout, amounts, _ = self._subgraph_args(token_in, token_out, amounts, allowed, None,
                                                    "quote_subgraph_orders")
        out = self._pools.quote_subgraph_orders(tin, tout, amounts, allowed, opts, kind)
        return out.paid, out.received, out.status, out

    def execute_subgraph_orders(self, token_in, token_out, amounts, allowed, limits=None, opts=None, kind=None):
        """Execute subgraph orders in order (cfmm_execute_subgraph_swap_orders), each re-solved on the
        state the earlier filled rows left, with an optional limit per row (exact-in: the minimum
        received; exact-out: the maximum paid): a row that misses it reverts.  Returns what
        quote_subgraph_orders returns and refreshes the pool objects the filled rows traded with from
        the device state, as execute_swaps does.  Single GPU."""
        tin, tout, amounts, limits = self._subgraph_args(token_in, token_out, amounts, allowed, limits,
                                                         "execute_subgraph_orders")
        out = self._pools.execute_subgraph_orders(tin, tout, amounts, allowed, limits, opts, kind)
        self._refresh_filled(out)
        return out.paid, out.received, out.status, out

    def _refresh_filled(self, out):
        """Refresh the pool objects the filled rows of a subgraph or basket execute traded with."""
        filled = np.flatnonzero(out.status == _lib.ORDER_FILLED)
        if len(filled):
            sel = np.concatenate([np.arange(out.leg_off[r], out.leg_off[r + 1]) for r in filled]).astype(np.int64)
            typ, idx = out.leg_type[sel], out.leg_pool[sel]
            if len(sel):
                self._refresh_swapped([(t, None, idx[typ == t]) for t in (0, 1, 2) if np.any(typ == t)])

    def _basket_args(self, token_out, baskets, allowed, limits, what):
        """(token_out, basket_off, basket_token, basket_amount, limits) from baskets: one {token:
        amount} dict or (tokens, amounts) pair per row."""
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        tout = np.asarray(token_out, dtype=np.int64).reshape(-1)
        if len(baskets) != len(tout):
            raise ValueError(f"{what}: token_out and baskets need one entry per row")
        off, toks, amts = [0], [], []
        for b in baskets:
            t, a = (list(b.keys()), list(b.values())) if isinstance(b, dict) else (list(b[0]), list(b[1]))
            if len(t) != len(a):
                raise ValueError(f"{what}: a basket needs one amount per token")
            toks += t
            amts += a
            off.append(len(toks))
        if limits is not None:
            limits = np.asarray(limits, dtype=np.float64).reshape(-1)
            if len(limits) != len(tout):
                raise ValueError(f"{what}: limits must have {len(tout)} entries")
        if allowed is None:
            raise ValueError(f"{what}: allowed (a mask over the tokens) is required")
        return (tout, np.array(off, np.int64), np.array(toks, np.int64), np.array(amts, np.float64).reshape(-1),
                limits)

    @staticmethod
    def _per_entry(out):
        return [out.paid[out.basket_off[r]:out.basket_off[r + 1]] for r in range(len(out.basket_off) - 1)]

    def _swap_basket_args(self, token_out, sells, buys, allowed, limits, what):
        """_basket_args over each row's sold entries then its bought entries, plus the entry kinds and
        each row's count of sold entries."""
        if len(sells) != len(buys):
            raise ValueError(f"{what}: sells and buys need one entry per row")
        rows, n_sell = [], []
        for s, b in zip(sells, buys):
            st, sa = (list(s.keys()), list(s.values())) if isinstance(s, dict) else (list(s[0]), list(s[1]))
            bt, ba = (list(b.keys()), list(b.values())) if isinstance(b, dict) else (list(b[0]), list(b[1]))
            if len(st) != len(sa) or len(bt) != len(ba):
                raise ValueError(f"{what}: sells and buys need one amount per token")
            rows.append((st + bt, sa + ba))
            n_sell.append(len(st))
        tout, off, toks, amts, limits = self._basket_args(token_out, rows, allowed, limits, what)
        kind = np.zeros(len(toks), np.uint8)
        for r, ns in enumerate(n_sell):
            kind[off[r] + ns:off[r + 1]] = _lib.SWAP_EXACT_OUT
        return tout, off, toks, amts, kind, limits, n_sell

    @staticmethod
    def _sold_bought(out, n_sell):
        per = Router._per_entry(out)
        return [p[:ns] for p, ns in zip(per, n_sell)], [0.0 - p[ns:] for p, ns in zip(per, n_sell)]

    def quote_basket_swap_orders(self, token_out, sells, buys, allowed, opts=None):
        """Sell and buy token baskets in one order per row, settled in token_out[r]: sells[r] and
        buys[r] are {token: amount} or (tokens, amounts) (together 1 to 16 distinct 1-based tokens,
        none of them token_out[r]; at least one bought token makes the row a buy row).  Each row
        maximises its net of token_out[r] over every pool among its tokens and the tokens t with
        allowed[t - 1], selling up to the sold amounts and buying at least the bought ones, one dual
        solve per row on the device (cfmm_quote_basket_swap_orders).  No state changes.  Returns (sold
        per row, bought per row as lists of arrays in the caller's order, the net of token_out [q]
        (negative when the row pays), status [q], detail); detail is DevicePools.quote_basket_orders'
        namespace.  Single GPU.  allowed may instead be one list of 1-based tokens per row (choose_hubs'
        output as it is): each row then runs over its own list, as the call with that list as its mask (the
        *_rows calls)."""
        tout, off, toks, amts, kind, _, n_sell = self._swap_basket_args(token_out, sells, buys, allowed, None,
                                                                         "quote_basket_swap_orders")
        out = self._pools.quote_basket_orders(tout, off, toks, amts, allowed, opts, kind)
        sold, bought = self._sold_bought(out, n_sell)
        return sold, bought, out.received, out.status, out

    def execute_basket_swap_orders(self, token_out, sells, buys, allowed, limits=None, opts=None):
        """Execute basket swap orders in order (cfmm_execute_basket_swap_orders), each re-solved on the
        state the earlier filled rows left, with an optional minimum net of token_out per row (negative:
        pay at most -limit; -inf allowed): a row below it reverts.  Returns what
        quote_basket_swap_orders returns and refreshes the pool objects the filled rows traded with
        from the device state.  Single GPU."""
        tout, off, toks, amts, kind, limits, n_sell = self._swap_basket_args(token_out, sells, buys, allowed, limits,
                                                                             "execute_basket_swap_orders")
        out = self._pools.execute_basket_orders(tout, off, toks, amts, allowed, limits, opts, kind)
        self._refresh_filled(out)
        sold, bought = self._sold_bought(out, n_sell)
        return sold, bought, out.received, out.status, out

    def quote_basket_orders(self, token_out, baskets, allowed, opts=None):
        """Sell each row's basket (baskets[r]: {token: amount} or (tokens, amounts); 1 to 16 distinct
        1-based tokens, none of them token_out[r]) for token_out[r] over every pool among them and the
        tokens t with allowed[t - 1] (a mask over the tokens), split optimally: route! with
        BasketLiquidation(token_out[r], Δin) over those pools, one dual solve per row on the device
        (cfmm_quote_basket_orders).  No state changes.  Returns (paid per entry as a list of arrays in
        the basket's order, received [q], status [q], detail): detail is DevicePools.
        quote_basket_orders' namespace.  Single GPU.  allowed may instead be one list of 1-based tokens per
        row (choose_hubs' output as it is): each row then runs over its own list, as the call with that list
        as its mask (the *_rows calls)."""
        tout, off, toks, amts, _ = self._basket_args(token_out, baskets, allowed, None, "quote_basket_orders")
        out = self._pools.quote_basket_orders(tout, off, toks, amts, allowed, opts)
        return self._per_entry(out), out.received, out.status, out

    def execute_basket_orders(self, token_out, baskets, allowed, limits=None, opts=None):
        """Execute basket orders in order (cfmm_execute_basket_orders), each re-solved on the state the
        earlier filled rows left, with an optional minimum received per row: a row below it reverts.
        Returns what quote_basket_orders returns and refreshes the pool objects the filled rows traded
        with from the device state.  Single GPU."""
        tout, off, toks, amts, limits = self._basket_args(token_out, baskets, allowed, limits,
                                                          "execute_basket_orders")
        out = self._pools.execute_basket_orders(tout, off, toks, amts, allowed, limits, opts)
        self._refresh_filled(out)
        return self._per_entry(out), out.received, out.status, out

    def _limit_args(self, token_out, sells, allowed, min_received, what):
        """_basket_args over sells[r]: {token: (amount, limit)} or (tokens, amounts, limits), plus the
        limit prices."""
        rows, lims = [], []
        for s in sells:
            if isinstance(s, dict):
                t = list(s.keys())
                pairs = [tuple(v) for v in s.values()]
                if any(len(v) != 2 for v in pairs):
                    raise ValueError(f"{what}: a sell needs (amount, limit) per token")
                a, c = [v[0] for v in pairs], [v[1] for v in pairs]
            else:
                if len(s) != 3:
                    raise ValueError(f"{what}: a sell is {{token: (amount, limit)}} or (tokens, amounts, limits)")
                t, a, c = list(s[0]), list(s[1]), list(s[2])
                if len(c) != len(t):
                    raise ValueError(f"{what}: a sell needs one limit per token")
            rows.append((t, a))
            lims += c
        tout, off, toks, amts, min_received = self._basket_args(token_out, rows, allowed, min_received, what)
        return tout, off, toks, amts, np.array(lims, np.float64).reshape(-1), min_received

    def quote_limit_orders(self, token_out, sells, allowed, opts=None):
        """Limit orders settled in token_out[r]: sells[r] is {token: (amount, limit)} or (tokens, amounts,
        limits) (1 to 16 distinct 1-based tokens, none of them token_out[r]).  Each entry sells up to its
        amount for as long as the margin pays at least `limit` of token_out[r] per unit, over every pool
        among the row's tokens and the tokens t with allowed[t - 1], one dual solve per row on the device
        (cfmm_quote_limit_orders); rows fill partially.  To buy with a budget, settle in the bought token
        and sell the budget token at limit 1 / (the highest price per unit bought).  No state changes.
        Returns (sold per entry as a list of arrays in the caller's order, received [q], surplus [q],
        status [q], detail); detail is DevicePools.quote_limit_orders' namespace.  Single GPU.  allowed may
        instead be one list of 1-based tokens per row (choose_hubs' output as it is): each row then runs
        over its own list, as the call with that list as its mask (the *_rows calls)."""
        tout, off, toks, amts, lims, _ = self._limit_args(token_out, sells, allowed, None, "quote_limit_orders")
        out = self._pools.quote_limit_orders(tout, off, toks, amts, lims, allowed, opts)
        return self._per_entry(out), out.received, out.surplus, out.status, out

    def execute_limit_orders(self, token_out, sells, allowed, min_received=None, opts=None):
        """Execute limit orders in order (cfmm_execute_limit_orders), each re-solved on the state the
        earlier filled rows left, with an optional minimum received per row: a row below it reverts.
        Returns what quote_limit_orders returns and refreshes the pool objects the filled rows traded
        with from the device state.  Single GPU."""
        tout, off, toks, amts, lims, min_received = self._limit_args(token_out, sells, allowed, min_received,
                                                                     "execute_limit_orders")
        out = self._pools.execute_limit_orders(tout, off, toks, amts, lims, allowed, min_received, opts)
        self._refresh_filled(out)
        return self._per_entry(out), out.received, out.surplus, out.status, out

    def _price_arb_args(self, prices, allowed, what):
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        if allowed is None:
            raise ValueError(f"{what}: allowed (a mask over the tokens) is required")
        prices = np.asarray(prices, dtype=np.float64)
        return prices.reshape(1, -1) if prices.ndim == 1 else prices

    def quote_price_arbitrage(self, prices, allowed, opts=None):
        """The best trades through every pool among each row's priced tokens against external prices:
        prices[r] gives one price per token t with allowed[t - 1], ascending (0 leaves a token out of
        the row; a 1-D array is one row).  Each row maximises Σ price·Ψ with no token's net negative,
        route! with LinearNonnegative over those pools, one dual solve per row on the device
        (cfmm_quote_price_arbitrage).  No state changes.  Returns (profit [q], status [q], detail):
        detail is DevicePools.quote_price_arbitrage's namespace.  Single GPU."""
        out = self._pools.quote_price_arbitrage(self._price_arb_args(prices, allowed, "quote_price_arbitrage"),
                                                allowed, opts)
        return out.profit, out.status, out

    def execute_price_arbitrage(self, prices, allowed, min_profit=None, opts=None):
        """Execute price arbitrage rows in order (cfmm_execute_price_arbitrage), each re-solved on the
        state the earlier filled rows left, with an optional minimum profit: a row below it reverts.
        Returns what quote_price_arbitrage returns and refreshes the pool objects the filled rows traded
        with from the device state.  Single GPU."""
        out = self._pools.execute_price_arbitrage(self._price_arb_args(prices, allowed, "execute_price_arbitrage"),
                                                  allowed, min_profit, opts)
        self._refresh_filled(out)
        return out.profit, out.status, out

    def _inventory_args(self, tokens, prices, holdings, what):
        """(allow_off, allow_token, price, holding) from one token list per row and one price (and
        holding) list per row aligned with it."""
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        if not is_row_lists(tokens):
            raise ValueError(f"{what}: tokens must be one list of 1-based tokens per row")
        q = len(tokens)
        off, tok = pack_row_lists(tokens, len(self.v), [[]] * q, [_lib.PRICE_ARB_MAX_TOKENS] * q, what)

        def aligned(vals, name):
            if len(vals) != q or any(len(np.atleast_1d(v)) != len(t) for v, t in zip(vals, tokens)):
                raise ValueError(f"{what}: {name} needs one list per row, aligned with its tokens")
            return np.concatenate([np.asarray(v, dtype=np.float64).reshape(-1) for v in vals]) if q else np.zeros(0)
        return off, tok, aligned(prices, "prices"), None if holdings is None else aligned(holdings, "holdings")

    def quote_inventory_arbitrage(self, tokens, prices, holdings=None, opts=None):
        """The best trades against external prices from inventory: row r lists tokens[r] (1-based,
        distinct, 1 to 258) with prices[r] and holdings[r] aligned with it (holdings None: nothing
        held).  Each row maximises Σ price·Ψ over every pool among its tokens, where a token's net may
        spend up to its holding (route! with cᵀΨ − I(Ψ + h >= 0)), one dual solve per row on the device
        (cfmm_quote_price_arbitrage_rows).  opts as DevicePools.quote_price_arbitrage_rows, "atol"
        included.  No state changes.  Returns (profit [q], status [q], detail): detail is
        DevicePools.quote_price_arbitrage_rows' namespace.  Single GPU."""
        off, tok, pr, h = self._inventory_args(tokens, prices, holdings, "quote_inventory_arbitrage")
        out = self._pools.quote_price_arbitrage_rows(off, tok, pr, h, opts)
        return out.profit, out.status, out

    def execute_inventory_arbitrage(self, tokens, prices, holdings=None, min_profit=None, opts=None):
        """Execute inventory arbitrage rows in order (cfmm_execute_price_arbitrage_rows), each re-solved
        on the state the earlier filled rows left, with an optional minimum profit: a row below it
        reverts.  Returns what quote_inventory_arbitrage returns and refreshes the pool objects the
        filled rows traded with from the device state.  Single GPU."""
        off, tok, pr, h = self._inventory_args(tokens, prices, holdings, "execute_inventory_arbitrage")
        out = self._pools.execute_price_arbitrage_rows(off, tok, pr, h, min_profit, opts)
        self._refresh_filled(out)
        return out.profit, out.status, out

    def _arbitrage_args(self, base, other, hubs, min_profit, what):
        if self._world > 1:
            raise NotImplementedError(f"{what} drives one GPU")
        base, other = np.asarray(base).reshape(-1), np.asarray(other).reshape(-1)
        if len(base) != len(other):
            raise ValueError(f"{what}: base and other need one entry per row")
        q = len(base)
        if isinstance(hubs, tuple) and len(hubs) == 2:  # (hub_off, hubs) as scan_arbitrage returns them
            hub_off, flat = (np.asarray(x, dtype=np.int64).reshape(-1) for x in hubs)
        else:
            per_row = [list(hubs)] * q if all(np.ndim(h) == 0 for h in hubs) else [list(h) for h in hubs]
            if len(per_row) != q:
                raise ValueError(f"{what}: hubs must be one list, or one list per row ({q})")
            hub_off = np.concatenate([[0], np.cumsum([len(h) for h in per_row])]).astype(np.int64)
            flat = np.array([int(x) for h in per_row for x in h], dtype=np.int64)
        if min_profit is not None:
            min_profit = np.asarray(min_profit, dtype=np.float64).reshape(-1)
            if len(min_profit) != q:
                raise ValueError(f"{what}: min_profit must have {q} entries")
        return base, other, hub_off, flat, min_profit

    def scan_arbitrage(self, base, min_profit, max_hubs: int = _lib.ROUTE_MAX_HUBS):
        """Find the arbitrage cycles that start and end in one of the base tokens (1-based, distinct):
        two pools of one pair that disagree (p → x → p) and triangles (p → x → y → p), each row (p, x)
        sized optimally over its pair's pools and up to max_hubs triangles (cfmm_scan_arbitrage).  Keeps
        the rows whose profit reaches min_profit (one value, or one per base token, in units of that
        base token), ordered by (base, profit descending, x).  No state changes.  Returns (row_base [n],
        row_other [n], (hub_off [n + 1], hubs [Σ]), profit [n], price [n]); pass the first three to
        execute_arbitrage with the minimum profits to close them.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("scan_arbitrage drives one GPU")
        _, rb, ro, hub_off, hubs, profit, price = self._pools.scan_arbitrage(base, min_profit, max_hubs)
        return rb, ro, (hub_off, hubs), profit, price

    def quote_arbitrage(self, base, other, hubs):
        """Size the cycles from base[j] through other[j] and back, directly and through each hub of
        `hubs` (one list for every row, one list per row, or (hub_off, hubs) as scan_arbitrage returns
        them), as route! with BasketLiquidation(base, 0) over the row's pools (cfmm_quote_arbitrage).
        Every row on the current state on its own.  Returns (profit [q], surplus_in [q], price [q],
        status [q]).  Single GPU."""
        base, other, off, flat, _ = self._arbitrage_args(base, other, hubs, None, "quote_arbitrage")
        return self._pools.quote_arbitrage(base, other, off, flat)[:4]

    def execute_arbitrage(self, base, other, hubs, min_profit=None):
        """Run arbitrage rows in order (cfmm_execute_arbitrage), each re-solved on the state the earlier
        rows left; a row whose profit is below min_profit[j] (None: 0) reverts.  Returns what
        quote_arbitrage returns and refreshes the pool objects of the filled rows' pairs from the
        device state, as execute_routed_orders does.  Single GPU."""
        base, other, off, flat, min_profit = self._arbitrage_args(base, other, hubs, min_profit, "execute_arbitrage")
        out = self._pools.execute_arbitrage(base, other, off, flat, min_profit)[:4]
        filled = np.flatnonzero(out[3] == _lib.ORDER_FILLED)
        if len(filled):
            sub = np.concatenate([[0], np.cumsum(np.diff(off)[filled])]).astype(np.int64)
            fh = np.concatenate([flat[off[r]:off[r + 1]] for r in filled]).astype(np.int64)
            a, b, _ = DevicePools.route_pairs(other[filled], base[filled], sub, fh)
            _, typ, idx, _ = self._pools.pair_pools(a, b)
            self._refresh_swapped([(t, None, idx[typ == t]) for t in (0, 1, 2) if np.any(typ == t)])
        return out

    def _refresh_swapped(self, groups):
        """The touched pool objects' R, or current_price / current_tick, from the device state."""
        for t, rows, loc in groups:
            touched = np.unique(loc)
            lo, hi = int(touched[0]), int(touched[-1]) + 1
            state, _ = self._pools.pool_state(t, lo, hi - lo)
            lst = self._type_lists[t]
            for k in touched:
                c = self.cfmms[lst[k]]
                if t == _lib.POOL_UNIV3:
                    c.current_price = float(state[k - lo])
                    c.current_tick = int(np.sum(c.lower_ticks >= c.current_price))
                else:
                    c.R = state[k - lo].copy()

    def modify_liquidity(self, list_indices, lo, hi, dL):
        """Mint (dL > 0) or burn (dL < 0) liquidity on the price range (lo[j], hi[j]] of the UniV3
        pool r.cfmms[list_indices[j]], rows in order (cfmm_modify_univ3_liquidity): boundaries that
        are new to a pool's ladder are inserted, and a row that would leave a tick below zero
        rejects the whole call.  Refreshes the touched pool objects (lower_ticks, liquidity,
        current_tick) from the device state.  Single GPU."""
        if self._world > 1:
            raise NotImplementedError("modify_liquidity drives one GPU")
        ids = np.asarray(list_indices, dtype=np.int64).reshape(-1)
        lo, hi, dL = (np.asarray(x, dtype=np.float64).reshape(-1) for x in (lo, hi, dL))
        if not (len(ids) == len(lo) == len(hi) == len(dL)):
            raise ValueError("modify_liquidity: list_indices, lo, hi, dL must have one entry per row")
        if len(ids) and (ids.min() < 0 or ids.max() >= len(self.cfmms)):
            raise IndexError("modify_liquidity: pool index out of range")
        lst = np.asarray(self._type_lists[2], dtype=np.int64)
        local = np.full(len(self.cfmms), -1, dtype=np.int64)
        local[lst] = np.arange(len(lst))
        loc = local[ids]
        if np.any(loc < 0):
            raise TypeError(f"modify_liquidity: r.cfmms[{int(ids[np.argmax(loc < 0)])}] is not a UniV3 pool")
        self._pools.modify_univ3_liquidity(loc, lo, hi, dL)
        if not len(ids):
            return
        touched = np.unique(loc)
        first = int(touched[0])
        off, lt, lq = self._pools.univ3_ticks(first, int(touched[-1]) + 1 - first)
        for k in touched:
            c = self.cfmms[lst[k]]
            s = slice(off[k - first], off[k - first + 1])
            c.lower_ticks, c.liquidity = lt[s].copy(), lq[s].copy()
            c.current_tick = int(np.sum(c.lower_ticks >= c.current_price))

    # one find_arb!(r, v) + folds; caches Ψ and acc like the reference caches Δs/Λs
    def _sweep(self, v, materialize=False):
        psi, acc = self._pools.sweep(v, materialize)
        if self._world > 1 and not self._pools.peer_attached:
            import torch
            import torch.distributed as dist
            buf = torch.from_numpy(np.append(psi, acc))
            if dist.get_backend(self._group) == "nccl":  # NCCL reduces device tensors only
                buf = buf.to(torch.device("cuda", self._pools.device))
            dist.all_reduce(buf, group=self._group)
            out = buf.cpu().numpy()
            psi, acc = out[:-1].copy(), float(out[-1])
        self._psi, self._acc = psi, acc
        if materialize:
            self._v_mat = np.array(v, dtype=np.float64)
            self._fetch_trades()

    def _fetch_trades(self):
        """r.Δs / r.Λs <- the trades of the last materialising sweep, in list order."""
        if True:
            D, L = self._pools.trades()
            Dl = np.zeros_like(D)
            Ll = np.zeros_like(L)
            Dl[self._order] = D
            Ll[self._order] = L
            if self._world > 1:
                import torch
                import torch.distributed as dist
                # shards are contiguous in list order: gather them back
                parts = [None] * self._world
                dist.all_gather_object(parts, (Dl, Ll), group=self._group)
                Dl = np.concatenate([q[0] for q in parts])
                Ll = np.concatenate([q[1] for q in parts])
            n = len(self.Δs)
            self.Δs[:] = Dl[:n]
            self.Λs[:] = Ll[:n]

    def sync_reserves(self):
        """Push the state of every pool to the device: cfmm.R of the Product/GeoMean pools,
        current_price and liquidity of the UniV3 pools (the reference reads the pool objects
        live on each sweep; call this after mutating them).  A UniV3 pool's tick prices are the
        device's current ladder: those of construction, grown by modify_liquidity (which keeps the
        pool objects in step).  Assigning other lower_ticks to a pool object does not move the
        device's boundaries; use modify_liquidity for that."""
        shard = self.cfmms[self._lo:self._hi]
        for t in (0, 1):
            ids = self._type_lists[t]
            if ids:
                self._pools.update_reserves(t, 0, np.array([shard[i].R for i in ids]))
        ids = self._type_lists[2]
        if ids:
            cs = [shard[i] for i in ids]
            self._pools.update_univ3(0, np.array([c.current_price for c in cs]),
                                     np.concatenate([c.liquidity for c in cs]))


def find_arb(*args):
    """find_arb!(r::Router, v) (src/router.jl:38-42) or
    find_arb!(Δ, Λ, cfmm, v) (src/cfmms.jl:130, 185, 339).  Both run on the GPU."""
    if len(args) == 2 and isinstance(args[0], Router):
        r, v = args
        r._sweep(np.asarray(v, dtype=np.float64), materialize=True)
        return None
    if len(args) == 4:
        D, L, cfmm, v = args
        if not isinstance(cfmm, CFMM):
            raise TypeError("find_arb!(Δ, Λ, cfmm, v): cfmm must be a CFMM")
        v = np.asarray(v, dtype=np.float64)
        if v.shape != (2,):
            raise ValueError("v must have length 2 (the prices of the pool's two tokens)")
        one = type(cfmm).__new__(type(cfmm))
        one.__dict__.update(cfmm.__dict__)
        one.Ai = np.array([1, 2], dtype=np.int64)
        r = Router(_NoObjective(), [one], 2)
        r._sweep(v, materialize=True)
        D[:] = r.Δs[0]
        L[:] = r.Λs[0]
        r._pools.close()
        return None
    raise TypeError("find_arb(r, v) or find_arb(Δ, Λ, cfmm, v)")


class _NoObjective(Objective):
    pass


def route(r: Router, v=None, verbose=False, m=5, factr=1e1, pgtol=1e-5,
          maxfun=15_000, maxiter=15_000, optimizer="host"):
    """route!(r; v, verbose, m, factr, pgtol, maxfun, maxiter) (src/router.jl:58-108).
    Overwrites r.Δs, r.Λs and r.v.

    optimizer="host" (default): L-BFGS-B on the host (scipy), one device sweep per function /
    gradient evaluation, as in the reference.  optimizer="device": the whole outer iteration runs
    on the GPU (cfmm_solve: projected L-BFGS, m = 5; objectives of the form linᵀν on a box, which
    both reference objectives are) and only scalars cross PCIe per evaluation; single GPU."""
    if optimizer == "device":
        lin = r.objective.linear_term()
        if lin is None:
            raise TypeError("the device solver needs an objective with linear_term()")
        if r._world > 1:
            raise NotImplementedError("optimizer='device' drives one GPU")
        n = len(r.v)
        x, info = r._pools.solve(r.objective.lower_limit(), lin=lin, upper=r.objective.upper_limit(),
                                 v0=None if v is None else np.asarray(v, dtype=np.float64),
                                 pgtol=pgtol, factr=factr, maxfun=maxfun, maxiter=maxiter)
        r.v[:] = x
        r._v_mat = x.copy()
        r._fetch_trades()
        r.last_result = info
        return None
    from scipy.optimize import minimize

    n = len(r.v)
    if v is None:
        r.v[:] = np.ones(n) / n  # router.jl:61
    else:
        r.v[:] = v
    lower = np.asarray(r.objective.lower_limit(), dtype=np.float64)
    upper = np.asarray(r.objective.upper_limit(), dtype=np.float64)
    bounds = [(lo if np.isfinite(lo) else None, up if np.isfinite(up) else None)
              for lo, up in zip(lower, upper)]

    def fn(x):  # router.jl:73-86
        if not np.array_equal(x, r.v):
            r._sweep(x)
            r.v[:] = x
        return r.objective.f(x) + r._acc

    def g(x):  # router.jl:89-102
        G = np.zeros(n)
        if not np.array_equal(x, r.v):
            r._sweep(x)
            r.v[:] = x
        r.objective.grad(G, x)
        G += r._psi  # G[c.Ai] .+= Λ .- Δ over all pools
        return G

    r._sweep(r.v)  # find_arb!(r, r.v), router.jl:104
    res = minimize(fn, r.v.copy(), jac=g, method="L-BFGS-B", bounds=bounds,
                   options=dict(maxcor=m, ftol=factr * np.finfo(np.float64).eps, gtol=pgtol,
                                maxfun=maxfun, maxiter=maxiter,
                                **({"iprint": 1} if verbose else {})))
    r.v[:] = res.x  # router.jl:106
    r._sweep(r.v, materialize=True)  # find_arb!(r, v), router.jl:107
    r.last_result = res
    return None


def netflows_(psi, r: Router):
    """netflows!(ψ, r) (src/router.jl:111-119): serial pool-order sum of the
    stored trades on the host (the reference's tests compare it for exact
    equality with another pool-order sum, test/arb.jl:16)."""
    psi[:] = 0.0
    for D, L, c in zip(r.Δs, r.Λs, r.cfmms):
        psi[c.Ai - 1] += L - D
    return None


def netflows(r: Router):
    psi = np.zeros_like(r.v)
    netflows_(psi, r)
    return psi


def univ3_moved_price(c: UniV3, v):
    """The price a UniV3 pool moves to when it trades at ν = v (include/cfmm_b200.h,
    cfmm_apply_trades): p = v[a]/v[b]; unchanged inside the no-trade band γq <= p <= q/γ,
    else min(p/γ, T₁) (upper walk, p < γq) or min(γp, T₁) (lower walk), unchanged if that
    target is NaN or not > 0.  The same IEEE operations as the device kernel: bit-identical."""
    with np.errstate(all="ignore"):
        q, g = np.float64(c.current_price), np.float64(c.gamma)
        p = np.float64(v[c.Ai[0] - 1]) / np.float64(v[c.Ai[1] - 1])
        lo = g * q
        if lo <= p and p <= q / g:
            return float(q)
        target = p / g if p < lo else g * p
        if not target > 0.0:
            return float(q)
        t1 = np.float64(c.lower_ticks[0])
        return float(target if target < t1 else t1)


def update_reserves(r: Router):
    """A working update_reserves!(r) (the reference's, src/router.jl:127-132,
    calls a per-CFMM method that is defined nowhere), on the host objects and on
    the device: R ← R + γΔ − Λ for the two-coin pools (test/cfmms.jl:10); a UniV3
    pool moves to the price its arbitrage walk traded it to (univ3_moved_price, at
    the ν of the last materialising sweep), with current_tick re-derived as the
    constructor does.  Retired pools (Router.set_active) are left unchanged."""
    v = getattr(r, "_v_mat", None)
    if v is None:
        v = r.v
    for D, L, c, retired in zip(r.Δs, r.Λs, r.cfmms, r._retired):
        if retired:  # retired pools keep their state (cfmm_set_active)
            continue
        if isinstance(c, (ProductTwoCoin, GeometricMeanTwoCoin)):
            c.R = c.R + c.gamma * D - L  # same operation order as the device kernel: bit-identical
        elif isinstance(c, UniV3):
            c.current_price = univ3_moved_price(c, v)
            c.current_tick = int(np.sum(c.lower_ticks >= c.current_price))
    r._pools.apply_trades()  # on the device, from the materialised trades: no upload
    return None
