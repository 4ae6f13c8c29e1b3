"""ctypes binding of libcfmm_b200.so (the C ABI declared in include/cfmm_b200.h).

The library is the product; this module only loads it.  There is no Python or
CPU fallback: if the shared object is missing, or no CUDA device is visible when
a context is created, the failure is raised to the caller.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# CFMM_B200_LIB: development override (A/B runs of two builds of the same ABI on one box)
LIB_PATH = os.environ.get("CFMM_B200_LIB") or os.path.join(_HERE, "libcfmm_b200.so")

CFMM_OK = 0
CFMM_ERR_INVALID = -1
CFMM_ERR_CUDA = -2
CFMM_ERR_STATE = -3
CFMM_ERR_NOMEM = -4
CFMM_ERR_COMM = -5

POOL_PRODUCT = 0
POOL_GEOMEAN = 1
POOL_UNIV3 = 2

# cfmm_execute_swap_orders: row kinds and per-row status
SWAP_EXACT_IN = 0
SWAP_EXACT_OUT = 1
ORDER_FILLED = 0
ORDER_LIMIT = 1
ORDER_UNREACHABLE = 2
ORDER_RETIRED = 3
# cfmm_quote_paths / cfmm_execute_paths
PATH_MAX_HOPS = 8
ROUTE_MAX_HUBS = 7  # CFMM_ROUTE_MAX_HUBS
# cfmm_find_order_paths
BEST_PATH_MAX_TOKENS = 1024
PATH_REPEATS_POOL = 4
# cfmm_quote_subgraph_(swap_)orders / cfmm_execute_subgraph_(swap_)orders
SUBGRAPH_MAX_TOKENS = 256
ORDER_NOT_CONVERGED = 5
# cfmm_quote_basket_(swap_)orders / cfmm_execute_basket_(swap_)orders, cfmm_quote/execute_limit_orders
BASKET_MAX_TOKENS = 16
# cfmm_quote_price_arbitrage / cfmm_execute_price_arbitrage
PRICE_ARB_MAX_TOKENS = SUBGRAPH_MAX_TOKENS + 2

COMM_HANDLE_BYTES = 128

class SolveOpts(C.Structure):
    _fields_ = [("max_iter", C.c_int), ("max_fun", C.c_int), ("pgtol", C.c_double), ("factr", C.c_double)]


class SolveInfo(C.Structure):
    _fields_ = [("iterations", C.c_int), ("fun_evals", C.c_int), ("status", C.c_int),
                ("f", C.c_double), ("pg_norm", C.c_double), ("solve_ms", C.c_double)]


class SubgraphOpts(C.Structure):
    _fields_ = [("max_iter", C.c_int), ("max_fun", C.c_int), ("rtol", C.c_double), ("factr", C.c_double)]


class PriceArbOpts(C.Structure):
    """cfmm_price_arb_opts: cfmm_subgraph_opts' fields, plus the absolute stop atol."""
    _fields_ = SubgraphOpts._fields_ + [("atol", C.c_double)]


class SubgraphOut(C.Structure):
    _fields_ = [("paid", C.POINTER(C.c_double)), ("received", C.POINTER(C.c_double)),
                ("status", C.POINTER(C.c_uint8)), ("solver_status", C.POINTER(C.c_int)),
                ("iterations", C.POINTER(C.c_int)), ("fun_evals", C.POINTER(C.c_int)),
                ("merit", C.POINTER(C.c_double)), ("tok_off", C.POINTER(C.c_int64)), ("tok_cap", C.c_int64),
                ("token", C.POINTER(C.c_int64)), ("nu", C.POINTER(C.c_double)), ("psi", C.POINTER(C.c_double)),
                ("leg_off", C.POINTER(C.c_int64)), ("leg_cap", C.c_int64), ("leg_type", C.POINTER(C.c_int)),
                ("leg_pool", C.POINTER(C.c_int64)), ("leg_delta", C.POINTER(C.c_double)),
                ("leg_lambda", C.POINTER(C.c_double))]


class BasketOut(SubgraphOut):
    """cfmm_basket_out: cfmm_subgraph_out's fields, with paid per basket entry."""


class LimitOut(C.Structure):
    """cfmm_limit_out: cfmm_basket_out's fields, plus the surplus per row."""
    _fields_ = SubgraphOut._fields_ + [("surplus", C.POINTER(C.c_double))]


class PriceArbOut(C.Structure):
    """cfmm_price_arb_out: cfmm_subgraph_out's fields, with the profit for paid and received."""
    _fields_ = [("profit", C.POINTER(C.c_double))] + SubgraphOut._fields_[2:]


# every symbol include/cfmm_b200.h declares: name -> (restype, argtypes)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int64)
_ctx = C.c_void_p
SYMBOLS = {
    "cfmm_create": (C.c_int, [C.POINTER(_ctx), C.c_int, C.c_int64]),
    "cfmm_destroy": (None, [_ctx]),
    "cfmm_last_error": (C.c_char_p, [_ctx]),
    "cfmm_version": (C.c_char_p, []),
    "cfmm_add_product": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip]),
    "cfmm_add_geomean": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip, _dp]),
    "cfmm_add_univ3": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip, _ip, _dp, _dp]),
    "cfmm_pool_file_write": (C.c_int, [C.c_char_p, C.c_int, C.c_int64, C.c_int64, _dp, _dp, _ip, _dp]),
    "cfmm_pool_file_info": (C.c_int, [C.c_char_p, C.POINTER(C.c_int), _ip, _ip]),
    "cfmm_add_pool_file": (C.c_int, [_ctx, C.c_char_p]),
    "cfmm_finalize": (C.c_int, [_ctx]),
    "cfmm_num_pools": (C.c_int64, [_ctx]),
    "cfmm_num_tokens": (C.c_int64, [_ctx]),
    "cfmm_sweep": (C.c_int, [_ctx, _dp, _dp, _dp, C.c_int]),
    "cfmm_sweep_device": (C.c_int, [_ctx, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "cfmm_sweep_device_view": (C.c_int, [_ctx, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "cfmm_get_trades": (C.c_int, [_ctx, _dp, _dp]),
    "cfmm_solve": (C.c_int, [_ctx, _dp, _dp, _dp, _dp, C.POINTER(SolveOpts), _dp, C.POINTER(SolveInfo)]),
    "cfmm_update_reserves": (C.c_int, [_ctx, C.c_int, C.c_int64, C.c_int64, _dp]),
    "cfmm_update_univ3": (C.c_int, [_ctx, C.c_int64, C.c_int64, _dp, _dp]),
    "cfmm_apply_trades": (C.c_int, [_ctx]),
    "cfmm_append_product": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip]),
    "cfmm_append_geomean": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip, _dp]),
    "cfmm_append_univ3": (C.c_int, [_ctx, C.c_int64, _dp, _dp, _ip, _ip, _dp, _dp]),
    "cfmm_set_active": (C.c_int, [_ctx, C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_uint8)]),
    "cfmm_get_pool_state": (C.c_int, [_ctx, C.c_int, C.c_int64, C.c_int64, _dp, C.POINTER(C.c_uint8)]),
    "cfmm_compact": (C.c_int, [_ctx]),
    "cfmm_quote_swaps": (C.c_int, [_ctx, C.c_int, C.c_int64, _ip, _dp, _dp]),
    "cfmm_execute_swaps": (C.c_int, [_ctx, C.c_int, C.c_int64, _ip, _dp, _dp]),
    "cfmm_quote_swaps_exact_out": (C.c_int, [_ctx, C.c_int, C.c_int64, _ip, _dp, _dp]),
    "cfmm_execute_swap_orders": (C.c_int, [_ctx, C.c_int, C.c_int64, _ip, C.POINTER(C.c_uint8), _dp, _dp, _dp, _dp,
                                           C.POINTER(C.c_uint8)]),
    "cfmm_quote_paths": (C.c_int, [_ctx, C.c_int64, _ip, C.POINTER(C.c_int), _ip, _ip, C.POINTER(C.c_uint8), _dp,
                                   _dp, _dp, C.POINTER(C.c_uint8)]),
    "cfmm_execute_paths": (C.c_int, [_ctx, C.c_int64, _ip, C.POINTER(C.c_int), _ip, _ip, C.POINTER(C.c_uint8), _dp,
                                     _dp, _dp, _dp, C.POINTER(C.c_uint8)]),
    "cfmm_pair_pools": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, C.c_int64, C.POINTER(C.c_int), _ip,
                                  C.POINTER(C.c_uint8)]),
    "cfmm_quote_split_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp, _dp, _dp,
                                          C.POINTER(C.c_uint8), _dp, _dp]),
    "cfmm_execute_split_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp, _dp, _dp,
                                            _dp, C.POINTER(C.c_uint8), _dp, _dp]),
    "cfmm_quote_routed_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _ip, _ip, _dp, _dp,
                                           _dp, C.POINTER(C.c_uint8), _dp, _dp, _dp, _dp]),
    "cfmm_execute_routed_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp, _ip, _ip, _dp,
                                             _dp, _dp, C.POINTER(C.c_uint8), _dp, _dp, _dp, _dp]),
    "cfmm_quote_arbitrage": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _ip, _dp, _dp, _dp, C.POINTER(C.c_uint8), _dp,
                                       _dp, _dp, _dp]),
    "cfmm_execute_arbitrage": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _dp, _ip, _ip, _dp, _dp, _dp, C.POINTER(C.c_uint8),
                                         _dp, _dp, _dp, _dp]),
    "cfmm_scan_arbitrage": (C.c_int, [_ctx, C.c_int64, _ip, _dp, C.c_int, C.c_int64, _ip, _ip, _ip, _ip, _ip, _dp,
                                      _dp]),
    "cfmm_choose_order_hubs": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, C.c_int,
                                         C.POINTER(C.c_uint8), _ip, _ip, _dp, _ip]),
    "cfmm_find_order_paths": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, C.c_int,
                                        C.POINTER(C.c_uint8), _ip, C.POINTER(C.c_int), _ip, _ip, _dp, _dp, _dp,
                                        C.POINTER(C.c_uint8)]),
    "cfmm_quote_token_values": (C.c_int, [_ctx, C.c_int64, _ip, C.POINTER(C.c_uint8), _dp, C.c_int,
                                          C.POINTER(C.c_uint8), _dp, C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), _ip,
                                          C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_int), _ip, _ip, _dp, _dp,
                                          C.POINTER(C.c_uint8)]),
    "cfmm_find_order_paths_net": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, C.c_int,
                                            C.POINTER(C.c_uint8), _dp, _ip, C.POINTER(C.c_int), _ip, _ip, _dp, _dp,
                                            _dp, C.POINTER(C.c_uint8), _dp]),
    "cfmm_quote_token_values_net": (C.c_int, [_ctx, C.c_int64, _ip, C.POINTER(C.c_uint8), _dp, C.c_int,
                                              C.POINTER(C.c_uint8), _dp, _dp, C.POINTER(C.c_uint8),
                                              C.POINTER(C.c_uint8), _dp, _ip, C.c_int64, _ip, _ip, _ip,
                                              C.POINTER(C.c_int), _ip, _ip, _dp, _dp, C.POINTER(C.c_uint8)]),
    "cfmm_quote_subgraph_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _dp, C.POINTER(C.c_uint8),
                                             C.POINTER(SubgraphOpts), C.POINTER(SubgraphOut)]),
    "cfmm_execute_subgraph_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _dp, _dp, C.POINTER(C.c_uint8),
                                               C.POINTER(SubgraphOpts), C.POINTER(SubgraphOut)]),
    "cfmm_quote_subgraph_swap_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp,
                                                  C.POINTER(C.c_uint8), C.POINTER(SubgraphOpts),
                                                  C.POINTER(SubgraphOut)]),
    "cfmm_execute_subgraph_swap_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp,
                                                    C.POINTER(C.c_uint8), C.POINTER(SubgraphOpts),
                                                    C.POINTER(SubgraphOut)]),
    "cfmm_quote_basket_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, C.POINTER(C.c_uint8),
                                           C.POINTER(SubgraphOpts), C.POINTER(BasketOut)]),
    "cfmm_execute_basket_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, _dp, C.POINTER(C.c_uint8),
                                             C.POINTER(SubgraphOpts), C.POINTER(BasketOut)]),
    "cfmm_quote_basket_swap_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_uint8), _dp,
                                                C.POINTER(C.c_uint8), C.POINTER(SubgraphOpts), C.POINTER(BasketOut)]),
    "cfmm_execute_basket_swap_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp,
                                                  C.POINTER(C.c_uint8), C.POINTER(SubgraphOpts),
                                                  C.POINTER(BasketOut)]),
    "cfmm_quote_limit_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, _dp, C.POINTER(C.c_uint8),
                                          C.POINTER(SubgraphOpts), C.POINTER(LimitOut)]),
    "cfmm_execute_limit_orders": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, _dp, _dp, C.POINTER(C.c_uint8),
                                            C.POINTER(SubgraphOpts), C.POINTER(LimitOut)]),
    "cfmm_quote_subgraph_swap_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _ip, _ip,
                                                       C.POINTER(SubgraphOpts), C.POINTER(SubgraphOut)]),
    "cfmm_execute_subgraph_swap_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, C.POINTER(C.c_uint8), _dp, _dp,
                                                         _ip, _ip, C.POINTER(SubgraphOpts), C.POINTER(SubgraphOut)]),
    "cfmm_quote_basket_swap_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_uint8), _dp, _ip,
                                                     _ip, C.POINTER(SubgraphOpts), C.POINTER(BasketOut)]),
    "cfmm_execute_basket_swap_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, C.POINTER(C.c_uint8), _dp,
                                                       _dp, _ip, _ip, C.POINTER(SubgraphOpts), C.POINTER(BasketOut)]),
    "cfmm_quote_limit_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, _dp, _ip, _ip,
                                               C.POINTER(SubgraphOpts), C.POINTER(LimitOut)]),
    "cfmm_execute_limit_orders_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _ip, _dp, _dp, _dp, _ip, _ip,
                                                 C.POINTER(SubgraphOpts), C.POINTER(LimitOut)]),
    "cfmm_quote_price_arbitrage": (C.c_int, [_ctx, C.c_int64, _dp, C.POINTER(C.c_uint8), C.POINTER(SubgraphOpts),
                                             C.POINTER(PriceArbOut)]),
    "cfmm_execute_price_arbitrage": (C.c_int, [_ctx, C.c_int64, _dp, _dp, C.POINTER(C.c_uint8),
                                               C.POINTER(SubgraphOpts), C.POINTER(PriceArbOut)]),
    "cfmm_quote_price_arbitrage_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _dp, _dp, C.POINTER(PriceArbOpts),
                                                  C.POINTER(PriceArbOut)]),
    "cfmm_execute_price_arbitrage_rows": (C.c_int, [_ctx, C.c_int64, _ip, _ip, _dp, _dp, _dp,
                                                    C.POINTER(PriceArbOpts), C.POINTER(PriceArbOut)]),
    "cfmm_modify_univ3_liquidity":(C.c_int, [_ctx, C.c_int64, _ip, _dp, _dp]),
    "cfmm_get_univ3_ticks": (C.c_int, [_ctx, C.c_int64, C.c_int64, _ip, _dp, _dp]),
    "cfmm_debug_pool_set_info": (C.c_int, [_ctx, C.c_int, _ip]),
    "cfmm_debug_compact_record": (C.c_int, [_ctx, C.c_int, _ip]),
    "cfmm_debug_l2_keep": (C.c_int, [_ctx, C.c_int, _ip]),
    "cfmm_set_option": (C.c_int, [_ctx, C.c_char_p, C.c_int64]),
    "cfmm_last_sweep_ms": (C.c_int, [_ctx, C.POINTER(C.c_float)]),
    "cfmm_launch_count": (C.c_int64, [_ctx]),
    "cfmm_profile_read": (C.c_int, [_ctx, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "cfmm_profile_read_times": (C.c_int, [_ctx, C.c_int, C.POINTER(C.c_float), C.c_int64, C.POINTER(C.c_int64)]),
    "cfmm_profile_reset": (C.c_int, [_ctx]),
    "cfmm_selftest_inrange_math": (C.c_int, [_ctx, _dp, _dp, C.c_int64, _ip]),
    "cfmm_debug_product_layout": (C.c_int, [C.c_int64, C.c_int64, _ip, C.c_int, C.c_int, C.c_int64, _ip,
                                          C.POINTER(C.c_int32), C.POINTER(C.c_uint8), _ip]),
    "cfmm_debug_read_trace": (C.c_int, [_ctx, C.POINTER(C.c_uint64), C.c_int64, _ip]),
    "cfmm_host_alloc": (C.c_void_p, [C.c_size_t]),
    "cfmm_host_free": (None, [C.c_void_p]),
    "cfmm_comm_export": (C.c_int, [_ctx, C.c_void_p]),
    "cfmm_comm_attach": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_void_p]),
    "cfmm_comm_detach": (C.c_int, [_ctx]),
    "cfmm_comm_check": (C.c_int, [_ctx]),
}

_lib = None


class CFMMError(RuntimeError):
    """A non-zero status from libcfmm_b200 (the analogue of a Julia exception
    thrown by the reference: ArgumentError / BoundsError / MethodError)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"libcfmm_b200 error {code}: {message}")
        self.code = code
        self.message = message


def load():
    """Load libcfmm_b200.so once and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (nvcc, sm_90a).  There is no CPU fallback for the sweep.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(lib, ctx, rc: int):
    if rc != CFMM_OK:
        msg = lib.cfmm_last_error(ctx)
        raise CFMMError(rc, msg.decode() if msg else "")
