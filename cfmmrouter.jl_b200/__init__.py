"""cfmmrouter.jl_b200 -- GPU-native dual-decomposition inner loop of
CFMMRouter.jl: the per-pool find_arb! sweep and the Ψ/acc folds of route!'s
L-BFGS-B callback run as hand-written sm_90a (H100) CUDA kernels behind the C ABI of
include/cfmm_b200.h; this package is the Python host-side mirror of the
reference's Router / route! / CFMM / Objective interface.

(The directory name contains a dot, so import it through the loader module at
the repo root:  `import cfmmrouter_b200 as cr`.)
"""
from ._lib import CFMMError, LIB_PATH, load as load_library
from .cfmms import CFMM, GeometricMeanTwoCoin, ProductTwoCoin, UniV3
from .objectives import (BasketLiquidation, BasketSwap, LimitBasket, LinearHoldings, LinearNonnegative, Objective,
                         Swap)
from .router import (DevicePools, Router, find_arb, netflows, netflows_, pool_file_info, route,
                     shard_range, update_reserves, write_pool_file)

__all__ = [
    "CFMM", "ProductTwoCoin", "GeometricMeanTwoCoin", "UniV3",
    "Objective", "LinearNonnegative", "LinearHoldings", "BasketLiquidation", "BasketSwap", "LimitBasket", "Swap",
    "Router", "route", "find_arb", "netflows", "netflows_", "update_reserves",
    "DevicePools", "shard_range", "write_pool_file", "pool_file_info", "CFMMError", "LIB_PATH", "load_library",
]
