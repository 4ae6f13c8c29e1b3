// sweep_kernels.cuh -- the dual-gradient sweep kernels (sm_90a).
//
// One launch per pool type evaluates find_arb! for every pool of that type at
// the current dual price ν (src/router.jl:38-42) and folds the result into
//   psi[0..n)  += A_i (Λ_i − Δ_i)            (src/router.jl:98-100)
//   psi[n]     += ν[A_i]ᵀ(Λ_i − Δ_i)         (src/router.jl:79-83, "acc")
// without ever materialising Δ, Λ (unless MAT: the final sweep, router.jl:107).
//
// Data layout (per pool type, SoA, sorted by first token at finalize):
//   R   : double2[m]  (R1, R2)          16 B   one LDG.128 per pool
//   gam : double [m]                     8 B
//   Ai  : int2   [m]  0-based (a, b)     8 B   -> 32 B/pool for ProductTwoCoin
//   w   : double2[m]  (geomean only)    16 B   -> 48 B/pool
// Because pools are sorted by token a, a warp's 32 consecutive pools almost
// always share `a`: the Ψ[a] contribution is reduced inside the warp
// (shuffle) and leaves as ONE red.global.add.f64; the Ψ[b] contribution is a
// direct red.global.add.f64 (skipped when the pool does not trade).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arb_math.cuh"

namespace cfmm {

constexpr unsigned kFull = 0xffffffffu;

// streaming loads: read-only path, do not allocate in L1 (L1 is kept for ν)
__device__ __forceinline__ double2 ld_stream(const double2* p) {
  double2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
               : "=d"(r.x), "=d"(r.y)
               : "l"(p));
  return r;
}
__device__ __forceinline__ double ld_stream(const double* p) {
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ int2 ld_stream(const int2* p) {
  int2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0, %1}, [%2];"
               : "=r"(r.x), "=r"(r.y)
               : "l"(p));
  return r;
}

// fire-and-forget fp64 add (RED.E.ADD.F64)
__device__ __forceinline__ void red_add(double* addr, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(addr), "d"(v) : "memory");
}

__device__ __forceinline__ double shfl_xor_f64(double v, int m) {
  return __shfl_xor_sync(kFull, v, m);
}

// Reduce `val` over runs of equal `key` inside the warp and issue one RED per
// run.  Runs are contiguous because pools are sorted by key; the common case
// (whole warp one key) takes the butterfly path.
__device__ __forceinline__ void warp_segmented_red(double* __restrict__ psi,
                                                   int key, double val,
                                                   int lane) {
  const int k0 = __shfl_sync(kFull, key, 0);
  if (__all_sync(kFull, key == k0)) {
    val += shfl_xor_f64(val, 16);
    val += shfl_xor_f64(val, 8);
    val += shfl_xor_f64(val, 4);
    val += shfl_xor_f64(val, 2);
    val += shfl_xor_f64(val, 1);
    if (lane == 0 && val != 0.0 && k0 >= 0) red_add(psi + k0, val);
    return;
  }
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const double up = __shfl_up_sync(kFull, val, d);
    const int kup = __shfl_up_sync(kFull, key, d);
    if (lane >= d && kup == key) val += up;
  }
  const int knext = __shfl_down_sync(kFull, key, 1);
  const bool tail = (lane == 31) || (knext != key);
  if (tail && val != 0.0 && key >= 0) red_add(psi + key, val);
}

// ---- pool-type policies ----------------------------------------------------

struct ProductPools {
  const double2* R;
  const double* gam;
  const int2* Ai;
  struct Pool {
    double2 R;
    double g;
  };
  __device__ __forceinline__ Pool load(int64_t i) const {
    Pool p;
    p.R = ld_stream(R + i);
    p.g = ld_stream(gam + i);
    return p;
  }
  __device__ __forceinline__ Trade arb(const Pool& p, double v1, double v2,
                                       bool exact, bool) const {
    return product_arb(p.R.x, p.R.y, p.g, v1, v2, exact);
  }
};

// A ProductTwoCoin pool without reserves (padding, retired) trades nothing (product_arb) and adds no
// 0·ν terms to acc, which would be NaN at ν = ∞ or NaN.
template <class Pool>
__device__ __forceinline__ bool no_reserves(const Pool&) { return false; }
__device__ __forceinline__ bool no_reserves(const ProductPools::Pool& p) { return p.R.x == 0.0 && p.R.y == 0.0; }

struct GeomeanPools {
  const double2* R;
  const double* gam;
  const int2* Ai;
  const double2* w;
  struct Pool {
    double2 R, w;
    double g;
  };
  __device__ __forceinline__ Pool load(int64_t i) const {
    Pool p;
    p.R = ld_stream(R + i);
    p.w = ld_stream(w + i);
    p.g = ld_stream(gam + i);
    return p;
  }
  __device__ __forceinline__ Trade arb(const Pool& p, double v1, double v2,
                                       bool exact, bool econ) const {
    if (econ && !exact) return geomean_arb_econ(p.R.x, p.R.y, p.w.x, p.w.y, p.g, v1, v2);
    return geomean_arb(p.R.x, p.R.y, p.w.x, p.w.y, p.g, v1, v2, exact);
  }
};

// Same pools; gradient-only sweeps take the power through exp2/log2 (see
// geomean_arb_econ<true>).  A separate policy type = separate kernel instantiations,
// so the validated GeomeanPools kernels are untouched.
struct GeomeanPoolsLog2 : GeomeanPools {
  __device__ __forceinline__ Trade arb(const Pool& p, double v1, double v2,
                                       bool exact, bool econ) const {
    if (econ && !exact) return geomean_arb_econ<true>(p.R.x, p.R.y, p.w.x, p.w.y, p.g, v1, v2);
    return geomean_arb(p.R.x, p.R.y, p.w.x, p.w.y, p.g, v1, v2, exact);
  }
};

struct Univ3Pools {
  static constexpr int kMinBlocks = 3;  // latency-bound walks: 24 warps per SM (<= 85 registers)
  const double2* f0;      // (k, R_1+α) of the current tick, per pool   \  the tick a walk starts in
  const double2* f1;      // (R_2+β, current_price)                      |  (arb_math.cuh, Univ3First):
  const double2* f2;      // (δmax↑, R_2)                                |  64 B per pool, pool order
  const double2* f3;      // (δmax↓, R_1)                               /
  const double* gam;
  const int2* Ai;
  const int2* tick;       // (tick_off, current_tick 1-based)
  const double* tickdata; // CSR, kTickStride doubles per tick (precomputed BoundedProduct, see arb_math.cuh)
  int64_t m;
  int total_ticks;
  struct Pool {
    double cp, g;
    int off, cur, nt;
    Univ3First first;
  };
  __device__ __forceinline__ Pool load(int64_t i) const {
    Pool p;
    const double2 a = ld_stream(f0 + i), b = ld_stream(f1 + i);
    p.first.k = a.x;
    p.first.ra = a.y;
    p.first.rb = b.x;
    p.first.up = f2 + i;
    p.first.dn = f3 + i;
    p.cp = b.y;
    p.g = ld_stream(gam + i);
    const int2 t = ld_stream(tick + i);
    p.off = t.x;
    p.cur = t.y;
    const int next = (i + 1 < m) ? ld_stream(tick + i + 1).x : total_ticks;
    p.nt = next - t.x;
    return p;
  }
  __device__ __forceinline__ Trade arb(const Pool& p, double v1, double v2,
                                       bool, bool) const {
    return univ3_arb(tickdata + (size_t)p.off * kTickStride, p.nt, p.first, p.cp, p.cur, p.g, v1, v2);
  }
};

// ---- the sweep kernel -------------------------------------------------------

constexpr int kSweepThreads = 256;

// resident CTAs per SM the register allocation must allow (P::kMinBlocks where a type asks for it)
template <class P, class = void>
struct MinBlocks {
  static constexpr int value = 1;
};
template <class P>
struct MinBlocks<P, decltype((void)P::kMinBlocks)> {
  static constexpr int value = P::kMinBlocks;
};

template <class P, bool MAT, int U>
__global__ void __launch_bounds__(kSweepThreads, MinBlocks<P>::value)
    sweep_kernel(P pools, const double* __restrict__ nu, double* __restrict__ psi,
                 int n_tokens, double2* __restrict__ outD,
                 double2* __restrict__ outL, int64_t m, int flags,
                 double* __restrict__ zero_next) {
  // zero the accumulator the NEXT sweep will use (ping-pong; replaces a memset launch)
  if (zero_next)
    for (int i = blockIdx.x * kSweepThreads + threadIdx.x; i <= n_tokens; i += gridDim.x * kSweepThreads)
      zero_next[i] = 0.0;
  // flags: bit0 = exact (all four closed forms); bits 1-3 are measurement
  // switches (skip the Ψ[b] RED / the Ψ[a] segmented RED / the acc fold) used
  // only by tools/explore.py to attribute time; the product never sets them.
  const bool exact = flags & 1;
  const bool skip_b = flags & 2, skip_a = flags & 4, skip_acc = flags & 8;
  // bit4: economized closed forms (gradient-only sweeps; never with MAT)
  const bool econ = !MAT && (flags & 16);
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (kSweepThreads / 32) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (kSweepThreads / 32);
  double acc = 0.0;

  for (int64_t base = warp * (32 * U); base < m; base += n_warps * (32 * U)) {
    typename P::Pool pool[U];
    int2 ai[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = base + u * 32 + lane;
      ok[u] = i < m;
      const int64_t ii = ok[u] ? i : (m - 1);
      pool[u] = pools.load(ii);
      ai[u] = ld_stream(pools.Ai + ii);
    }
    double v1[U], v2[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      v1[u] = __ldg(nu + ai[u].x);
      v2[u] = __ldg(nu + ai[u].y);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      Trade t = pools.arb(pool[u], v1[u], v2[u], exact, econ);
      if (MAT && ok[u]) {
        const int64_t i = base + u * 32 + lane;
        outD[i] = make_double2(t.d1, t.d2);
        outL[i] = make_double2(t.l1, t.l2);
      }
      double f1 = t.l1 - t.d1;  // Λ − Δ on token a
      double f2 = t.l2 - t.d2;  // Λ − Δ on token b
      if (!ok[u]) {
        f1 = 0.0;
        f2 = 0.0;
      }
      // dot(Λ, ν[Ai]) − dot(Δ, ν[Ai])
      const double c = (t.l1 * v1[u] + t.l2 * v2[u]) - (t.d1 * v1[u] + t.d2 * v2[u]);
      if (!skip_acc) acc += (ok[u] && !no_reserves(pool[u])) ? c : 0.0;
      if (f2 != 0.0 && !skip_b) red_add(psi + ai[u].y, f2);
      if (!skip_a) warp_segmented_red(psi, ok[u] ? ai[u].x : -1, f1, lane);
    }
  }

  // acc: warp shuffle -> one RED per warp into psi[n_tokens]
  acc += shfl_xor_f64(acc, 16);
  acc += shfl_xor_f64(acc, 8);
  acc += shfl_xor_f64(acc, 4);
  acc += shfl_xor_f64(acc, 2);
  acc += shfl_xor_f64(acc, 1);
  __shared__ double s_acc[kSweepThreads / 32];
  if (lane == 0) s_acc[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < kSweepThreads / 32; ++w) s += s_acc[w];
    if (s != 0.0) red_add(psi + n_tokens, s);
  }
}

// ---- helpers ----------------------------------------------------------------

// gather rows of a sorted array back to insertion order: dst[orig[i]] = src[i]
__global__ void scatter_trades_kernel(const double2* __restrict__ D,
                                      const double2* __restrict__ L,
                                      const int64_t* __restrict__ orig,
                                      double2* __restrict__ outD,
                                      double2* __restrict__ outL, int64_t m) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  int64_t o = orig[i];
  if (o < 0) return;  // padding pool
  const bool swapped = (o >> 62) & 1;  // stored with its two tokens exchanged
  o &= ~(1ll << 62);
  const double2 d = D[i], l = L[i];
  outD[o] = swapped ? make_double2(d.y, d.x) : d;
  outL[o] = swapped ? make_double2(l.y, l.x) : l;
}

// apply_trade from the materialised trades of the same device order; *out_of_range is raised when
// a new reserve leaves the guard-free range.  active (device order, 0 = retired; null = all active)
// skips retired pools.
__global__ void apply_trades_kernel(double2* __restrict__ R, const double* __restrict__ gam,
                                    const double2* __restrict__ D, const double2* __restrict__ L,
                                    const int64_t* __restrict__ gidx, int64_t m,
                                    const uint8_t* __restrict__ active, int* __restrict__ out_of_range) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  if (gidx[i] < 0) return;  // padding pool
  if (active && !active[i]) return;  // retired pool: its zeroed reserves stay, its state is parked
  const double g = gam[i];
  const double2 r = R[i], d = D[i], l = L[i];
  const double2 n = apply_trade(r, g, d, l);
  R[i] = n;
  if (!in_fast_range(n.x) || !in_fast_range(n.y)) atomicOr(out_of_range, 1);
}

// R[pos[j]] = newR[j]; a retired pool (active[p] == 0; active may be null) gets it in its parked
// state instead, which becomes live when the pool is restored
__global__ void update_reserves_kernel(double2* __restrict__ R,
                                       const int64_t* __restrict__ pos,
                                       const double2* __restrict__ newR,
                                       int64_t count, const uint8_t* __restrict__ active,
                                       double2* __restrict__ park) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  const int64_t p = pos[j];
  if (active && !active[p])
    park[p] = newR[j];
  else
    R[p] = newR[j];
}

// Retire (flag 0) or restore (flag 1) the two-coin pools at device positions pos[j]: a retired
// pool's reserves move to park and R becomes (0, 0), the no-trade state of the padding pools.
// The host lists only pools whose flag changes.
__global__ void set_active_kernel(double2* __restrict__ R, double2* __restrict__ park,
                                  uint8_t* __restrict__ active, const int64_t* __restrict__ pos,
                                  int64_t count, int flag) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  const int64_t p = pos[j];
  if (R) {
    if (flag) {
      R[p] = park[p];
    } else {
      park[p] = R[p];
      R[p] = make_double2(0.0, 0.0);
    }
  }
  active[p] = (uint8_t)flag;
}

// Pool state in listing order (cfmm_get_pool_state): the pools at device positions pos[j].  Two-coin
// (R non-null): out[2j..2j+1] = the reserves as ingested (a pool stored with its tokens exchanged,
// bit 62 of gidx, is swapped back), the parked ones for a retired pool.  UniV3 (price non-null,
// the price word of f1): out[j] = the current price.
__global__ void gather_state_kernel(const double2* __restrict__ R, const double2* __restrict__ park,
                                    const uint8_t* __restrict__ active, const double2* __restrict__ price,
                                    const int64_t* __restrict__ gidx, const int64_t* __restrict__ pos,
                                    int64_t count, double* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  const int64_t p = pos[j];
  if (price) {
    out[j] = price[p].y;
    return;
  }
  const double2 r = (active && !active[p]) ? park[p] : R[p];
  const bool swapped = (gidx[p] >> 62) & 1;
  out[2 * j] = swapped ? r.y : r.x;
  out[2 * j + 1] = swapped ? r.x : r.y;
}

}  // namespace cfmm
