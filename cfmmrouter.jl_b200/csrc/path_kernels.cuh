// path_kernels.cuh -- multi-hop swap paths against the device-resident pools (sm_90a;
// cfmm_quote_paths / cfmm_execute_paths, include/cfmm_b200.h).  Off the sweep path.
//
// A path j is the hops hop_off[j] .. hop_off[j+1]) of a CSR list; hop h is a pool of set
// hop_set[h] (kPathSets sets: 2·type + 1 for the appended pools) at device position hop_pos[h].
// Every hop is priced with the per-pool pieces of swap_kernels.cuh (SwapPool<TYPE>: f, exact_out,
// execute), dispatched at run time on the hop's type; nothing here restates pool arithmetic.  The
// pools of one path are distinct (checked on the host), so a path's hops never see each other:
// a path is priced against the state before it and, when it fills, each hop runs the transition
// of swap_execute_kernel with its tender.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "swap_kernels.cuh"

namespace cfmm {

constexpr int kPathSets = 6;

// The six pool sets as the path kernels see them, kept in device memory (a hop's set is a run-time
// index, and an array in kernel parameter space indexed at run time would be copied to local
// memory).  Ai is the device-order token pair of d_Ai (0-based, stored order).  The rest is what an
// execute launch writes besides the pools: per set, a reserve that left the guard-free range and
// "a filled path moved a pool here"; per UniV3 set, the pools whose price moved (one entry per
// moving hop: a pool crossed by several paths of one call can appear more than once).
struct PathSets {
  SwapSet s[kPathSets];
  const int2* Ai[kPathSets];
  int* out_of_range;            // [kPathSets]
  int* touched;                 // [kPathSets]
  int64_t* moved[2];            // UniV3 main, UniV3 tail
  unsigned long long* n_moved;  // [2]
};

constexpr double kPathInf = __builtin_huge_val();

// f of hop (k, p) for a tender x of the ingest token tok1 (token 1) or token 2: cfmm_quote_swaps
// bit for bit; a zero tender receives 0, as a (0, 0) row there.
__device__ __forceinline__ double path_hop_f(const PathSets* P, int k, int64_t p, double x, bool tok1) {
  if (!(x > 0.0)) return 0.0;
  const SwapSet& s = P->s[k];
  switch (k >> 1) {
    case 0: return swap_pool<0>(s, p).f(x, tok1);
    case 1: return swap_pool<1>(s, p).f(x, tok1);
    default: return swap_pool<2>(s, p).f(x, tok1);
  }
}

// x* of hop (k, p) for a wanted output y (swap_quote_exact_out_kernel's search); 0 for y = 0.
__device__ __forceinline__ double path_hop_exact_out(const PathSets* P, int k, int64_t p, double y, bool tok1) {
  if (!(y > 0.0)) return 0.0;
  const SwapSet& s = P->s[k];
  switch (k >> 1) {
    case 0: return swap_pool<0>(s, p).exact_out(y, tok1);
    case 1: return swap_pool<1>(s, p).exact_out(y, tok1);
    default: return swap_pool<2>(s, p).exact_out(y, tok1);
  }
}

template <int TYPE>
__device__ __forceinline__ double path_two_coin_execute(const PathSets* P, int k, int64_t p, double x, bool tok1) {
  const SwapSet& s = P->s[k];
  SwapPool<TYPE> pool = swap_pool<TYPE>(s, p);
  const double l = pool.execute(x, tok1);
  s.R[p] = pool.R;
  if (!in_fast_range(pool.R.x) || !in_fast_range(pool.R.y)) atomicOr(P->out_of_range + k, 1);
  return l;
}

// Run the transition of swap_execute_kernel for a tender x > 0 on hop (k, p) and store the pool's
// new state.  A UniV3 pool's current tick (tick[p].y) is stored with its new price: a later level
// of the same call walks from it before the tick records are rebuilt at the end of the call.
__device__ __forceinline__ double path_hop_execute(const PathSets* P, int k, int64_t p, double x, bool tok1) {
  P->touched[k] = 1;
  if ((k >> 1) == 0) return path_two_coin_execute<0>(P, k, p, x, tok1);
  if ((k >> 1) == 1) return path_two_coin_execute<1>(P, k, p, x, tok1);
  const SwapSet& s = P->s[k];
  SwapPool<2> pool = swap_pool<2>(s, p);
  const double q0 = pool.q;
  const double l = pool.execute(x, tok1);
  if (pool.q != q0) {
    reinterpret_cast<double*>(s.u.f1 + p)[1] = pool.q;
    reinterpret_cast<int*>(s.u.tick + p)[1] = pool.cur;
    P->moved[k & 1][atomicAdd(P->n_moved + (k & 1), 1ull)] = p;
  }
  return l;
}

// Token check, before anything is written: one thread per path walks its token from token_in[j]
// (1-based) through the pools' ingest token pairs.  A ProductTwoCoin pool stored with its tokens
// exchanged (bit 62 of gidx) is mapped back to ingest order.  hop_tok1[h] = the hop tenders its
// pool's token 1.  The first hop (in CSR order) whose pool does not hold the current token is
// recorded in *first_bad (atomicMin; left at its initial value when every hop is good).
__global__ void path_check_kernel(const PathSets* __restrict__ P, int64_t q, const int64_t* __restrict__ hop_off,
                                  const uint8_t* __restrict__ hop_set, const int64_t* __restrict__ hop_pos,
                                  const int64_t* __restrict__ token_in, uint8_t* __restrict__ hop_tok1,
                                  unsigned long long* __restrict__ first_bad) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q) return;
  int64_t t = token_in[j] - 1;
  for (int64_t h = hop_off[j]; h < hop_off[j + 1]; ++h) {
    const int k = hop_set[h];
    const int64_t p = hop_pos[h];
    const int2 a = P->Ai[k][p];
    const bool sw = (k >> 1) < 2 && ((P->s[k].gidx[p] >> 62) & 1);
    const int64_t t1 = sw ? a.y : a.x, t2 = sw ? a.x : a.y;
    if (t == t1) {
      hop_tok1[h] = 1;
      t = t2;
    } else if (t == t2) {
      hop_tok1[h] = 0;
      t = t1;
    } else {
      atomicMin(first_bad, (unsigned long long)h);
      return;
    }
  }
}

// One path, priced against the current state of its pools (include/cfmm_b200.h, cfmm_quote_paths):
// exact-in forward from x₁ = amount, passing on max(λ_h, 0); exact-out backward from y_n = amount
// through each hop's x*.  Writes every hop's tender and received and the path's status.  EXEC
// (cfmm_execute_paths): the path's limit decides, and a filled path then runs each hop's transition
// with its tender.  A path that does not fill reports zeros.
template <bool EXEC>
__device__ __forceinline__ void path_run(const PathSets* P, int64_t j, const int64_t* hop_off, const uint8_t* hop_set,
                                         const int64_t* hop_pos, const uint8_t* hop_tok1, const uint8_t* kind,
                                         const double* amount, const double* limit, double* tender,
                                         double* received, uint8_t* status) {
  const int64_t h0 = hop_off[j], h1 = hop_off[j + 1];
  uint8_t st = 0;  // CFMM_ORDER_FILLED
  for (int64_t h = h0; h < h1; ++h) {
    const SwapSet& s = P->s[hop_set[h]];
    if (s.active && !s.active[hop_pos[h]]) st = 3;  // CFMM_ORDER_RETIRED
  }
  if (st == 0) {
    if (kind[j] == 0) {
      double x = amount[j], lam = 0.0;
      for (int64_t h = h0; h < h1; ++h) {
        lam = path_hop_f(P, hop_set[h], hop_pos[h], x, hop_tok1[h]);
        tender[h] = x;
        received[h] = lam;
        x = lam > 0.0 ? lam : 0.0;
      }
      if (EXEC && lam < (limit ? limit[j] : 0.0)) st = 1;  // CFMM_ORDER_LIMIT
    } else {
      double y = amount[j];
      for (int64_t h = h1 - 1; h >= h0; --h) {
        const int k = hop_set[h];
        const bool tok1 = hop_tok1[h];
        const double x = path_hop_exact_out(P, k, hop_pos[h], y, tok1);
        if (x == kPathInf) {
          st = 2;  // CFMM_ORDER_UNREACHABLE
          break;
        }
        tender[h] = x;
        received[h] = path_hop_f(P, k, hop_pos[h], x, tok1);
        y = x;
      }
      if (EXEC && st == 0 && y > (limit ? limit[j] : kPathInf)) st = 1;
    }
  }
  if (st != 0) {
    for (int64_t h = h0; h < h1; ++h) {
      tender[h] = 0.0;
      received[h] = 0.0;
    }
  } else if (EXEC) {
    for (int64_t h = h0; h < h1; ++h) {
      const double x = tender[h];
      if (x > 0.0) received[h] = path_hop_execute(P, hop_set[h], hop_pos[h], x, hop_tok1[h]);
    }
  }
  status[j] = st;
}

// Quotes: one thread per path, every path on the current state on its own.
__global__ void path_quote_kernel(const PathSets* __restrict__ P, int64_t q, const int64_t* __restrict__ hop_off,
                                  const uint8_t* __restrict__ hop_set, const int64_t* __restrict__ hop_pos,
                                  const uint8_t* __restrict__ hop_tok1, const uint8_t* __restrict__ kind,
                                  const double* __restrict__ amount, double* tender, double* received,
                                  uint8_t* __restrict__ status) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q) return;
  path_run<false>(P, j, hop_off, hop_set, hop_pos, hop_tok1, kind, amount, nullptr, tender, received, status);
}

// Execution of one level: one thread per path of paths[0 .. n).  The paths of a level touch
// disjoint pools, and every earlier level is complete (stream order), so each thread reads and
// writes its own pools only.
__global__ void path_execute_kernel(const PathSets* __restrict__ P, const int64_t* __restrict__ paths, int64_t n,
                                    const int64_t* __restrict__ hop_off, const uint8_t* __restrict__ hop_set,
                                    const int64_t* __restrict__ hop_pos, const uint8_t* __restrict__ hop_tok1,
                                    const uint8_t* __restrict__ kind, const double* __restrict__ amount,
                                    const double* __restrict__ limit, double* tender, double* received,
                                    uint8_t* __restrict__ status) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  path_run<true>(P, paths[i], hop_off, hop_set, hop_pos, hop_tok1, kind, amount, limit, tender, received, status);
}

}  // namespace cfmm
