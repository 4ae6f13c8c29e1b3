// hub_kernels.cuh -- the hub choice of cfmm_choose_order_hubs (sm_90a, include/cfmm_b200.h).  Off the
// sweep path: no sweep kernel reads anything these kernels add.
//
// One warp per order row (j → i).  The lanes walk the shorter of j's and i's adjacency lists
// (arb_scan_kernels.cuh), bisect the longer for common neighbours h, and score each allowed h by the
// best single two-hop route j → h → i: exact-in the most i that δ of j buys through the best {j, h}
// pool and then the best {h, i} pool; exact-out the least j that buys y of i the same way backwards.
// Each quote is path_hop_f / path_hop_exact_out, cfmm_quote_swaps / cfmm_quote_swaps_exact_out bit
// for bit.  Every lane keeps its best max_hubs hubs; the warp merges the lists.  Max, min and the
// (score, token) ranking do not depend on the evaluation order, so the result does not depend on
// the launch shape.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arb_scan_kernels.cuh"

namespace cfmm {

// The tender side of one pair pool, as a path hop: its set, position and whether the tendered token
// t is the pool's ingest token 1 (a two-coin pool stored exchanged is mapped back).
struct HubHop {
  int k;
  int64_t p;
  bool tok1, active;
};

__device__ __forceinline__ HubHop hub_hop(const PathSets* P, int64_t entry, int64_t t) {
  const SplitPool sp = split_pool(P, entry, t, 1.0);
  return HubHop{sp.k, sp.p, sp.x_is_j != sp.sw, sp.active};
}

// The largest exact-in quote for x of t over the active pools of pair k (NaNs ignored; 0 if none).
__device__ __forceinline__ double hub_best_f(const PathSets* P, PairIndexView ix, int32_t k, int64_t t, double x) {
  double best = 0.0;
  for (int64_t e = ix.off[k]; e < ix.off[k + 1]; ++e) {
    const HubHop h = hub_hop(P, ix.pool[e], t);
    if (!h.active) continue;
    const double v = path_hop_f(P, h.k, h.p, x, h.tok1);
    if (v > best) best = v;
  }
  return best;
}

// The smallest exact-out tender of t for y over the active pools of pair k (NaNs ignored; +inf if
// none reaches y).
__device__ __forceinline__ double hub_best_exact_out(const PathSets* P, PairIndexView ix, int32_t k, int64_t t,
                                                     double y) {
  double best = kPathInf;
  for (int64_t e = ix.off[k]; e < ix.off[k + 1]; ++e) {
    const HubHop h = hub_hop(P, ix.pool[e], t);
    if (!h.active) continue;
    const double v = path_hop_exact_out(P, h.k, h.p, y, h.tok1);
    if (v < best) best = v;
  }
  return best;
}

// Row r: n_elig[r] = its eligible hubs, nhub[r] = min(n_elig, max_hubs), and the chosen hubs (1-based)
// and scores at hub[max_hubs·r ..], score[max_hubs·r ..], best first.  The rank key is out_h
// (exact-in) or −in_h (exact-out), descending, then h ascending; an eligible key is > −inf.
__global__ void hub_choice_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A,
                                  const int64_t* __restrict__ token_in, const int64_t* __restrict__ token_out,
                                  const uint8_t* __restrict__ kind, const double* __restrict__ amount, int64_t q,
                                  int max_hubs, const uint8_t* __restrict__ allowed, int64_t* __restrict__ nhub,
                                  int64_t* __restrict__ hub, double* __restrict__ score,
                                  int64_t* __restrict__ n_elig) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= q) return;
  const int32_t j = (int32_t)(token_in[r] - 1), i = (int32_t)(token_out[r] - 1);
  const bool out = kind[r] != 0;
  const double amt = amount[r];
  const int64_t j0 = A.off[j], j1 = A.off[j + 1], i0 = A.off[i], i1 = A.off[i + 1];
  const bool walk_j = j1 - j0 <= i1 - i0;
  const int64_t w0 = walk_j ? j0 : i0, w1 = walk_j ? j1 : i1, s0 = walk_j ? i0 : j0, s1 = walk_j ? i1 : j1;
  constexpr double kNone = -__builtin_huge_val();
  double sc[kRouteMaxHubs];
  int32_t yy[kRouteMaxHubs];
#pragma unroll
  for (int m = 0; m < kRouteMaxHubs; ++m) {
    sc[m] = kNone;  // empty: every eligible key ranks before it
    yy[m] = INT32_MAX;
  }
  int64_t count = 0;
  for (int64_t e = w0 + lane; amt > 0.0 && e < w1; e += 32) {
    const int32_t h = A.nbr[e];
    if (allowed && !allowed[h]) continue;
    int64_t lo = s0, hi = s1;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (A.nbr[mid] < h)
        lo = mid + 1;
      else
        hi = mid;
    }
    if (lo == s1 || A.nbr[lo] != h) continue;
    const int32_t kjh = walk_j ? A.pair[e] : A.pair[lo], khi = walk_j ? A.pair[lo] : A.pair[e];
    double key;
    if (!out) {
      const double x = hub_best_f(P, ix, kjh, j, amt);
      const double o = hub_best_f(P, ix, khi, h, x);
      key = o > 0.0 ? o : kNone;
    } else {
      const double c = hub_best_exact_out(P, ix, khi, h, amt);
      const double x = c < kPathInf ? hub_best_exact_out(P, ix, kjh, j, c) : kPathInf;
      key = x < kPathInf ? -x : kNone;
    }
    if (!(key > kNone)) continue;
    ++count;
    double s = key;
    int32_t yv = h;
#pragma unroll
    for (int m = 0; m < kRouteMaxHubs; ++m) {  // insert, the displaced entry moving down
      if (m < max_hubs && arb_before(s, yv, sc[m], yy[m])) {
        const double ts = sc[m];
        const int32_t ty = yy[m];
        sc[m] = s;
        yy[m] = yv;
        s = ts;
        yv = ty;
      }
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) count += __shfl_xor_sync(kFull, count, m);
  // merge the lanes' lists: max_hubs rounds of a warp-wide best head, popped by the lane holding it
  int taken = 0;
  for (int t = 0; t < max_hubs; ++t) {
    double bs = sc[0];
    int32_t by = yy[0];
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      const double os = __shfl_xor_sync(kFull, bs, m);
      const int32_t oy = __shfl_xor_sync(kFull, by, m);
      if (arb_before(os, oy, bs, by)) {
        bs = os;
        by = oy;
      }
    }
    if (!(bs > kNone)) break;  // no eligible entry left (uniform across the warp)
    if (yy[0] == by) {
      hub[(int64_t)max_hubs * r + t] = by + 1;
      score[(int64_t)max_hubs * r + t] = out ? -bs : bs;
#pragma unroll
      for (int m = 0; m + 1 < kRouteMaxHubs; ++m) {
        sc[m] = sc[m + 1];
        yy[m] = yy[m + 1];
      }
      sc[kRouteMaxHubs - 1] = kNone;
      yy[kRouteMaxHubs - 1] = INT32_MAX;
    }
    ++taken;
  }
  if (lane == 0) {
    nhub[r] = taken;
    n_elig[r] = count;
  }
}

}  // namespace cfmm
