// route_kernels.cuh -- orders routed over their pair's pools and two-hop routes through hub tokens
// (sm_90a; cfmm_quote_routed_orders / cfmm_execute_routed_orders, include/cfmm_b200.h).  Off the
// sweep path: no sweep kernel reads anything these kernels add.
//
// A row sells token j for token i over the pools of (j, i) and, for each of its hubs h, the pools of
// (j, h) and (h, i); pools between two hubs are not used.  With ν_i = 1, ν_j = s and ν_h = t_h, each
// hub price only enters its own hub's pools, so route!'s dual with Swap separates: for fixed s, t_h
// is the root of "hub h's pools net to zero in h" (an inner ordinal search per hub), and s* is the
// split's search on N(s), the net intake of j over all the row's pools.  One CTA runs a row: warp 0
// owns the direct pools, warp 1 + h owns hub h's pools, and warp partials meet in shared memory in
// a fixed order.  The pool views, legs, boundaries, searches and transitions are split_kernels.cuh's.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "split_kernels.cuh"

namespace cfmm {

constexpr int kRouteMaxHubs = 7;  // CFMM_ROUTE_MAX_HUBS
constexpr int kRouteThreads = 32 * (1 + kRouteMaxHubs);

// The rows of one call (device arrays; tokens 1-based).  Row r's pair lists start at
// r + 2·hub_off[r] in pair / leg_off: (j, i), then (j, h), (h, i) for each of its hubs in order.
struct RouteRows {
  const int64_t* token_in;
  const int64_t* token_out;
  const uint8_t* kind;
  const double* amount;
  const double* limit;    // null: none
  const int64_t* hub_off; // [q+1]
  const int64_t* hubs;    // [Σ]
  const int64_t* pair;    // [q + 2Σ]: index into the pair index, -1: no pool holds the pair
  const int64_t* leg_off; // [q + 2Σ + 1]
  double* paid;
  double* received;
  double* price;
  uint8_t* status;
  double* hub_price;      // [Σ] or null
  double* hub_surplus;    // [Σ] or null
  double* leg_delta;      // [2L] or null
  double* leg_lambda;
};

// The pools one warp owns for a row: list a (the direct pair, or (j, h)) and list b ((h, i); empty
// for the direct warp), with the token of each list whose price is the list's first (j for list a,
// h for list b).
struct RouteWarp {
  const int64_t* a;
  const int64_t* b;
  int64_t ca, cb;
  int64_t ta, tb;
  bool hub;
};

__device__ __forceinline__ RouteWarp route_warp(const PairIndexView& ix, const RouteRows& R, int64_t row, int w,
                                                int64_t tj) {
  RouteWarp W;
  const int64_t base = row + 2 * R.hub_off[row];
  const int64_t pa = R.pair[w == 0 ? base : base + 2 * w - 1];
  const int64_t pb = w == 0 ? -1 : R.pair[base + 2 * w];
  W.a = pa >= 0 ? ix.pool + ix.off[pa] : nullptr;
  W.ca = pa >= 0 ? ix.off[pa + 1] - ix.off[pa] : 0;
  W.b = pb >= 0 ? ix.pool + ix.off[pb] : nullptr;
  W.cb = pb >= 0 ? ix.off[pb + 1] - ix.off[pb] : 0;
  W.ta = tj;
  W.tb = w == 0 ? -1 : R.hubs[R.hub_off[row] + w - 1] - 1;
  W.hub = w != 0;
  return W;
}

// Pool t of the warp's lists at ν_j = s, ν_h = th, ν_i = 1: split_pool's view with the two prices of
// its tokens (list a: j at s, the other at th for a hub warp and 1 for the direct warp; list b: h at
// th, i at 1).
__device__ __forceinline__ SplitPool route_pool(const PathSets* P, const RouteWarp& W, int64_t t, double s, double th,
                                                bool& inb) {
  inb = t >= W.ca;
  SplitPool sp = split_pool(P, inb ? W.b[t - W.ca] : W.a[t], inb ? W.tb : W.ta, 1.0);
  const double pa = inb ? th : s, pb = (inb || !W.hub) ? 1.0 : th;
  sp.v1 = sp.x_is_j ? pa : pb;
  sp.v2 = sp.x_is_j ? pb : pa;
  return sp;
}

struct RouteSums {
  double n, o, h;  // net intake of j, output of i, the trader's net of h
};

// The warp's sums at (s, th), warp-wide (split_sums' tree: lane l adds the terms of pools l, l + 32,
// … of list a then list b from +0.0, then the xor butterfly).  A pool adds nothing to a sum whose
// token it does not hold.
__device__ __forceinline__ RouteSums route_sums(const PathSets* P, const RouteWarp& W, double s, double th, int lane) {
  double n = 0.0, o = 0.0, h = 0.0;
  const int64_t cnt = W.ca + W.cb;
  for (int64_t t = lane; t < cnt; t += 32) {
    bool inb;
    const SplitPool sp = route_pool(P, W, t, s, th, inb);
    const Trade tr = split_legs(P, sp);
    // x_is_j: the pool's stored token 1 is the list's first token
    const double first_in = sp.x_is_j ? __dsub_rn(tr.d1, tr.l1) : __dsub_rn(tr.d2, tr.l2);
    const double other_out = sp.x_is_j ? __dsub_rn(tr.l2, tr.d2) : __dsub_rn(tr.l1, tr.d1);
    if (inb) {  // (h, i): h is the first token
      o = __dadd_rn(o, other_out);
      h = __dadd_rn(h, sp.x_is_j ? __dsub_rn(tr.l1, tr.d1) : __dsub_rn(tr.l2, tr.d2));
    } else {
      n = __dadd_rn(n, first_in);
      if (W.hub)
        h = __dadd_rn(h, other_out);
      else
        o = __dadd_rn(o, other_out);
    }
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    n = __dadd_rn(n, __shfl_xor_sync(kFull, n, m));
    o = __dadd_rn(o, __shfl_xor_sync(kFull, o, m));
    h = __dadd_rn(h, __shfl_xor_sync(kFull, h, m));
  }
  return {n, o, h};
}

// Row `row`, CTA-wide (blockDim.x = 32·(1 + the call's largest hub count); every thread takes every
// CTA-level branch).  EXEC: the limit decides, and a filled row applies cfmm_apply_trades' transition
// at its ν to each of its pools.  ARB: an arbitrage row (cfmm_quote_arbitrage), the exact-in row with
// δ = 0 that runs its search: j = the other token x, i = the base token p, kind and amount unread,
// the limit is the minimum profit, paid reports the surplus 0 − N(s*) and received the profit O(s*);
// a row whose pair {x, p} no pool holds is unreachable, and leg_off may be null when there are no legs.
template <bool EXEC, bool ARB = false>
__device__ __forceinline__ void route_row(const PathSets* P, const PairIndexView& ix, const RouteRows& R, int64_t row,
                                          const SplitMoved& mv) {
  __shared__ double sh_n[1 + kRouteMaxHubs], sh_o[1 + kRouteMaxHubs], sh_b1[1 + kRouteMaxHubs],
      sh_b2[1 + kRouteMaxHubs];
  __shared__ int sh_flag[1 + kRouteMaxHubs];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nh = (int)(R.hub_off[row + 1] - R.hub_off[row]);
  const bool mine = w <= nh;  // this warp owns the direct pools or a hub's
  const int64_t tj = R.token_in[row] - 1;
  const bool out = !ARB && R.kind[row] == 1;
  const double amt = ARB ? 0.0 : R.amount[row];
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  const double lim = R.limit ? R.limit[row] : (out ? inf : 0.0);
  RouteWarp W{};
  if (mine) W = route_warp(ix, R, row, w, tj);
  uint8_t st = 0;  // CFMM_ORDER_FILLED
  if (ARB && R.pair[row + 2 * R.hub_off[row]] < 0) st = 2;
  double s = 0.0;
  double N = 0.0, O = 0.0;
  int64_t th = kSplitOrdMin;  // this hub warp's t_h at s*, as an ordinal
  double hs = 0.0;            // and its surplus there
  if (ARB ? st == 0 : amt > 0.0) {  // a routed row with amount 0 fills with zeros and runs no search
    // start: the largest no-trade boundary per list, and whether the list has an active pool
    if (mine) {
      double b1 = -inf, b2 = -inf;
      bool a1 = false, a2 = false;
      for (int64_t t = lane; t < W.ca + W.cb; t += 32) {
        bool inb;
        const SplitPool sp = route_pool(P, W, t, 1.0, 1.0, inb);
        const double b = split_boundary(P, sp);
        if (inb) {
          a2 = a2 || sp.active;
          b2 = b > b2 ? b : b2;
        } else {
          a1 = a1 || sp.active;
          b1 = b > b1 ? b : b1;
        }
      }
#pragma unroll
      for (int m = 16; m >= 1; m >>= 1) {
        const double o1 = __shfl_xor_sync(kFull, b1, m), o2 = __shfl_xor_sync(kFull, b2, m);
        b1 = o1 > b1 ? o1 : b1;
        b2 = o2 > b2 ? o2 : b2;
      }
      const int f = (__any_sync(kFull, a1) ? 1 : 0) | (__any_sync(kFull, a2) ? 2 : 0);
      if (lane == 0) {
        sh_b1[w] = b1;
        sh_b2[w] = b2;
        sh_flag[w] = f;
      }
    }
    __syncthreads();
    double e = sh_b1[0];
    bool any = sh_flag[0] != 0;
    for (int h = 1; h <= nh; ++h) {
      any = any || sh_flag[h] != 0;
      if (sh_flag[h] == 3) {  // a composite route: the hub has active pools on both sides
        const double c = __dmul_rn(sh_b1[h], sh_b2[h]);
        e = c > e ? c : e;
      }
    }
    int64_t tprev = 0;
    if (mine && W.hub) tprev = split_start(sh_b2[w]);
    __syncthreads();
    if (!any) {
      st = 2;  // CFMM_ORDER_UNREACHABLE
    } else {
      bool bad = false;  // some hub's pools net < 0 in h even at t = DBL_MAX
      double n_last = 0.0, o_last = 0.0, h_last = 0.0;
      int64_t t_last = 0;
      const auto test = [&](int64_t c) {
        if (bad) return false;
        const double sv = __longlong_as_double(c);
        if (w == 0) {
          const RouteSums r = route_sums(P, W, sv, 1.0, lane);
          if (lane == 0) {
            sh_n[0] = r.n;
            sh_o[0] = r.o;
          }
        } else if (mine) {
          RouteSums last = {0.0, 0.0, 0.0}, at_hi = last;
          int64_t tlo = 0, thi = 0;
          const int rc = split_search(
              tprev, tlo, thi,
              [&](int64_t ct) {
                last = route_sums(P, W, sv, __longlong_as_double(ct), lane);
                return !(last.h >= 0.0);  // H_h < 0 (or NaN): t_h is still too small
              },
              [&](bool is_lo) {
                if (!is_lo) at_hi = last;
              });
          if (rc != 1) {
            tprev = thi;
            t_last = thi;
            h_last = at_hi.h;
          }
          if (lane == 0) {
            sh_n[w] = at_hi.n;
            sh_o[w] = at_hi.o;
            sh_flag[w] = rc == 1;
          }
        }
        __syncthreads();
        double n = sh_n[0], o = sh_o[0];
        for (int h = 1; h <= nh; ++h) {
          n = __dadd_rn(n, sh_n[h]);
          o = __dadd_rn(o, sh_o[h]);
          bad = bad || sh_flag[h] != 0;
        }
        __syncthreads();
        n_last = n;
        o_last = o;
        if (bad) return false;
        return out ? o >= amt : !(n <= amt);  // exact-in: N > δ, a NaN counts as true
      };
      double n_lo = 0.0, o_lo = 0.0, h_lo = 0.0, n_hi = 0.0, o_hi = 0.0, h_hi = 0.0;
      int64_t t_lo = kSplitOrdMin, t_hi = kSplitOrdMin;
      const auto keep = [&](bool is_lo) {
        if (is_lo) {
          n_lo = n_last;
          o_lo = o_last;
          t_lo = t_last;
          h_lo = h_last;
        } else {
          n_hi = n_last;
          o_hi = o_last;
          t_hi = t_last;
          h_hi = h_last;
        }
      };
      int64_t lo = 0, hi = 0;
      const int rc = split_search(split_start(e), lo, hi, test, keep);
      if (rc != 0 || bad) {
        st = 2;
      } else {
        s = __longlong_as_double(out ? lo : hi);
        N = out ? n_lo : n_hi;
        O = out ? o_lo : o_hi;
        th = out ? t_lo : t_hi;
        hs = out ? h_lo : h_hi;
        if (EXEC && (out ? N > lim : O < lim)) st = 1;  // CFMM_ORDER_LIMIT; an equal limit fills
      }
    }
  }
  const bool filled = st == 0 && (ARB || amt > 0.0);
  // legs (list order) and, on execute, the transition of each pool at (s*, t_h*)
  if (mine) {
    const double tv = __longlong_as_double(th);
    const int64_t base = row + 2 * R.hub_off[row];
    const int64_t l0 = (ARB && !R.leg_off) ? 0 : R.leg_off[w == 0 ? base : base + 2 * w - 1];
    for (int64_t t = lane; t < W.ca + W.cb; t += 32) {
      bool inb;
      split_leg<EXEC>(
          P, filled, [&] { return route_pool(P, W, t, s, tv, inb); }, mv, R.leg_delta, R.leg_lambda, l0 + t);
    }
    if (lane == 0 && W.hub) {
      const int64_t g = R.hub_off[row] + w - 1;
      if (R.hub_price) R.hub_price[g] = (st == 2 || !(ARB || amt > 0.0)) ? 0.0 : tv;
      if (R.hub_surplus) R.hub_surplus[g] = filled ? hs : 0.0;
    }
  }
  if (threadIdx.x == 0) {
    R.paid[row] = filled ? (ARB ? __dsub_rn(0.0, N) : N) : 0.0;
    R.received[row] = filled ? O : 0.0;
    R.price[row] = st == 2 ? 0.0 : s;
    R.status[row] = st;
  }
}

// Quotes: one CTA per row, every row on the current state on its own.
__global__ void __launch_bounds__(kRouteThreads, 1) route_quote_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                    RouteRows R) {
  route_row<false>(P, ix, R, blockIdx.x, SplitMoved{});
}

// Execution of one level: rows[0 .. gridDim.x), one CTA each.  Rows of a level share no token pair,
// so no pool; a level runs on the state the earlier levels left.
__global__ void __launch_bounds__(kRouteThreads, 1) route_execute_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                      RouteRows R, const int64_t* __restrict__ rows,
                                                                      SplitMoved mv) {
  route_row<true>(P, ix, R, rows[blockIdx.x], mv);
}

// Arbitrage rows (cfmm_quote_arbitrage / cfmm_execute_arbitrage, and the solve of
// cfmm_scan_arbitrage): route_row's ARB mode, launched as the routed kernels are.
__global__ void __launch_bounds__(kRouteThreads, 1) arb_quote_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                  RouteRows R) {
  route_row<false, true>(P, ix, R, blockIdx.x, SplitMoved{});
}

__global__ void __launch_bounds__(kRouteThreads, 1) arb_execute_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                    RouteRows R, const int64_t* __restrict__ rows,
                                                                    SplitMoved mv) {
  route_row<true, true>(P, ix, R, rows[blockIdx.x], mv);
}

}  // namespace cfmm
