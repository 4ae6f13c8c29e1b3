// arb_scan_kernels.cuh -- the candidate search of cfmm_scan_arbitrage (sm_90a, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// Token adjacency.  From the pair index's distinct keys (split_kernels.cuh): for pair k = {a, b} the
// entries a → b and b → a, radix-sorted by (token, neighbour); adj_off[t] .. adj_off[t+1] are token t's
// neighbours ascending, each with its pair index (32-bit tokens and pairs).
//
// Rates.  rate[2k] = r(lo → hi) and rate[2k + 1] = r(hi → lo) for pair k with tokens lo < hi: the
// largest split_boundary over the pair's active pools with the selling token in j's role (the bit
// pattern the routed search starts from), 0 when no pool is active; NaNs are ignored.
//
// Candidates.  One warp per (base p, neighbour x): the pair score r(p→x)·r(x→p) and, for each common
// neighbour y of p and x, the triangle score; the row's hubs are the best passing triangles.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "route_kernels.cuh"

namespace cfmm {

constexpr double kArbScreen = 1.0 - 0x1p-40;  // a cycle score passes when it is > this

// ---- adjacency --------------------------------------------------------------------------------
// Pair k: its two directed entries, keyed token·n + neighbour, valued k.
__global__ void adj_entries_kernel(const int64_t* __restrict__ keys, int64_t n_pairs, int64_t n_tokens,
                                   int64_t* __restrict__ akey, int32_t* __restrict__ apair) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_pairs) return;
  const int64_t a = keys[k] / n_tokens, b = keys[k] % n_tokens;
  akey[2 * k] = a * n_tokens + b;
  akey[2 * k + 1] = b * n_tokens + a;
  apair[2 * k] = (int32_t)k;
  apair[2 * k + 1] = (int32_t)k;
}

// The neighbour of each sorted entry, and (threads 0 .. n_tokens) each token's first entry.
__global__ void adj_finish_kernel(const int64_t* __restrict__ skey, int64_t m, int64_t n_tokens,
                                  int32_t* __restrict__ nbr, int64_t* __restrict__ off) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < m) nbr[e] = (int32_t)(skey[e] % n_tokens);
  if (e <= n_tokens) {
    const int64_t key = e * n_tokens;
    int64_t lo = 0, hi = m;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (skey[mid] < key)
        lo = mid + 1;
      else
        hi = mid;
    }
    off[e] = lo;
  }
}

// ---- rates ------------------------------------------------------------------------------------
// One thread per entry t of the pair index's pool list (pair k: off[k] <= t < off[k+1]).  The max is
// an atomicMax on the int64 bits of non-negative doubles: exact, so independent of the order.
__global__ void arb_rates_kernel(const PathSets* __restrict__ P, const int64_t* __restrict__ off,
                                 const int64_t* __restrict__ pool, const int64_t* __restrict__ keys, int64_t n_pairs,
                                 int64_t n_tokens, long long* __restrict__ rate) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= off[n_pairs]) return;
  int64_t lo = 0, hi = n_pairs;  // the last k with off[k] <= t
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (off[mid] <= t)
      lo = mid;
    else
      hi = mid;
  }
  const int64_t a = keys[lo] / n_tokens, b = keys[lo] % n_tokens;  // a < b
  const SplitPool sa = split_pool(P, pool[t], a, 1.0);
  if (!sa.active) return;
  const double rab = split_boundary(P, sa);
  const double rba = split_boundary(P, split_pool(P, pool[t], b, 1.0));
  if (rab > 0.0) atomicMax(rate + 2 * lo, (long long)__double_as_longlong(rab));
  if (rba > 0.0) atomicMax(rate + 2 * lo + 1, (long long)__double_as_longlong(rba));
}

// ---- candidates -------------------------------------------------------------------------------
struct AdjView {
  const int64_t* off;   // [n_tokens + 1]
  const int32_t* nbr;   // [2·n_pairs]
  const int32_t* pair;  // [2·n_pairs]
};

// r(u → v) over pair k
__device__ __forceinline__ double arb_rate(const double* rate, int32_t k, int32_t u, int32_t v) {
  return rate[2 * (int64_t)k + (u > v ? 1 : 0)];
}

// (s1, y1) ranks before (s2, y2): score descending, then token ascending
__device__ __forceinline__ bool arb_before(double s1, int32_t y1, double s2, int32_t y2) {
  return s1 > s2 || (s1 == s2 && y1 < y2);
}

// Slot w = slot_off[b] + e of the call: base b (0-based token base[b]) and its e-th neighbour x.
// flag[w]: the row (p, x) qualifies; nhub[w]: its hub count (0 unless flagged); hub[7w ..]: its hubs
// (0-based) best first; lists[15w ..]: the pairs {x, p}, then {x, y}, {y, p} per hub.
__global__ void arb_candidates_kernel(AdjView A, const double* __restrict__ rate, const int64_t* __restrict__ base,
                                      const int64_t* __restrict__ slot_off, int64_t nb, int max_hubs,
                                      int64_t* __restrict__ flag, int64_t* __restrict__ nhub,
                                      int32_t* __restrict__ hub, int32_t* __restrict__ lists) {
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= slot_off[nb]) return;
  int64_t bl = 0, bh = nb;  // the last b with slot_off[b] <= w
  while (bh - bl > 1) {
    const int64_t mid = (bl + bh) >> 1;
    if (slot_off[mid] <= w)
      bl = mid;
    else
      bh = mid;
  }
  const int32_t p = (int32_t)(base[bl] - 1);
  const int64_t ep = A.off[p] + (w - slot_off[bl]);
  const int32_t x = A.nbr[ep], kpx = A.pair[ep];
  const double r_px = arb_rate(rate, kpx, p, x), r_xp = arb_rate(rate, kpx, x, p);
  const bool pair_pass = __dmul_rn(r_px, r_xp) > kArbScreen;
  // common neighbours: walk the shorter list, bisect the longer
  const int64_t p0 = A.off[p], p1 = A.off[p + 1], x0 = A.off[x], x1 = A.off[x + 1];
  const bool walk_p = p1 - p0 <= x1 - x0;
  const int64_t w0 = walk_p ? p0 : x0, w1 = walk_p ? p1 : x1, s0 = walk_p ? x0 : p0, s1 = walk_p ? x1 : p1;
  double sc[kRouteMaxHubs];
  int32_t yy[kRouteMaxHubs], ka[kRouteMaxHubs], kb[kRouteMaxHubs];
#pragma unroll
  for (int i = 0; i < kRouteMaxHubs; ++i) {
    sc[i] = -1.0;  // empty: every passing score ranks before it
    yy[i] = INT32_MAX;
    ka[i] = kb[i] = -1;
  }
  bool any = false;
  for (int64_t e = w0 + lane; e < w1; e += 32) {
    const int32_t y = A.nbr[e];
    int64_t lo = s0, hi = s1;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (A.nbr[mid] < y)
        lo = mid + 1;
      else
        hi = mid;
    }
    if (lo == s1 || A.nbr[lo] != y) continue;
    const int32_t kpy = walk_p ? A.pair[e] : A.pair[lo], kxy = walk_p ? A.pair[lo] : A.pair[e];
    const double t1 = __dmul_rn(__dmul_rn(r_px, arb_rate(rate, kxy, x, y)), arb_rate(rate, kpy, y, p));
    const double t2 = __dmul_rn(__dmul_rn(arb_rate(rate, kpy, p, y), arb_rate(rate, kxy, y, x)), r_xp);
    const bool q1 = t1 > kArbScreen, q2 = t2 > kArbScreen;
    if (!q1 && !q2) continue;
    any = true;
    double s = !q2 ? t1 : !q1 ? t2 : (t2 > t1 ? t2 : t1);  // the larger passing product
    int32_t yv = y, a = kxy, b = kpy;
#pragma unroll
    for (int i = 0; i < kRouteMaxHubs; ++i) {  // insert, the displaced entry moving down
      if (i < max_hubs && arb_before(s, yv, sc[i], yy[i])) {
        const double ts = sc[i];
        const int32_t ty = yy[i], ta = ka[i], tb = kb[i];
        sc[i] = s;
        yy[i] = yv;
        ka[i] = a;
        kb[i] = b;
        s = ts;
        yv = ty;
        a = ta;
        b = tb;
      }
    }
  }
  const bool emit = pair_pass || __any_sync(kFull, any);
  if (lane == 0) flag[w] = emit;
  // merge the lanes' lists: max_hubs rounds of a warp-wide best head, popped by the lane holding it
  int count = 0;
  for (int r = 0; r < max_hubs; ++r) {
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
    if (!(bs > kArbScreen)) break;  // no passing entry left (uniform across the warp)
    if (yy[0] == by) {
      if (emit) {
        hub[kRouteMaxHubs * w + r] = by;
        lists[(1 + 2 * kRouteMaxHubs) * w + 1 + 2 * r] = ka[0];
        lists[(1 + 2 * kRouteMaxHubs) * w + 2 + 2 * r] = kb[0];
      }
#pragma unroll
      for (int i = 0; i + 1 < kRouteMaxHubs; ++i) {
        sc[i] = sc[i + 1];
        yy[i] = yy[i + 1];
        ka[i] = ka[i + 1];
        kb[i] = kb[i + 1];
      }
      sc[kRouteMaxHubs - 1] = -1.0;
      yy[kRouteMaxHubs - 1] = INT32_MAX;
    }
    ++count;
  }
  if (lane == 0) {
    nhub[w] = emit ? count : 0;
    if (emit) lists[(1 + 2 * kRouteMaxHubs) * w] = kpx;
  }
}

// Flagged slot w becomes routed-row c = row_pos[w] with hubs from g = hub_pos[w] (exclusive sums of
// flag and nhub over the slots): arbitrage rows with j = x, i = p, in slot order, so in (base index,
// x) order.  Thread n_slots writes hub_off[n_rows].
__global__ void arb_rows_kernel(AdjView A, const int64_t* __restrict__ base, const int64_t* __restrict__ slot_off,
                                int64_t nb, const int64_t* __restrict__ flag, const int64_t* __restrict__ nhub,
                                const int32_t* __restrict__ hub, const int32_t* __restrict__ lists,
                                const int64_t* __restrict__ row_pos, const int64_t* __restrict__ hub_pos,
                                int64_t* __restrict__ token_in, int64_t* __restrict__ token_out,
                                int64_t* __restrict__ row_b, int64_t* __restrict__ hub_off,
                                int64_t* __restrict__ hubs, int64_t* __restrict__ pair) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n_slots = slot_off[nb];
  if (w == n_slots) hub_off[row_pos[n_slots]] = hub_pos[n_slots];
  if (w >= n_slots || !flag[w]) return;
  int64_t bl = 0, bh = nb;
  while (bh - bl > 1) {
    const int64_t mid = (bl + bh) >> 1;
    if (slot_off[mid] <= w)
      bl = mid;
    else
      bh = mid;
  }
  const int64_t c = row_pos[w], g = hub_pos[w], nh = nhub[w];
  const int64_t p = base[bl] - 1;
  token_in[c] = A.nbr[A.off[p] + (w - slot_off[bl])] + 1;
  token_out[c] = p + 1;
  row_b[c] = bl;
  hub_off[c] = g;
  const int32_t* L = lists + (1 + 2 * kRouteMaxHubs) * w;
  pair[c + 2 * g] = L[0];
  for (int64_t h = 0; h < nh; ++h) {
    hubs[g + h] = hub[kRouteMaxHubs * w + h] + 1;
    pair[c + 2 * g + 1 + 2 * h] = L[1 + 2 * h];
    pair[c + 2 * g + 2 + 2 * h] = L[2 + 2 * h];
  }
}

// Solved row c is kept when it filled with profit >= min_profit[its base]: keep[c] (and its sort key,
// the profit's bits complemented, so that an ascending sort puts the largest profit first).
__global__ void arb_keep_kernel(const uint8_t* __restrict__ status, const double* __restrict__ profit,
                                const int64_t* __restrict__ row_b, const double* __restrict__ min_profit, int64_t q,
                                int64_t* __restrict__ keep, uint64_t* __restrict__ key) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > q) return;
  if (c == q) {
    keep[c] = 0;
    return;
  }
  keep[c] = status[c] == 0 && profit[c] >= min_profit[row_b[c]];
  key[c] = ~(uint64_t)__double_as_longlong(profit[c]);
}

// Kept rows in (base index, x) order, compacted: sel[keep_pos[c]] = c, with its profit key.
__global__ void arb_select_kernel(const int64_t* __restrict__ keep_pos, const uint64_t* __restrict__ key, int64_t q,
                                  int64_t* __restrict__ sel, uint64_t* __restrict__ sel_key) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= q || keep_pos[c + 1] == keep_pos[c]) return;
  sel[keep_pos[c]] = c;
  sel_key[keep_pos[c]] = key[c];
}

// The base index of each row of v, the key of the second (stable) sort.
__global__ void arb_base_key_kernel(const int64_t* __restrict__ v, int64_t n, const int64_t* __restrict__ row_b,
                                    uint32_t* __restrict__ b) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) b[k] = (uint32_t)row_b[v[k]];
}

// Output row k of the first min(found, cap): the solved row sel[k].
__global__ void arb_output_kernel(const int64_t* __restrict__ sel, int64_t n, const int64_t* __restrict__ token_in,
                                  const int64_t* __restrict__ token_out, const int64_t* __restrict__ hub_off,
                                  const int64_t* __restrict__ hubs, const double* __restrict__ profit,
                                  const double* __restrict__ price, int64_t* __restrict__ o_base,
                                  int64_t* __restrict__ o_other, int64_t* __restrict__ o_count,
                                  int64_t* __restrict__ o_hubs, double* __restrict__ o_profit,
                                  double* __restrict__ o_price) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int64_t c = sel[k];
  o_base[k] = token_out[c];
  o_other[k] = token_in[c];
  const int64_t g = hub_off[c], nh = hub_off[c + 1] - g;
  o_count[k] = nh;
  for (int h = 0; h < kRouteMaxHubs; ++h) o_hubs[kRouteMaxHubs * k + h] = h < nh ? hubs[g + h] : 0;
  o_profit[k] = profit[c];
  o_price[k] = price[c];
}

}  // namespace cfmm
