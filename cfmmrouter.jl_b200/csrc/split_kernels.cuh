// split_kernels.cuh -- orders split across every pool of their token pair (sm_90a; cfmm_pair_pools /
// cfmm_quote_split_orders / cfmm_execute_split_orders, include/cfmm_b200.h).  Off the sweep path: no
// sweep kernel reads anything these kernels add.
//
// Pair index.  Every pool (all three types, main sets and tails) gets the key min(a,b)·n + max(a,b)
// of its 0-based token pair, written at its global insertion index (pair_key_kernel), with the value
// (set << 56) | device position.  A stable radix sort on the key and a run-length pass (cub, on the
// host side) give the CSR over distinct pairs: keys[0 .. n_pairs) ascending, the pair's pools
// pool[off[k] .. off[k+1]) in global insertion order.  Lookups bisect keys (pair_lookup_kernel).
//
// A row sells token j (token_in) for token i (token_out) over the pair's pools.  With ν_i = 1 and
// ν_j = s, pool k's legs are find_arb! at ν[Ai] (product_arb, geomean_arb, and the UniV3 walk of
// src/cfmms.jl:339-395 from the raw state); N(s) = Σ (Δ_j − Λ_j) and O(s) = Σ (Λ_i − Δ_i) in a fixed
// warp order (split_sums).  One warp runs the scalar search for s* of a row (split_row).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arb_math.cuh"
#include "path_kernels.cuh"
#include "sweep_kernels.cuh"
#include "univ3_state.cuh"

namespace cfmm {

// ---- pair index -------------------------------------------------------------------------------
constexpr int kPairSetShift = 56;  // a pair entry: (set << 56) | device position
constexpr int64_t kPairPosMask = (1ll << kPairSetShift) - 1;

__device__ __forceinline__ int64_t pair_key(int64_t a, int64_t b, int64_t n) {
  return a < b ? a * n + b : b * n + a;
}

// One thread per device position of set k: the key and entry of the pool there, at its global
// insertion index (padding positions, gidx < 0, write nothing).
__global__ void pair_key_kernel(const int2* __restrict__ Ai, const int64_t* __restrict__ gidx, int64_t m, int k,
                                int64_t n_tokens, int64_t* __restrict__ keys, int64_t* __restrict__ entries) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  const int64_t g = gidx[p];
  if (g < 0) return;
  const int64_t i = g & ~(1ll << 62);
  const int2 a = Ai[p];
  keys[i] = pair_key(a.x, a.y, n_tokens);
  entries[i] = ((int64_t)k << kPairSetShift) | p;
}

// Row r: the pair (ta[r], tb[r]) (1-based, distinct) as an index into keys (-1: no pool holds it)
// and its pool count.
__global__ void pair_lookup_kernel(const int64_t* __restrict__ keys, int64_t n_pairs, const int64_t* __restrict__ off,
                                   const int64_t* __restrict__ ta, const int64_t* __restrict__ tb, int64_t q,
                                   int64_t n_tokens, int64_t* __restrict__ pair, int64_t* __restrict__ count) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= q) return;
  const int64_t key = pair_key(ta[r] - 1, tb[r] - 1, n_tokens);
  int64_t lo = 0, hi = n_pairs;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (keys[mid] < key)
      lo = mid + 1;
    else
      hi = mid;
  }
  const bool hit = lo < n_pairs && keys[lo] == key;
  pair[r] = hit ? lo : -1;
  count[r] = hit ? off[lo + 1] - off[lo] : 0;
}

// cfmm_pair_pools, one thread per listed pool: rows' pools in row order (cum: exclusive sum of the
// rows' counts), as pair entries.
__global__ void pair_gather_kernel(const int64_t* __restrict__ off, const int64_t* __restrict__ pool,
                                   const int64_t* __restrict__ pair, const int64_t* __restrict__ cum, int64_t q,
                                   int64_t total, int64_t* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t r = univ3_listed(cum, q, t);  // the last row whose first listed pool is <= t
  out[t] = pool[off[pair[r]] + (t - cum[r])];
}

// ---- pool response at s -------------------------------------------------------------------------

// find_arb! of one UniV3 pool (src/cfmms.jl:339-395) at (v1, v2), walked from the raw state: every
// tick through univ3_compute_at_tick, the per-tick step through univ3_tick.  These are the values
// the tick records hold (univ3_ticks_kernel), so the result is univ3_arb's bit for bit, and it is
// right before the records of a pool that moved in this call are rebuilt.
__device__ __forceinline__ Trade univ3_arb_raw(const Univ3State& u, int64_t p, double g, double v1, double v2) {
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  const double q = univ3_price(u, p);
  const double pr = __ddiv_rn(v1, v2);
  const double lo = __dmul_rn(g, q);
  if (lo <= pr && pr <= __ddiv_rn(q, g)) return t;  // no-arb interval :347
  const bool up = pr < lo;
  const double price = __ddiv_rn(up ? pr : 1.0, up ? g : __dmul_rn(g, pr));
  const int off = u.tick[p].x, nt = univ3_tick_end(u, p) - off, cur = u.tick[p].y;
  const double* lower = u.lower + off;
  const double* liq = u.liq + off;
  double dsum = 0.0, lsum = 0.0;
  for (int idx = cur; up ? idx <= nt : idx >= 1; idx += up ? 1 : -1) {
    if (liq[idx - 1] == 0.0) continue;  // is_empty_pool: skipped, not terminal (:354-357, :376-379)
    const Univ3Tick k = univ3_compute_at_tick(liq[idx - 1], lower[idx - 1], idx < nt ? lower[idx] : 0.0, q, idx, cur);
    const double ra = __dadd_rn(k.R1, k.alpha), rb = __dadd_rn(k.R2, k.beta);
    if (!univ3_tick(
            k.k, up ? ra : rb, price, idx == cur,
            [&]() {
              return up ? make_double2(__dsub_rn(__ddiv_rn(k.k, k.beta), ra), k.R2)
                        : make_double2(__dsub_rn(__ddiv_rn(k.k, k.alpha), rb), k.R1);
            },
            [&]() { return up ? rb : ra; }, dsum, lsum))
      break;
  }
  const double dn = __ddiv_rn(dsum, g);
  if (up) {
    t.d1 = dn;
    t.l2 = lsum;
  } else {
    t.d2 = dn;
    t.l1 = lsum;
  }
  return t;
}

// One pool of a pair, as a row sees it: stored token pair, whether its stored token 1 is the row's
// j, whether it is stored with its tokens exchanged (two-coin, bit 62 of gidx), and active.
struct SplitPool {
  int k;
  int64_t p;
  bool x_is_j, sw, active;
  double v1, v2;  // ν at its stored tokens
};

__device__ __forceinline__ SplitPool split_pool(const PathSets* P, int64_t entry, int64_t tj, double s) {
  SplitPool sp;
  sp.k = (int)(entry >> kPairSetShift);
  sp.p = entry & kPairPosMask;
  const SwapSet& S = P->s[sp.k];
  const int2 a = P->Ai[sp.k][sp.p];
  sp.x_is_j = a.x == tj;
  sp.sw = (sp.k >> 1) < 2 && ((S.gidx[sp.p] >> 62) & 1);
  sp.active = !S.active || S.active[sp.p];
  sp.v1 = sp.x_is_j ? s : 1.0;
  sp.v2 = sp.x_is_j ? 1.0 : s;
  return sp;
}

// The pool's legs at s in its stored token order: the find_arb! a materialising sweep runs
// (sweep_kernel with exact = 0; the other closed forms give the same bits); (0, 0) when retired.
__device__ __forceinline__ Trade split_legs(const PathSets* P, const SplitPool& sp) {
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  if (!sp.active) return t;
  const SwapSet& S = P->s[sp.k];
  const double g = S.gam[sp.p];
  switch (sp.k >> 1) {
    case 0: {
      const double2 R = S.R[sp.p];
      return product_arb(R.x, R.y, g, sp.v1, sp.v2, false);
    }
    case 1: {
      const double2 R = S.R[sp.p], w = S.w[sp.p];
      return geomean_arb(R.x, R.y, w.x, w.y, g, sp.v1, sp.v2, false);
    }
    default:
      return univ3_arb_raw(S.u, sp.p, g, sp.v1, sp.v2);
  }
}

// The s below which the pool starts to take j (include/cfmm_b200.h); NaN when retired.
__device__ __forceinline__ double split_boundary(const PathSets* P, const SplitPool& sp) {
  if (!sp.active) return __longlong_as_double(0x7ff8000000000000ll);
  const SwapSet& S = P->s[sp.k];
  const double g = S.gam[sp.p];
  if ((sp.k >> 1) == 2) {
    const double q = univ3_price(S.u, sp.p);
    return sp.x_is_j ? __dmul_rn(g, q) : __ddiv_rn(g, q);
  }
  const double2 R = S.R[sp.p];
  const double ri = sp.x_is_j ? R.y : R.x, rj = sp.x_is_j ? R.x : R.y;
  if ((sp.k >> 1) == 0) return __ddiv_rn(__dmul_rn(g, ri), rj);
  const double2 w = S.w[sp.p];
  const double wi = sp.x_is_j ? w.y : w.x, wj = sp.x_is_j ? w.x : w.y;
  return __ddiv_rn(__dmul_rn(__dmul_rn(g, wj), ri), __dmul_rn(wi, rj));
}

struct SplitSums {
  double n, o;  // N(s): net intake of j; O(s): output of i
};

// N(s) and O(s) over the pair's pools pools[0 .. cnt), warp-wide: lane l sums the terms of pools
// l, l + 32, … from +0.0, then the xor butterfly 16, 8, 4, 2, 1 (every lane ends with the same bits).
__device__ __forceinline__ SplitSums split_sums(const PathSets* P, const int64_t* pools, int64_t cnt, int64_t tj,
                                                double s, int lane) {
  double n = 0.0, o = 0.0;
  for (int64_t t = lane; t < cnt; t += 32) {
    const SplitPool sp = split_pool(P, pools[t], tj, s);
    const Trade tr = split_legs(P, sp);
    n = __dadd_rn(n, sp.x_is_j ? __dsub_rn(tr.d1, tr.l1) : __dsub_rn(tr.d2, tr.l2));
    o = __dadd_rn(o, sp.x_is_j ? __dsub_rn(tr.l2, tr.d2) : __dsub_rn(tr.l1, tr.d1));
  }
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    n = __dadd_rn(n, __shfl_xor_sync(kFull, n, m));
    o = __dadd_rn(o, __shfl_xor_sync(kFull, o, m));
  }
  return {n, o};
}

// ---- one row ------------------------------------------------------------------------------------
constexpr int64_t kSplitOrdMin = 0x0010000000000000ll;  // the ordinal of DBL_MIN
constexpr int64_t kSplitOrdMax = kSwapOrdMax;           // DBL_MAX

// The search of a row's s* (and of a hub's t_h, route_kernels.cuh) on the ordinals
// [kSplitOrdMin, kSplitOrdMax], from o: gallop 1, 2, 4, … ordinals up or down, then bisect.
// test(c) evaluates at c and returns enough(c) (true at small c); keep(is_lo) files that evaluation
// as lo's or hi's.  0: a bracket, enough(lo), !enough(hi), hi = lo + 1.  1: enough at o(DBL_MAX)
// (lo = o(DBL_MAX)).  2: !enough at o(DBL_MIN) (hi = o(DBL_MIN)).  At most 1 + 63 + 62 tests.
template <class Test, class Keep>
__device__ __forceinline__ int split_search(int64_t o, int64_t& lo, int64_t& hi, Test&& test, Keep&& keep) {
  if (test(o)) {
    lo = o;
    keep(true);
    for (int64_t step = 1;; step <<= 1) {
      if (lo == kSplitOrdMax) return 1;
      const int64_t c = kSplitOrdMax - lo <= step ? kSplitOrdMax : lo + step;
      if (test(c)) {
        lo = c;
        keep(true);
      } else {
        hi = c;
        keep(false);
        break;
      }
    }
  } else {
    hi = o;
    keep(false);
    for (int64_t step = 1;; step <<= 1) {
      if (hi == kSplitOrdMin) return 2;
      const int64_t c = hi - kSplitOrdMin <= step ? kSplitOrdMin : hi - step;
      if (test(c)) {
        lo = c;
        keep(true);
        break;
      }
      hi = c;
      keep(false);
    }
  }
  while (hi - lo > 1) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (test(mid)) {
      lo = mid;
      keep(true);
    } else {
      hi = mid;
      keep(false);
    }
  }
  return 0;
}

// The ordinal a search starts from: o(e) clamped to [o(DBL_MIN), o(DBL_MAX)], o(DBL_MIN) for a NaN.
__device__ __forceinline__ int64_t split_start(double e) {
  const int64_t o = !(e >= 0x1p-1022) ? kSplitOrdMin : __double_as_longlong(e);
  return o > kSplitOrdMax ? kSplitOrdMax : o;
}

// The rows of one call (device arrays, row-indexed; tokens 1-based).
struct SplitRows {
  const int64_t* token_in;
  const int64_t* token_out;
  const uint8_t* kind;
  const double* amount;
  const double* limit;    // null: none
  const int64_t* pair;    // index into the pair index, -1: no pool holds the pair
  const int64_t* leg_off; // [q+1]: row r's legs are leg_off[r] .. leg_off[r+1])
  double* paid;
  double* received;
  double* price;
  uint8_t* status;
  double* leg_delta;      // [2L] or null
  double* leg_lambda;
};

struct PairIndexView {
  const int64_t* off;
  const int64_t* pool;
};

// The UniV3 pools a filled row moved (one flag per device position of each UniV3 set, so a pool
// moved by several rows is listed once).
struct SplitMoved {
  uint8_t* flag[2];
};

// A row's last pass over one of its pools (split_row, route_row).  For a filled row, the pool
// pool() builds at the row's ν: its legs; on EXEC, for an active pool, cfmm_apply_trades'
// transition (two-coin: apply_trade and the out-of-range flag; UniV3: univ3_moved_price and the
// new current tick written in place, the pool listed once per call).  The legs, (0, 0) when the
// row did not fill or the pool is retired, go in ingest order to leg l when leg_delta is set.
template <bool EXEC, class Pool>
__device__ __forceinline__ void split_leg(const PathSets* P, bool filled, Pool&& pool, const SplitMoved& mv,
                                          double* leg_delta, double* leg_lambda, int64_t l) {
  Trade tr;
  tr.d1 = tr.d2 = tr.l1 = tr.l2 = 0.0;
  if (filled) {
    const SplitPool sp = pool();
    tr = split_legs(P, sp);
    if (EXEC && sp.active) {
      const SwapSet& S = P->s[sp.k];
      if ((sp.k >> 1) < 2) {
        const double2 n = apply_trade(S.R[sp.p], S.gam[sp.p], make_double2(tr.d1, tr.d2), make_double2(tr.l1, tr.l2));
        S.R[sp.p] = n;
        if (!in_fast_range(n.x) || !in_fast_range(n.y)) P->out_of_range[sp.k] = 1;
      } else {
        const double q = univ3_price(S.u, sp.p);
        const double qn = univ3_moved_price(S.u, sp.p, q, S.gam[sp.p], __ddiv_rn(sp.v1, sp.v2));
        if (qn != q) {
          const int off = S.u.tick[sp.p].x;
          reinterpret_cast<double*>(S.u.f1 + sp.p)[1] = qn;
          reinterpret_cast<int*>(S.u.tick + sp.p)[1] =
              univ3_tick_of(S.u.lower + off, univ3_tick_end(S.u, sp.p) - off, qn);
          uint8_t* f = mv.flag[sp.k & 1];
          if (!f[sp.p]) {  // rows of one launch share no pool, so the check and the set do not race
            f[sp.p] = 1;
            P->moved[sp.k & 1][atomicAdd(P->n_moved + (sp.k & 1), 1ull)] = sp.p;
          }
        }
      }
      P->touched[sp.k] = 1;
    }
    if (sp.sw) {
      const double d = tr.d1, lm = tr.l1;
      tr.d1 = tr.d2;
      tr.l1 = tr.l2;
      tr.d2 = d;
      tr.l2 = lm;
    }
  }
  if (leg_delta) {
    leg_delta[2 * l] = tr.d1;
    leg_delta[2 * l + 1] = tr.d2;
    leg_lambda[2 * l] = tr.l1;
    leg_lambda[2 * l + 1] = tr.l2;
  }
}

// Row `row` on the current state of its pair's pools, warp-wide (every lane takes every branch).
// EXEC: the limit decides, and a filled row applies cfmm_apply_trades' transition at its ν to each
// of the pair's pools.
template <bool EXEC>
__device__ __forceinline__ void split_row(const PathSets* P, const PairIndexView& ix, const SplitRows& R, int64_t row,
                                          const SplitMoved& mv, int lane) {
  const int64_t pr = R.pair[row];
  const int64_t* pools = pr >= 0 ? ix.pool + ix.off[pr] : nullptr;
  const int64_t cnt = pr >= 0 ? ix.off[pr + 1] - ix.off[pr] : 0;
  const int64_t tj = R.token_in[row] - 1;
  const bool out = R.kind[row] == 1;
  const double amt = R.amount[row];
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  const double lim = R.limit ? R.limit[row] : (out ? inf : 0.0);
  uint8_t st = 0;  // CFMM_ORDER_FILLED
  double s = 0.0;
  SplitSums at = {0.0, 0.0};
  if (amt > 0.0) {
    // start: the largest no-trade boundary over the active pools
    double e = -inf;
    bool any = false;
    for (int64_t t = lane; t < cnt; t += 32) {
      const SplitPool sp = split_pool(P, pools[t], tj, 1.0);
      const double b = split_boundary(P, sp);
      any = any || sp.active;
      e = b > e ? b : e;
    }
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) {
      const double o = __shfl_xor_sync(kFull, e, m);
      e = o > e ? o : e;
    }
    if (!__any_sync(kFull, any)) {
      st = 2;  // CFMM_ORDER_UNREACHABLE
    } else {
      SplitSums r, slo = at, shi = at;
      int64_t lo = 0, hi = 0;
      const int rc = split_search(
          split_start(e), lo, hi,
          [&](int64_t c) {
            r = split_sums(P, pools, cnt, tj, __longlong_as_double(c), lane);
            return out ? r.o >= amt : !(r.n <= amt);  // exact-in: N > δ, a NaN counts as true
          },
          [&](bool is_lo) { (is_lo ? slo : shi) = r; });
      if (rc != 0) {
        st = 2;
      } else {
        s = __longlong_as_double(out ? lo : hi);
        at = out ? slo : shi;
        if (EXEC && (out ? at.n > lim : at.o < lim)) st = 1;  // CFMM_ORDER_LIMIT; an equal limit fills
      }
    }
  }
  const bool filled = st == 0 && amt > 0.0;
  // legs (ingest order) and, on execute, the transition of each pool
  const int64_t l0 = R.leg_off[row];
  for (int64_t t = lane; t < cnt; t += 32)
    split_leg<EXEC>(P, filled, [&] { return split_pool(P, pools[t], tj, s); }, mv, R.leg_delta, R.leg_lambda, l0 + t);
  __syncwarp();  // the next row of this warp reads the state the lanes just wrote
  if (lane == 0) {
    R.paid[row] = filled ? at.n : 0.0;
    R.received[row] = filled ? at.o : 0.0;
    R.price[row] = st == 2 ? 0.0 : s;
    R.status[row] = st;
  }
}

constexpr int kSplitThreads = 256;

// Quotes: one warp per row, every row on the current state on its own.
__global__ void __launch_bounds__(kSplitThreads) split_quote_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                    SplitRows R, int64_t q) {
  const int64_t w = ((int64_t)blockIdx.x * kSplitThreads + threadIdx.x) >> 5;
  if (w >= q) return;
  split_row<false>(P, ix, R, w, SplitMoved{}, threadIdx.x & 31);
}

// Execution: one warp per distinct pair (a pool belongs to one pair, so warps share no pool); its rows
// seg_rows[seg_off[w] .. seg_off[w+1]) run in batch order, each on the state the earlier ones left.
__global__ void __launch_bounds__(kSplitThreads) split_execute_kernel(const PathSets* __restrict__ P, PairIndexView ix,
                                                                      SplitRows R, const int64_t* __restrict__ seg_off,
                                                                      const int64_t* __restrict__ seg_rows,
                                                                      int64_t n_seg, SplitMoved mv) {
  const int64_t w = ((int64_t)blockIdx.x * kSplitThreads + threadIdx.x) >> 5;
  if (w >= n_seg) return;
  for (int64_t r = seg_off[w]; r < seg_off[w + 1]; ++r) split_row<true>(P, ix, R, seg_rows[r], mv, threadIdx.x & 31);
}

}  // namespace cfmm
