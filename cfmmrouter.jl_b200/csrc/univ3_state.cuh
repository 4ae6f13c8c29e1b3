// univ3_state.cuh -- the device-resident state of UniV3 pools (sm_90a): the per-tick
// BoundedProduct records the sweep walks read, rebuilt from the raw tick data (lower tick
// prices, liquidity, current price) at cfmm_finalize, on cfmm_update_univ3, on
// cfmm_apply_trades and on cfmm_modify_univ3_liquidity, whose ladder merge, row replay and CSR
// splice kernels are here too.  This is the library's only implementation of compute_at_tick
// (src/cfmms.jl:294-313).
//
// Raw state, kept on the device in the CSR order of the tick records (device pool order):
//   lower, liq : double[total_ticks]      16 B per tick
//   f1[p].y    : the pool's current price (the same word the sweep reads it from)
//   tick[p]    : (tick_off, current_tick 1-based)
// Derived state, rewritten in place (sweep graphs captured earlier keep valid pointers):
//   tickdata   : two 32-byte direction records per tick (arb_math.cuh, kTickStride)
//   f0..f3     : the current tick's records per pool (Univ3First)
//   tick[p].y  : current_tick
// A retired pool (cfmm_set_active; active[p] == 0) keeps its raw state; its derived records are
// built with zero liquidity, so every tick is is_empty_pool and the sweep trades nothing.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arb_math.cuh"

namespace cfmm {

struct Univ3State {
  double2* f0;          // (k, R_1+α) of the current tick
  double2* f1;          // (R_2+β, current_price)
  double2* f2;          // (δmax↑, R_2)
  double2* f3;          // (δmax↓, R_1)
  int2* tick;           // (tick_off, current_tick)
  double* tickdata;     // kTickStride doubles per tick
  const double* lower;  // CSR, strictly decreasing within a pool
  double* liq;          // CSR
  const uint8_t* active;  // device order, 0 = retired; null = every pool active
  int64_t m;
  int64_t total_ticks;
};

__device__ __forceinline__ double univ3_price(const Univ3State& s, int64_t p) {
  return reinterpret_cast<const double*>(s.f1 + p)[1];
}

__device__ __forceinline__ int univ3_tick_end(const Univ3State& s, int64_t p) {
  return p + 1 < s.m ? s.tick[p + 1].x : (int)s.total_ticks;
}

// searchsortedlast(lower_ticks, price, rev=true) (src/cfmms.jl:235) over one pool's nt ticks,
// i.e. the number of leading ticks >= price.  The ticks are strictly decreasing, so the leading
// run is found by bisection; ties count as >=, a NaN price gives 0 (both as the linear count).
__device__ __forceinline__ int univ3_tick_of(const double* lower, int nt, double price) {
  int lo = 0, hi = nt;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (lower[mid] >= price)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// The listed pool a listing-order tick t belongs to: the last j < count with cum[j] <= t.
__device__ __forceinline__ int64_t univ3_listed(const int64_t* cum, int64_t count, int64_t t) {
  int64_t lo = 0, hi = count - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (cum[mid] <= t)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// The number of entries of the ascending pos[0..count) that are < p.
__device__ __forceinline__ int64_t univ3_rank(const int64_t* pos, int64_t count, int64_t p) {
  int64_t lo = 0, hi = count;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (pos[mid] < p)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// current_tick of pools pos[j] (pos == nullptr: pool j), j < count, after an optional price
// push new_price[j] (univ3_tick_of).
__global__ void univ3_current_tick_kernel(Univ3State s, const int64_t* __restrict__ pos,
                                          const double* __restrict__ new_price, int64_t count) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  const int64_t p = pos ? pos[j] : j;
  double price;
  if (new_price) {
    price = new_price[j];
    reinterpret_cast<double*>(s.f1 + p)[1] = price;
  } else {
    price = univ3_price(s, p);
  }
  const int off = s.tick[p].x, nt = univ3_tick_end(s, p) - off;
  reinterpret_cast<int*>(s.tick + p)[1] = univ3_tick_of(s.lower + off, nt, price);
}

// One tick's BoundedProduct (src/cfmms.jl:272-278) from the raw state.
struct Univ3Tick {
  double k, alpha, beta, R1, R2;
};

// compute_at_tick (src/cfmms.jl:294-313): tick idx (1-based) of a pool at `price` whose current
// tick is cur, with liquidity k and bounds pplus = lower_ticks[idx], pminus = lower_ticks[idx+1]
// (0 for the last tick).  IEEE operations in the reference's order, written as intrinsics because
// nvcc contracts a*b+c to an FMA by default.  The library's only copy of this arithmetic: the
// tick records (univ3_ticks_kernel) and the swap walks (swap_kernels.cuh) both call it.
__device__ __forceinline__ Univ3Tick univ3_compute_at_tick(double k, double pplus, double pminus, double price,
                                                           int idx, int cur) {
  Univ3Tick t;
  t.k = k;
  t.alpha = __dsqrt_rn(__ddiv_rn(k, pplus));
  t.beta = __dsqrt_rn(__dmul_rn(k, pminus));
  const double pp = idx > cur ? pplus : (idx < cur ? pminus : price);
  t.R1 = __dsub_rn(__dsqrt_rn(__ddiv_rn(k, pp)), t.alpha);
  t.R2 = __dsub_rn(__dsqrt_rn(__dmul_rn(k, pp)), t.beta);
  return t;
}

// compute_at_tick (src/cfmms.jl:294-313) for every tick of pools pos[j] (pos == nullptr: of all
// pools), one thread per tick: cum[j] .. cum[j+1]-1 are the listed pools' ticks in listing order
// (cum == nullptr: the device CSR itself).  new_liq (optional, indexed like the listing) is
// stored first.  The records are bit-identical to compute_at_tick's (univ3_compute_at_tick).
__global__ void univ3_ticks_kernel(Univ3State s, const int64_t* __restrict__ pos,
                                   const int64_t* __restrict__ cum, int64_t count, int64_t n_ticks,
                                   const double* __restrict__ new_liq) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_ticks) return;
  int64_t p, ti;
  int off, nt;
  if (pos) {
    const int64_t lo = univ3_listed(cum, count, t);
    p = pos[lo];
    ti = t - cum[lo];
    off = s.tick[p].x;
    nt = (int)(cum[lo + 1] - cum[lo]);
  } else {
    int64_t lo = 0, hi = s.m - 1;  // last pool whose first tick is <= t (every pool has a tick)
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (s.tick[mid].x <= t)
        lo = mid;
      else
        hi = mid - 1;
    }
    p = lo;
    off = s.tick[p].x;
    ti = t - off;
    nt = univ3_tick_end(s, p) - off;
  }
  const int64_t q = off + ti;
  double k;
  if (new_liq) {
    k = new_liq[t];
    s.liq[q] = k;
  } else {
    k = s.liq[q];
  }
  if (s.active && !s.active[p]) k = 0.0;  // retired: empty ticks (the raw liquidity stays)
  const double price = univ3_price(s, p);
  const int cur = s.tick[p].y;
  const int idx = (int)ti + 1;  // 1-based
  const double pplus = s.lower[q];                            // tick_high_price :252
  const double pminus = ti + 1 < nt ? s.lower[q + 1] : 0.0;   // tick_low_price :255-259
  const Univ3Tick tk = univ3_compute_at_tick(k, pplus, pminus, price, idx, cur);
  const double alpha = tk.alpha, beta = tk.beta, R1 = tk.R1, R2 = tk.R2;
  const double ra = __dadd_rn(R1, alpha);
  const double rb = __dadd_rn(R2, beta);
  const double dmax_up = __dsub_rn(__ddiv_rn(k, beta), ra);
  const double dmax_dn = __dsub_rn(__ddiv_rn(k, alpha), rb);
  double2* up = reinterpret_cast<double2*>(s.tickdata + (size_t)off * kTickStride + (size_t)ti * 4);
  double2* dn = reinterpret_cast<double2*>(s.tickdata + (size_t)off * kTickStride + (size_t)(nt + ti) * 4);
  up[0] = make_double2(k, ra);
  up[1] = make_double2(dmax_up, R2);
  dn[0] = make_double2(k, rb);
  dn[1] = make_double2(dmax_dn, R1);
  if (idx == cur) {  // the tick a walk starts in: also per pool (the price word of f1 stays)
    s.f0[p] = make_double2(k, ra);
    reinterpret_cast<double*>(s.f1 + p)[0] = rb;
    s.f2[p] = make_double2(dmax_up, R2);
    s.f3[p] = make_double2(dmax_dn, R1);
  }
}

// The post-trade price of pool p of s (include/cfmm_b200.h, cfmm_apply_trades) at price q, fee g,
// for pr = ν[a]/ν[b]: the no-trade band exactly as univ3_arb computes it; the target p/γ (upper
// walk) or γ·p (lower walk), unchanged if it is NaN or not > 0, else clamped to the first lower
// tick.  Returns q when the price stays.  The first lower tick is only read for a target > 0.
__device__ __forceinline__ double univ3_moved_price(const Univ3State& s, int64_t p, double q, double g, double pr) {
  const double lo = __dmul_rn(g, q);
  if (lo <= pr && pr <= __ddiv_rn(q, g)) return q;
  const double target = pr < lo ? __ddiv_rn(pr, g) : __dmul_rn(g, pr);
  if (!(target > 0.0)) return q;
  const double t1 = s.lower[s.tick[p].x];
  return target < t1 ? target : t1;
}

// The post-trade price of every pool, from the ν of the last materialising sweep.  Pools whose
// price changes get it stored in f1 and are listed.
__global__ void univ3_move_kernel(Univ3State s, const double* __restrict__ gam, const int2* __restrict__ Ai,
                                  const double* __restrict__ nu, int64_t* __restrict__ moved,
                                  unsigned long long* __restrict__ n_moved) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= s.m) return;
  if (s.active && !s.active[p]) return;  // retired pools do not trade and do not move
  const double q = univ3_price(s, p);
  const int2 ai = Ai[p];
  const double qn = univ3_moved_price(s, p, q, gam[p], __ddiv_rn(nu[ai.x], nu[ai.y]));
  if (qn == q) return;
  reinterpret_cast<double*>(s.f1 + p)[1] = qn;
  moved[atomicAdd(n_moved, 1ull)] = p;
}

// ---- liquidity changes (cfmm_modify_univ3_liquidity; include/cfmm_b200.h) ---------------------
// The touched pools are listed in ascending device position: pos[j], their rows (indices into the
// call's range / dL, batch order) rows[row_off[j] .. row_off[j+1]), and their distinct candidate
// boundaries cand[cand_off[j] .. cand_off[j+1]), strictly decreasing.

// One pool's ladder merged with its candidates (out_lower == nullptr: counted only).  A candidate
// equal to a ladder boundary bit for bit adds nothing; any other one splits the tick it falls in
// and inherits that tick's liquidity, or 0 above T₁.  Returns the new tick count.
__device__ __forceinline__ int64_t univ3_merge_ladder(const double* lower, const double* liq, int nt,
                                                      const double* cand, int64_t nc, double* out_lower,
                                                      double* out_liq) {
  int a = 0;
  int64_t b = 0, n = 0;
  double inherit = 0.0;
  while (a < nt || b < nc) {
    double x, l;
    if (b == nc || (a < nt && lower[a] >= cand[b])) {
      if (b < nc && lower[a] == cand[b]) ++b;
      x = lower[a];
      l = inherit = liq[a];
      ++a;
    } else {
      x = cand[b];
      l = inherit;
      ++b;
    }
    if (out_lower) {
      out_lower[n] = x;
      out_liq[n] = l;
    }
    ++n;
  }
  return n;
}

// Stage A, one thread per touched pool: its new tick count (cum == nullptr) or its new ladder with
// inherited liquidities, written to out_lower / out_liq from cum[j] on (listing order).
__global__ void univ3_liq_ladder_kernel(Univ3State s, const int64_t* __restrict__ pos,
                                        const int64_t* __restrict__ cand_off, const double* __restrict__ cand,
                                        int64_t count, int64_t* __restrict__ new_nt, const int64_t* __restrict__ cum,
                                        double* __restrict__ out_lower, double* __restrict__ out_liq) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  const int64_t p = pos[j];
  const int off = s.tick[p].x, nt = univ3_tick_end(s, p) - off;
  const int64_t c0 = cand_off[j], nc = cand_off[j + 1] - c0;
  if (cum)
    univ3_merge_ladder(s.lower + off, s.liq + off, nt, cand + c0, nc, out_lower + cum[j], out_liq + cum[j]);
  else
    new_nt[j] = univ3_merge_ladder(s.lower + off, s.liq + off, nt, cand + c0, nc, nullptr, nullptr);
}

// Stage A, one thread per new tick: the pool's rows in batch order, each adding dL (one IEEE
// addition) when lo < T <= hi for the tick's upper bound T.  A tick left < 0 or not finite
// records its row in *first_bad (atomicMin: the call reports the lowest such row).
__global__ void univ3_liq_apply_kernel(const int64_t* __restrict__ cum, int64_t count, int64_t n_ticks,
                                       const int64_t* __restrict__ row_off, const int64_t* __restrict__ rows,
                                       const double* __restrict__ range, const double* __restrict__ dL,
                                       const double* __restrict__ new_lower, double* __restrict__ new_liq,
                                       unsigned long long* __restrict__ first_bad) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_ticks) return;
  const int64_t j = univ3_listed(cum, count, t);
  const double T = new_lower[t];
  double L = new_liq[t];
  for (int64_t k = row_off[j]; k < row_off[j + 1]; ++k) {
    const int64_t r = rows[k];
    if (range[2 * r] < T && T <= range[2 * r + 1]) {
      L = __dadd_rn(L, dL[r]);
      if (!(L >= 0.0 && isfinite(L))) {
        atomicMin(first_bad, (unsigned long long)r);
        return;
      }
    }
  }
  new_liq[t] = L;
}

// Stage B (tick counts changed), one thread per pool: its first tick in the new CSR, shifted by
// the growth of the touched pools before it (shift[k]: of the first k listed pools).
__global__ void univ3_splice_offsets_kernel(const int2* __restrict__ old_tick, int2* __restrict__ new_tick, int64_t m,
                                            const int64_t* __restrict__ pos, const int64_t* __restrict__ shift,
                                            int64_t count) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= m) return;
  new_tick[p] = make_int2((int)(old_tick[p].x + shift[univ3_rank(pos, count, p)]), 0);
}

// Stage B, one thread per tick of the new CSR: a touched pool's tick from the stage-A ladders
// (listing order, cum), any other pool's from the old CSR.
__global__ void univ3_splice_ticks_kernel(const int2* __restrict__ old_tick, const int2* __restrict__ new_tick,
                                          int64_t m, int64_t new_total, const int64_t* __restrict__ pos,
                                          const int64_t* __restrict__ cum, int64_t count,
                                          const double* __restrict__ scr_lower, const double* __restrict__ scr_liq,
                                          const double* __restrict__ old_lower, const double* __restrict__ old_liq,
                                          double* __restrict__ out_lower, double* __restrict__ out_liq) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= new_total) return;
  int64_t lo = 0, hi = m - 1;  // last pool whose first tick is <= t (every pool has a tick)
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (new_tick[mid].x <= t)
      lo = mid;
    else
      hi = mid - 1;
  }
  const int64_t p = lo, ti = t - new_tick[p].x, k = univ3_rank(pos, count, p);
  if (k < count && pos[k] == p) {
    out_lower[t] = scr_lower[cum[k] + ti];
    out_liq[t] = scr_liq[cum[k] + ti];
  } else {
    out_lower[t] = old_lower[old_tick[p].x + ti];
    out_liq[t] = old_liq[old_tick[p].x + ti];
  }
}

// cfmm_get_univ3_ticks, one thread per listed tick: the ladders of pools pos[j] in listing order.
__global__ void univ3_gather_ticks_kernel(Univ3State s, const int64_t* __restrict__ pos,
                                          const int64_t* __restrict__ cum, int64_t count, int64_t n_ticks,
                                          double* __restrict__ lower_out, double* __restrict__ liq_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_ticks) return;
  const int64_t j = univ3_listed(cum, count, t);
  const int64_t q = s.tick[pos[j]].x + (t - cum[j]);
  lower_out[t] = s.lower[q];
  liq_out[t] = s.liq[q];
}

}  // namespace cfmm
