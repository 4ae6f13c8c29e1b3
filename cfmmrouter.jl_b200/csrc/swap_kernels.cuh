// swap_kernels.cuh -- quotes and in-order execution of swaps against the device-resident pools
// (sm_90a; cfmm_quote_swaps / cfmm_execute_swaps, include/cfmm_b200.h).  Off the sweep path:
// no sweep kernel reads anything these kernels add.
//
// A row is a tender (x1, x2) of one pool, at most one side > 0.  With δ = γ·x (forward_trade's
// γ*Δ[1], src/cfmms.jl:445) the amount received on the other side is
//   ProductTwoCoin        forward_amount of the BoundedProduct (R₁R₂, 0, 0, R₁, R₂) (:411-414):
//                         λ₂ = min(R₂, R₂ − k/(R₁ + δ)), k = R₁·R₂
//   GeometricMeanTwoCoin  from the invariant R₁^w₁·R₂^w₂: λ₂ = R₂·(1 − (R₁/(R₁+δ))^η), η = w₁/w₂,
//                         evaluated as −R₂·expm1(−η·log1p(δ/R₁)) and clamped to [0, R₂]
//   UniV3                 forward_trade (:436-449): the tick walk of trade_through_pools over the
//                         upper ticks (token 1) or the flipped lower ticks (token 2)
// and symmetrically for a token-2 tender.  Execute moves a two-coin pool to (R + γΔ) − Λ (the
// operations of apply_trades_kernel) and a UniV3 pool to the price its walk ended at
// (univ3_walk).  Tender and received are in the pool's ingest token order; a ProductTwoCoin pool
// stored with its tokens exchanged (bit 62 of gidx) is exchanged on the way in and out.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "arb_math.cuh"
#include "univ3_state.cuh"

namespace cfmm {

// The arrays of one pool set (main or tail) the swap kernels read and write, in device order.
struct SwapSet {
  double2* R;             // two-coin reserves, stored order
  const double* gam;
  const double2* w;       // GeometricMeanTwoCoin weights (null for the other types)
  const int64_t* gidx;    // global insertion index; bit 62 = stored with its tokens exchanged
  const uint8_t* active;  // 0 = retired; null = every pool active
  Univ3State u;           // UniV3 only
};

// λ out of a two-coin pool for a net tender d of the token whose reserve is r_in (weights: w_in
// of the tendered token, w_out of the other; GeometricMeanTwoCoin only).
template <int TYPE>
__device__ __forceinline__ double two_coin_out(double r_in, double r_out, double d, double w_in, double w_out) {
  if constexpr (TYPE == 0) {
    const double k = __dmul_rn(r_in, r_out);
    const double l = __dsub_rn(r_out, __ddiv_rn(k, __dadd_rn(r_in, d)));
    return r_out < l ? r_out : l;  // min(R₂, λ) of forward_amount (NaN propagates as there)
  } else {
    const double eta = __ddiv_rn(w_in, w_out);
    const double u = __dmul_rn(eta, log1p(__ddiv_rn(d, r_in)));
    const double l = __dmul_rn(r_out, -expm1(-u));
    return l < 0.0 ? 0.0 : (l > r_out ? r_out : l);
  }
}

// Λ of the tender (x1, x2), both in stored order, against reserves r (stored order).
template <int TYPE>
__device__ __forceinline__ double2 two_coin_quote(double2 r, double g, double2 w, double x1, double x2) {
  if (x1 > 0.0) return make_double2(0.0, two_coin_out<TYPE>(r.x, r.y, __dmul_rn(g, x1), w.x, w.y));
  if (x2 > 0.0) return make_double2(two_coin_out<TYPE>(r.y, r.x, __dmul_rn(g, x2), w.y, w.x), 0.0);
  return make_double2(0.0, 0.0);
}

struct Univ3Walk {
  double lambda;  // received
  double price;   // q′ (== the start price when !moved)
  bool moved;
};

// forward_trade of one UniV3 pool (src/cfmms.jl:401-449) from the raw state: ticks lower[0..nt),
// liquidities liq[0..nt), at `price` with current tick cur (1-based), for the net tender d of
// token 1 (tok1) or token 2.  The walk visits cur, cur+1, .. nt (token 1) or cur, cur-1, .. 1
// (token 2, on the flipped ticks), each tick through univ3_compute_at_tick, and stops in the
// first tick whose max_amount_pos exceeds what is left of d.  max_amount_pos follows the
// reference's branch: an empty tick (k = 0) gives 0 rather than k/β − (R₁+α) = NaN.
// The new price (include/cfmm_b200.h, cfmm_execute_swaps): inside the ending tick idx with δ′
// left, y = (R₁+α) + δ′ and q′ = (k/y)/y (token 1) or y = (R₂+β) + δ′ and q′ = (y/k)·y (token 2),
// clamped to [lo(idx), hi(idx)]; after the walk exhausted every non-empty tick it reached, the
// far boundary of the last one (lo for token 1, hi for token 2); unchanged if it walked none.
__device__ __forceinline__ Univ3Walk univ3_walk(const double* lower, const double* liq, int nt, double price,
                                                int cur, double d, bool tok1) {
  Univ3Walk r;
  r.price = price;
  r.moved = false;
  double lam = 0.0;
  int last = 0;  // last non-empty tick walked (0 = none)
  const int step = tok1 ? 1 : -1;
  for (int idx = cur; tok1 ? idx <= nt : idx >= 1; idx += step) {
    const double hi = lower[idx - 1], lo = idx < nt ? lower[idx] : 0.0;
    const Univ3Tick t = univ3_compute_at_tick(liq[idx - 1], hi, lo, price, idx, cur);
    // flip_sides (src/cfmms.jl:289) for a token-2 tender
    const double a = tok1 ? t.alpha : t.beta, b = tok1 ? t.beta : t.alpha;
    const double r_in = tok1 ? t.R1 : t.R2, r_out = tok1 ? t.R2 : t.R1;
    const double ra = __dadd_rn(r_in, a);
    const double mx = b > 0.0 ? __dsub_rn(__ddiv_rn(t.k, b), ra) : (a > 0.0 ? __longlong_as_double(0x7ff0000000000000ll) : 0.0);
    if (mx > d) {
      const double y = __dadd_rn(ra, d);
      double l = __dsub_rn(__dadd_rn(r_out, b), __ddiv_rn(t.k, y));
      l = r_out < l ? r_out : l;
      r.lambda = __dadd_rn(lam, l);
      double q = tok1 ? __ddiv_rn(__ddiv_rn(t.k, y), y) : __dmul_rn(__ddiv_rn(y, t.k), y);
      q = q < lo ? lo : (q > hi ? hi : q);
      r.price = q;
      r.moved = true;
      return r;
    }
    lam = __dadd_rn(lam, r_out);
    d = __dsub_rn(d, mx);
    if (t.k != 0.0) last = idx;
  }
  r.lambda = lam;
  if (last > 0) {
    r.price = tok1 ? (last < nt ? lower[last] : 0.0) : lower[last - 1];
    r.moved = true;
  }
  return r;
}

// ---- exact-output rows and slippage limits (cfmm_quote_swaps_exact_out / cfmm_execute_swap_orders)
// f(x) is the exact-input quote of a tender x > 0 on one side at the pool's current state:
// two_coin_out with δ = γ·x, or univ3_walk(..., γ·x, ...).lambda.  swap_quote_kernel is f on a
// row's tendered side, so f is cfmm_quote_swaps bit for bit (a zero tender receives (0, 0)).
//
// An exact-output row wanting y > 0 takes x* with f(x*) >= y and f(pred(x*)) < y (or x* = 0),
// searched on the ordinals of the doubles in [0, DBL_MAX] (a double >= 0 read as an int64 is
// monotone in the double): from the closed-form estimate e, gallop 1, 2, 4, .. ordinals away from
// e until f brackets y, then bisect the bracket to adjacent doubles.  Every loop is bounded by the
// 63-bit ordinal range: at most 1 + 63 + 62 evaluations of f (include/cfmm_b200.h).

constexpr int64_t kSwapOrdMax = 0x7fefffffffffffffll;  // the ordinal of DBL_MAX

// The ordinal the search starts from: a NaN or non-positive estimate starts at the least
// subnormal, an infinite one at DBL_MAX.
__device__ __forceinline__ int64_t swap_start_ord(double e) {
  if (!(e > 0.0)) return 1;
  const int64_t o = __double_as_longlong(e);
  return o > kSwapOrdMax ? kSwapOrdMax : o;
}

// The ordinal of the crossing x* of f through y > 0 found from the estimate e; -1 when
// f(DBL_MAX) < y (unreachable).  f(0) = 0 < y is known and never evaluated.
template <class F>
__device__ __forceinline__ int64_t swap_crossing(const F& f, double y, double e) {
  const int64_t o = swap_start_ord(e);
  int64_t lo = 0, hi = o;
  if (f(__longlong_as_double(o)) >= y) {  // gallop down: hi stays a tender that reaches y
    for (int64_t step = 1; hi > 1; step <<= 1) {
      const int64_t c = hi - step;
      if (c <= 0) break;  // lo = 0
      if (f(__longlong_as_double(c)) >= y) {
        hi = c;
      } else {
        lo = c;
        break;
      }
    }
  } else {  // gallop up: lo stays a tender that falls short
    lo = o;
    for (int64_t step = 1;; step <<= 1) {
      if (lo == kSwapOrdMax) return -1;
      const int64_t c = kSwapOrdMax - lo <= step ? kSwapOrdMax : lo + step;
      if (f(__longlong_as_double(c)) >= y) {
        hi = c;
        break;
      }
      lo = c;
    }
  }
  while (hi - lo > 1) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (f(__longlong_as_double(mid)) >= y)
      hi = mid;
    else
      lo = mid;
  }
  return hi;
}

// The two-coin estimate of the tender that receives y from (r_in, r_out), fee γ (+inf when
// y >= r_out):  ProductTwoCoin        e = ((r_in·r_out)/(r_out − y) − r_in)/γ
//               GeometricMeanTwoCoin  e = (r_in·expm1(−log1p(−(y/r_out))/η))/γ, η = w_in/w_out
template <int TYPE>
__device__ __forceinline__ double two_coin_estimate(double r_in, double r_out, double g, double y, double w_in,
                                                    double w_out) {
  if (!(y < r_out)) return __longlong_as_double(0x7ff0000000000000ll);
  double d;
  if constexpr (TYPE == 0) {
    d = __dsub_rn(__ddiv_rn(__dmul_rn(r_in, r_out), __dsub_rn(r_out, y)), r_in);
  } else {
    const double eta = __ddiv_rn(w_in, w_out);
    d = __dmul_rn(r_in, expm1(__ddiv_rn(-log1p(-__ddiv_rn(y, r_out)), eta)));
  }
  return __ddiv_rn(d, g);
}

// The UniV3 estimate: the reverse of univ3_walk.  Walking the same ticks in the same direction,
// a tick whose R_out covers what is still wanted (y′ <= R_out) is inverted,
// δ′ = k/((R_out + β) − y′) − (R_in + α), and e = (s + δ′)/γ, where s sums the max_amount_pos of
// the ticks before it; any other tick adds its max_amount_pos to s and takes R_out off y′.  +inf
// when the ticks run out first.
__device__ __forceinline__ double univ3_estimate(const double* lower, const double* liq, int nt, double price,
                                                 int cur, double g, double y, bool tok1) {
  double s = 0.0;
  const int step = tok1 ? 1 : -1;
  for (int idx = cur; tok1 ? idx <= nt : idx >= 1; idx += step) {
    const double hi = lower[idx - 1], lo = idx < nt ? lower[idx] : 0.0;
    const Univ3Tick t = univ3_compute_at_tick(liq[idx - 1], hi, lo, price, idx, cur);
    const double a = tok1 ? t.alpha : t.beta, b = tok1 ? t.beta : t.alpha;
    const double r_in = tok1 ? t.R1 : t.R2, r_out = tok1 ? t.R2 : t.R1;
    const double ra = __dadd_rn(r_in, a);
    if (y <= r_out) {
      const double d = __dsub_rn(__ddiv_rn(t.k, __dsub_rn(__dadd_rn(r_out, b), y)), ra);
      return __ddiv_rn(__dadd_rn(s, d), g);
    }
    const double mx = b > 0.0 ? __dsub_rn(__ddiv_rn(t.k, b), ra) : (a > 0.0 ? __longlong_as_double(0x7ff0000000000000ll) : 0.0);
    s = __dadd_rn(s, mx);
    y = __dsub_rn(y, r_out);
  }
  return __longlong_as_double(0x7ff0000000000000ll);
}

// One pool at its current state, for every swap kernel: a tender of the ingest token tok1
// (token 1) or token 2.  f, estimate and the transition of one filled row.
template <int TYPE>
struct SwapPool {
  // two-coin
  double2 R, w;
  bool sw;
  // UniV3
  const double* lower;
  const double* liq;
  int nt, cur;
  double q;
  double g;

  __device__ __forceinline__ double f(double x, bool tok1) const {
    if constexpr (TYPE == 2) {
      return univ3_walk(lower, liq, nt, q, cur, __dmul_rn(g, x), tok1).lambda;
    } else {
      const bool in_x = tok1 != sw;  // the tender's reserve is R.x
      return two_coin_out<TYPE>(in_x ? R.x : R.y, in_x ? R.y : R.x, __dmul_rn(g, x), in_x ? w.x : w.y,
                                in_x ? w.y : w.x);
    }
  }

  __device__ __forceinline__ double estimate(double y, bool tok1) const {
    if constexpr (TYPE == 2) {
      return univ3_estimate(lower, liq, nt, q, cur, g, y, tok1);
    } else {
      const bool in_x = tok1 != sw;
      return two_coin_estimate<TYPE>(in_x ? R.x : R.y, in_x ? R.y : R.x, g, y, in_x ? w.x : w.y, in_x ? w.y : w.x);
    }
  }

  // x* for y > 0; +inf when unreachable
  __device__ __forceinline__ double exact_out(double y, bool tok1) const {
    const int64_t o = swap_crossing([&](double x) { return f(x, tok1); }, y, estimate(y, tok1));
    return o < 0 ? __longlong_as_double(0x7ff0000000000000ll) : __longlong_as_double(o);
  }

  // Execute a tender x > 0: two-coin reserves move to (R + γΔ) − Λ (apply_trade), a UniV3 pool to
  // the price its walk ended at and that price's current tick.  Returns what it received.
  __device__ __forceinline__ double execute(double x, bool tok1) {
    if constexpr (TYPE == 2) {
      const Univ3Walk wk = univ3_walk(lower, liq, nt, q, cur, __dmul_rn(g, x), tok1);
      if (wk.moved) {
        q = wk.price;
        cur = univ3_tick_of(lower, nt, q);
      }
      return wk.lambda;
    } else {
      const double d1 = tok1 != sw ? x : 0.0, d2 = tok1 != sw ? 0.0 : x;
      const double2 l = two_coin_quote<TYPE>(R, g, w, d1, d2);
      R = apply_trade(R, g, make_double2(d1, d2), l);
      return tok1 != sw ? l.y : l.x;
    }
  }
};

template <int TYPE>
__device__ __forceinline__ SwapPool<TYPE> swap_pool(const SwapSet& s, int64_t p) {
  SwapPool<TYPE> P;
  P.g = s.gam[p];
  if constexpr (TYPE == 2) {
    const int off = s.u.tick[p].x;
    P.nt = univ3_tick_end(s.u, p) - off;
    P.lower = s.u.lower + off;
    P.liq = s.u.liq + off;
    P.q = univ3_price(s.u, p);
    P.cur = s.u.tick[p].y;
  } else {
    P.R = s.R[p];
    P.w = TYPE == 1 ? s.w[p] : make_double2(0.0, 0.0);
    P.sw = (s.gidx[p] >> 62) & 1;
  }
  return P;
}

// ---- kernels, all over SwapPool
// Quotes (cfmm_quote_swaps): one thread per row.  rows[j] is the row's index in the call (tender / received
// [2·row, 2·row+1], ingest order), pos[j] its pool's device position in this set.  A retired pool
// or a zero tender receives (0, 0) and reads nothing of the pool.
template <int TYPE>
__global__ void swap_quote_kernel(SwapSet s, const int64_t* __restrict__ rows, const int64_t* __restrict__ pos,
                                  int64_t n, const double* __restrict__ tender, double* __restrict__ received) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t row = rows[j], p = pos[j];
  double2 out = make_double2(0.0, 0.0);
  if (!s.active || s.active[p]) {
    const double x1 = tender[2 * row], x2 = tender[2 * row + 1];
    if (x1 > 0.0 || x2 > 0.0) {
      const bool tok1 = x1 > 0.0;
      const double l = swap_pool<TYPE>(s, p).f(tok1 ? x1 : x2, tok1);
      out = tok1 ? make_double2(0.0, l) : make_double2(l, 0.0);
    }
  }
  received[2 * row] = out.x;
  received[2 * row + 1] = out.y;
}

// Execution (cfmm_execute_swaps): one thread per distinct pool.  seg_pos[k] is the k-th pool's device position, its
// rows are seg_rows[seg_off[k] .. seg_off[k+1]) in batch order.  The thread reads the pool's
// state once, applies the rows in order (each sees the ones before it), writes every row's
// received and the final state once.  Two-coin: *out_of_range is raised when a new reserve
// leaves the guard-free range.  UniV3: the new price goes to the price word of f1, and pools
// whose price changed are listed in moved (their derived state is rebuilt afterwards by
// univ3_current_tick_kernel / univ3_ticks_kernel, as after cfmm_apply_trades).
template <int TYPE>
__global__ void swap_execute_kernel(SwapSet s, const int64_t* __restrict__ seg_pos,
                                    const int64_t* __restrict__ seg_off, const int64_t* __restrict__ seg_rows,
                                    int64_t n_seg, const double* __restrict__ tender,
                                    double* __restrict__ received, int64_t* __restrict__ moved,
                                    unsigned long long* __restrict__ n_moved, int* __restrict__ out_of_range) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_seg) return;
  const int64_t p = seg_pos[k], r0 = seg_off[k], r1 = seg_off[k + 1];
  if (s.active && !s.active[p]) {  // retired: receives nothing, its parked state stays
    for (int64_t r = r0; r < r1; ++r) {
      const int64_t row = seg_rows[r];
      received[2 * row] = 0.0;
      received[2 * row + 1] = 0.0;
    }
    return;
  }
  SwapPool<TYPE> P = swap_pool<TYPE>(s, p);
  const double q0 = TYPE == 2 ? P.q : 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const int64_t row = seg_rows[r];
    const double x1 = tender[2 * row], x2 = tender[2 * row + 1];
    double2 out = make_double2(0.0, 0.0);
    if (x1 > 0.0 || x2 > 0.0) {
      const bool tok1 = x1 > 0.0;
      const double l = P.execute(tok1 ? x1 : x2, tok1);
      out = tok1 ? make_double2(0.0, l) : make_double2(l, 0.0);
    }
    received[2 * row] = out.x;
    received[2 * row + 1] = out.y;
  }
  if constexpr (TYPE == 2) {
    if (P.q != q0) {
      reinterpret_cast<double*>(s.u.f1 + p)[1] = P.q;
      moved[atomicAdd(n_moved, 1ull)] = p;
    }
  } else {
    s.R[p] = P.R;
    if (!in_fast_range(P.R.x) || !in_fast_range(P.R.y)) atomicOr(out_of_range, 1);
  }
}

// Exact-output quotes: one thread per row, addressed as in swap_quote_kernel.  want (0, y) tenders
// token 1, (y, 0) token 2; tender gets (x*, 0) or (0, x*), +inf for x* when y cannot be reached
// or the pool is retired, (0, 0) for y = 0.
template <int TYPE>
__global__ void swap_quote_exact_out_kernel(SwapSet s, const int64_t* __restrict__ rows,
                                            const int64_t* __restrict__ pos, int64_t n,
                                            const double* __restrict__ want, double* __restrict__ tender) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int64_t row = rows[j], p = pos[j];
  const double y1 = want[2 * row], y2 = want[2 * row + 1];
  double x = 0.0;
  const bool tok1 = y2 > 0.0;
  if (y1 > 0.0 || y2 > 0.0) {
    if (s.active && !s.active[p])
      x = __longlong_as_double(0x7ff0000000000000ll);
    else
      x = swap_pool<TYPE>(s, p).exact_out(tok1 ? y2 : y1, tok1);
  }
  tender[2 * row] = tok1 ? x : 0.0;
  tender[2 * row + 1] = tok1 ? 0.0 : x;
}

// Order rows: one thread per distinct pool, grouped as for swap_execute_kernel.  Each row, in
// batch order against the running state: kind 0 tenders its amount and reverts when it receives
// less than limit (0 without limits); kind 1 tenders x* for its wanted amount and reverts when y
// is unreachable or x* > limit (+inf without limits).  Only filled rows move the running state;
// the state and the moved list / out-of-range flag are written as swap_execute_kernel writes them.
template <int TYPE>
__global__ void swap_execute_orders_kernel(SwapSet s, const int64_t* __restrict__ seg_pos,
                                           const int64_t* __restrict__ seg_off, const int64_t* __restrict__ seg_rows,
                                           int64_t n_seg, const uint8_t* __restrict__ kind,
                                           const double* __restrict__ amount, const double* __restrict__ limit,
                                           double* __restrict__ paid, double* __restrict__ received,
                                           uint8_t* __restrict__ status, int64_t* __restrict__ moved,
                                           unsigned long long* __restrict__ n_moved, int* __restrict__ out_of_range) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_seg) return;
  const int64_t p = seg_pos[k], r0 = seg_off[k], r1 = seg_off[k + 1];
  const bool retired = s.active && !s.active[p];
  SwapPool<TYPE> P;
  if (!retired) P = swap_pool<TYPE>(s, p);
  const double q0 = TYPE == 2 && !retired ? P.q : 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const int64_t row = seg_rows[r];
    const double a1 = amount[2 * row], a2 = amount[2 * row + 1];
    const bool out = kind[row] == 1;
    const double inf = __longlong_as_double(0x7ff0000000000000ll);
    const double lim = limit ? limit[row] : (out ? inf : 0.0);
    const bool tok1 = out ? a2 > 0.0 : a1 > 0.0;  // the tender is token 1
    const double amt = a1 > 0.0 ? a1 : a2;
    double x = 0.0, lam = 0.0;
    uint8_t st = 0;  // CFMM_ORDER_FILLED
    if (retired) {
      st = 3;  // CFMM_ORDER_RETIRED
    } else if (!out) {
      x = amt;
      lam = x > 0.0 ? P.f(x, tok1) : 0.0;
      if (lam < lim) st = 1;  // CFMM_ORDER_LIMIT
    } else if (amt > 0.0) {
      x = P.exact_out(amt, tok1);
      if (x == inf) st = 2;  // CFMM_ORDER_UNREACHABLE
      else if (x > lim) st = 1;
    }
    if (st == 0) {
      if (x > 0.0) lam = P.execute(x, tok1);
    } else {
      x = 0.0;
      lam = 0.0;
    }
    paid[2 * row] = tok1 ? x : 0.0;
    paid[2 * row + 1] = tok1 ? 0.0 : x;
    received[2 * row] = tok1 ? 0.0 : lam;
    received[2 * row + 1] = tok1 ? lam : 0.0;
    status[row] = st;
  }
  if (retired) return;
  if constexpr (TYPE == 2) {
    if (P.q != q0) {
      reinterpret_cast<double*>(s.u.f1 + p)[1] = P.q;
      moved[atomicAdd(n_moved, 1ull)] = p;
    }
  } else {
    s.R[p] = P.R;
    if (!in_fast_range(P.R.x) || !in_fast_range(P.R.y)) atomicOr(out_of_range, 1);
  }
}

}  // namespace cfmm
