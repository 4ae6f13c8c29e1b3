// arb_math.cuh -- per-pool closed-form arbitrage, fp64, device side.
//
// Each function names the reference lines it reproduces (paths relative to the
// CFMMRouter.jl tree).  Every arithmetic step that the reference performs is
// written with an explicitly rounded intrinsic (__dmul_rn, __ddiv_rn, ...) so
// that nvcc can never contract a*b+c into an FMA: the reference (Julia) does
// not fuse, and ProductTwoCoin / UniV3 results are therefore bit-identical to
// an IEEE evaluation of the reference's expressions in the reference's order.
#pragma once
#include <cuda_runtime.h>

namespace cfmm {

struct Trade {
  double d1, d2;  // Δ[1], Δ[2]  (tendered)
  double l1, l2;  // Λ[1], Λ[2]  (received)
};

// R <- (R + γ·Δ) − Λ (the update the reference's tests use, test/cfmms.jl:10: R⁺ = R + γ*Δ - Λ)
__device__ __forceinline__ double2 apply_trade(double2 r, double g, double2 d, double2 l) {
  double2 n;
  n.x = __dsub_rn(__dadd_rn(r.x, __dmul_rn(g, d.x)), l.x);
  n.y = __dsub_rn(__dadd_rn(r.y, __dmul_rn(g, d.y)), l.y);
  return n;
}

// Julia's max(x, 0) on Float64: NaN propagates; max(-0.0, 0) == +0.0.
__device__ __forceinline__ double jl_max0(double x) {
  return (x != x) ? x : (x > 0.0 ? x : 0.0);
}

// Margins of the side-selection predicates.  A side is skipped only when the
// exact-arithmetic sign of its closed form is decided by a relative margin
// that dwarfs the few-ulp rounding error of the reference expression; ties
// inside the margin take the full reference form, so results stay identical.
constexpr double kProdHi = 1.0 + 0x1p-40;
constexpr double kProdLo = 1.0 - 0x1p-40;
constexpr double kGeoHi = 1.0 + 0x1p-30;
constexpr double kGeoLo = 1.0 - 0x1p-30;
// The side-selection certificates (and the guard-free div/sqrt of
// product_tma.cuh) assume that no intermediate of the reference expression
// underflows or overflows.  With every input in [2^-100, 2^101) all products,
// quotients and roots of the ProductTwoCoin forms stay within 2^±510.
__device__ __forceinline__ bool in_fast_range(double v) {
  return (unsigned)(__double2hiint(v) - 0x39B00000) < (0x46400000u - 0x39B00000u);
}
// tighter window for the GeometricMean forms (powers up to r^24): [2^-32, 2^32)
__device__ __forceinline__ bool in_geo_range(double v) {
  return (unsigned)(__double2hiint(v) - 0x3DF00000) < (0x41F00000u - 0x3DF00000u);
}

// ---------------------------------------------------------------------------
// ProductTwoCoin -- src/cfmms.jl:125-126 (prod_arb_δ / prod_arb_λ), :130-140
// ---------------------------------------------------------------------------

// All four closed forms exactly as written in the reference.
__device__ __forceinline__ Trade product_full(double R1, double R2, double g,
                                              double v1, double v2) {
  Trade t;
  const double k = __dmul_rn(R1, R2);               // k = R[1]*R[2]      :132
  const double m21 = __ddiv_rn(v2, v1);             // v[2]/v[1]
  const double m12 = __ddiv_rn(v1, v2);             // v[1]/v[2]
  const double g21 = __dmul_rn(g, m21);             // γ*m == m*γ bitwise
  const double g12 = __dmul_rn(g, m12);
  // prod_arb_δ(m, r, k, γ) = max(sqrt(γ*m*k) - r, 0)/γ                  :125
  t.d1 = __ddiv_rn(jl_max0(__dsub_rn(__dsqrt_rn(__dmul_rn(g21, k)), R1)), g);
  t.d2 = __ddiv_rn(jl_max0(__dsub_rn(__dsqrt_rn(__dmul_rn(g12, k)), R2)), g);
  // prod_arb_λ(m, r, k, γ) = max(r - sqrt(k/(m*γ)), 0)                  :126
  t.l1 = jl_max0(__dsub_rn(R1, __dsqrt_rn(__ddiv_rn(k, g12))));
  t.l2 = jl_max0(__dsub_rn(R2, __dsqrt_rn(__ddiv_rn(k, g21))));
  return t;
}

// Same results, evaluating only the side that can be non-zero.
//   Δ1, Λ2 > 0  <=>  γ·v2·R2 > v1·R1        (pool underprices token 1)
//   Δ2, Λ1 > 0  <=>  γ·v1·R1 > v2·R2
// and with γ <= 1 at most one holds.  The non-zero pair shares γ·m, so it
// costs 3 div + 2 sqrt instead of 6 div + 4 sqrt.
// A pool without reserves (a padding pool of the device layout, a retired pool) trades nothing at
// any price; the full forms would give NaN for it where a price is 0, ∞ or NaN (sqrt(∞·0), 0/0).
__device__ __forceinline__ Trade product_arb(double R1, double R2, double g,
                                             double v1, double v2, bool exact) {
  const bool no_reserves = R1 == 0.0 && R2 == 0.0;
  if (exact && !no_reserves) return product_full(R1, R2, g, v1, v2);
  const double uA = __dmul_rn(v1, R1);
  const double uB = __dmul_rn(v2, R2);
  const double tA = __dmul_rn(g, uB);
  const double tB = __dmul_rn(g, uA);
  const bool sane = in_fast_range(R1) && in_fast_range(R2) && in_fast_range(g) &&
                    in_fast_range(v1) && in_fast_range(v2);
  const bool zA = tA < __dmul_rn(uA, kProdLo);  // Δ1 = Λ2 = 0 for certain
  const bool zB = tB < __dmul_rn(uB, kProdLo);  // Δ2 = Λ1 = 0 for certain
  const bool fA = (tA > __dmul_rn(uA, kProdHi)) && zB;
  const bool fB = (tB > __dmul_rn(uB, kProdHi)) && zA;
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  if (sane && (fA || fB)) {
    const double ra = fA ? R1 : R2;  // reserve of the tendered token
    const double rb = fA ? R2 : R1;  // reserve of the received token
    const double m = fA ? __ddiv_rn(v2, v1) : __ddiv_rn(v1, v2);
    const double k = __dmul_rn(R1, R2);
    const double gm = __dmul_rn(g, m);
    const double da =
        __ddiv_rn(jl_max0(__dsub_rn(__dsqrt_rn(__dmul_rn(gm, k)), ra)), g);
    const double lb = jl_max0(__dsub_rn(rb, __dsqrt_rn(__ddiv_rn(k, gm))));
    if (fA) {
      t.d1 = da;
      t.l2 = lb;
    } else {
      t.d2 = da;
      t.l1 = lb;
    }
    return t;
  }
  if ((sane && zA && zB) || no_reserves) return t;  // strictly inside the no-trade band, or no pool
  return product_full(R1, R2, g, v1, v2);
}

// ---------------------------------------------------------------------------
// GeometricMeanTwoCoin -- src/cfmms.jl:180-181 (geom_arb_δ / geom_arb_λ), :185-196
// ---------------------------------------------------------------------------

// geom_arb_δ(m,r1,r2,η,γ) = max((γ*m*η*r1*r2^η)^(1/(η+1)) - r2, 0)/γ      :180
__device__ __forceinline__ double geom_arb_delta(double m, double r1, double r2,
                                                 double e, double g) {
  const double base = __dmul_rn(
      __dmul_rn(__dmul_rn(__dmul_rn(g, m), e), r1), pow(r2, e));
  const double ex = __ddiv_rn(1.0, __dadd_rn(e, 1.0));
  return __ddiv_rn(jl_max0(__dsub_rn(pow(base, ex), r2)), g);
}
// geom_arb_λ(m,r1,r2,η,γ) = max(r1 - ((r2*r1^(1/η))/(η*γ*m))^(η/(1+η)), 0) :181
__device__ __forceinline__ double geom_arb_lambda(double m, double r1,
                                                  double r2, double e,
                                                  double g) {
  const double base = __ddiv_rn(__dmul_rn(r2, pow(r1, __ddiv_rn(1.0, e))),
                                __dmul_rn(__dmul_rn(e, g), m));
  const double ex = __ddiv_rn(e, __dadd_rn(1.0, e));
  return jl_max0(__dsub_rn(r1, pow(base, ex)));
}

__device__ __forceinline__ Trade geomean_full(double R1, double R2, double w1,
                                              double w2, double g, double v1,
                                              double v2) {
  Trade t;
  const double eta = __ddiv_rn(w1, w2);     // η = w[1]/w[2]               :188
  const double etai = __ddiv_rn(1.0, eta);  // 1/η
  const double m21 = __ddiv_rn(v2, v1);
  const double m12 = __ddiv_rn(v1, v2);
  t.d1 = geom_arb_delta(m21, R2, R1, eta, g);    // :190
  t.d2 = geom_arb_delta(m12, R1, R2, etai, g);   // :191
  t.l1 = geom_arb_lambda(m12, R1, R2, etai, g);  // :193
  t.l2 = geom_arb_lambda(m21, R2, R1, eta, g);   // :194
  return t;
}

//   Δ1, Λ2 > 0  <=>  γ·v2·w1·R2 > v1·w2·R1 ;   Δ2, Λ1 > 0  <=>  γ·v1·w2·R1 > v2·w1·R2
// Evaluating only the live side costs 4 pow instead of 8.
__device__ __forceinline__ Trade geomean_arb(double R1, double R2, double w1,
                                             double w2, double g, double v1,
                                             double v2, bool exact) {
  if (exact) return geomean_full(R1, R2, w1, w2, g, v1, v2);
  const double uA = __dmul_rn(__dmul_rn(v1, w2), R1);
  const double uB = __dmul_rn(__dmul_rn(v2, w1), R2);
  const double tA = __dmul_rn(g, uB);
  const double tB = __dmul_rn(g, uA);
  const double eta = __ddiv_rn(w1, w2);
  // the margin argument needs a moderate exponent, (t/u)^(1/(η+1)), and no
  // overflow/underflow inside the powers: inputs in [2^-32, 2^32), η in [1/24, 24]
  const bool sane = in_geo_range(R1) && in_geo_range(R2) && in_geo_range(v1) &&
                    in_geo_range(v2) && in_geo_range(g) && (eta > 1.0 / 24.0) && (eta < 24.0);
  const bool zA = tA < __dmul_rn(uA, kGeoLo);
  const bool zB = tB < __dmul_rn(uB, kGeoLo);
  const bool fA = (tA > __dmul_rn(uA, kGeoHi)) && zB;
  const bool fB = (tB > __dmul_rn(uB, kGeoHi)) && zA;
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  if (sane && (fA || fB)) {
    const double m = fA ? __ddiv_rn(v2, v1) : __ddiv_rn(v1, v2);
    const double r1 = fA ? R2 : R1;
    const double r2 = fA ? R1 : R2;
    const double e = fA ? eta : __ddiv_rn(1.0, eta);
    const double d = geom_arb_delta(m, r1, r2, e, g);   // Δ of r2's token
    const double l = geom_arb_lambda(m, r1, r2, e, g);  // Λ of r1's token
    if (fA) {
      t.d1 = d;
      t.l2 = l;
    } else {
      t.d2 = d;
      t.l1 = l;
    }
    return t;
  }
  if (sane && zA && zB) return t;
  return geomean_full(R1, R2, w1, w2, g, v1, v2);
}

// Economized GeometricMean trade for gradient-only sweeps (per-pool values not
// observable; see product_tma.cuh for the argument).  With the traded side
// chosen as above, t = num/den = γ·m·e·r1/r2 > 1 and u = t^(1/(e+1)):
//     Δ_tendered = r2·(u − 1)/γ ,   Λ_received = r1·(1 − u/t)
// which is src/cfmms.jl:180-181 with r2 and r1 factored out of the powers
// (1/(e+1) = w_received/(w1+w2)).  One pow instead of four.
// LOG2EXP2: u = exp2(ex·log2(ratio)) instead of pow(ratio, ex); the default of gradient-only
// sweeps (option "geomean_log2" = 1, on this kernel and on the TMA kernel).  The absolute error
// of ex·log2(ratio) grows with |log2 ratio| (<= 64 in the admitted range) and becomes a relative
// error of u.  Measured per flow on an H100 80GB HBM3 against extended precision, in units of
// eps·(R + γ|flow|)/γ: <= 1.4 + 2·|ex·log2 ratio|, 38.4 at most (tests/test_gpu_pool_readout.py).
template <bool LOG2EXP2 = false>
__device__ __forceinline__ Trade geomean_arb_econ(double R1, double R2, double w1,
                                                  double w2, double g, double v1,
                                                  double v2) {
  const double uA = __dmul_rn(__dmul_rn(v1, w2), R1);
  const double uB = __dmul_rn(__dmul_rn(v2, w1), R2);
  const double tA = __dmul_rn(g, uB);
  const double tB = __dmul_rn(g, uA);
  const double eta = __ddiv_rn(w1, w2);
  const bool sane = in_geo_range(R1) && in_geo_range(R2) && in_geo_range(v1) &&
                    in_geo_range(v2) && in_geo_range(g) && (eta > 1.0 / 24.0) && (eta < 24.0);
  const bool zA = tA < __dmul_rn(uA, kGeoLo);
  const bool zB = tB < __dmul_rn(uB, kGeoLo);
  const bool fA = (tA > __dmul_rn(uA, kGeoHi)) && zB;
  const bool fB = (tB > __dmul_rn(uB, kGeoHi)) && zA;
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  if (sane && (fA || fB)) {
    const double num = fA ? tA : tB;
    const double den = fA ? uA : uB;
    const double ra = fA ? R1 : R2;  // reserve of the tendered token
    const double rb = fA ? R2 : R1;  // reserve of the received token
    const double ratio = num / den;
    const double ex = (fA ? w2 : w1) / (w1 + w2);
    double u;
    if constexpr (LOG2EXP2)
      u = exp2(ex * log2(ratio));
    else
      u = pow(ratio, ex);
    const double d = ra * (u - 1.0) / g;
    const double l = rb * (1.0 - u / ratio);
    if (fA) {
      t.d1 = d;
      t.l2 = l;
    } else {
      t.d2 = d;
      t.l1 = l;
    }
    return t;
  }
  if (sane && zA && zB) return t;
  return geomean_full(R1, R2, w1, w2, g, v1, v2);
}

// ---------------------------------------------------------------------------
// UniV3 -- src/cfmms.jl:251-259, 272-289, 294-313, 321-337, 339-395
// ---------------------------------------------------------------------------

// Every tick's BoundedProduct (src/cfmms.jl:272-278, built by compute_at_tick
// :294-313) depends only on pool state (liquidity, tick prices, current price),
// never on ν.  It is therefore evaluated only when that state changes (cfmm_finalize,
// cfmm_update_univ3, cfmm_apply_trades: the rebuild kernels of univ3_state.cuh), with
// the same IEEE operations in the same order, and stored per pool as two
// DIRECTION BLOCKS of one 32-byte record per tick (kTickStride doubles per tick in all):
//   "upper" walk (towards lower prices), block 0, tick i:  [k, R_1+α, δmax↑ = k/β − (R_1+α), R_2]
//   "lower" walk (the flipped pool, :289), block 1, tick i: [k, R_2+β, δmax↓ = k/α − (R_2+β), R_1]
// A walk reads consecutive 32-byte records of ONE block -- four ticks per 128-byte line, so the
// dependent loads of a walk mostly hit the line its first record brought in -- and the one extra
// value the tick it STOPS in needs (R_2+β for the upper walk, R_1+α for the lower) is the second
// double of the same tick's record in the OTHER block.  (Round 1: one 64-byte record per tick,
// both sectors needed per visit, 2.33x the algorithmic DRAM traffic; first form of round 2: 128
// bytes per tick, one touched sector per 128-byte line.)
// A visited tick costs find_arb_pos only (2 sqrt + 2 div), bit-identically.
constexpr int kTickStride = 8;

// The tick a walk STARTS in (the current tick) is additionally stored per pool, in pool order,
// as four coalesced double2 streams (Univ3First): (k, R_1+α), (R_2+β, current_price),
// (δmax↑, R_2), (δmax↓, R_1) -- 64 bytes per pool, every byte of which a trading pool uses.
// On the CSR-only form the DRAM reads are several times the 48 MB algorithmic of config 4,
// because one touched 32-byte sector of a 128-byte tick costs a 128-byte fetch, behind a
// dependent load (tick_off -> record).  Most walks end in the tick they start in: they now read
// pool-indexed streams only, and the CSR is touched by the walks that cross a boundary.
struct Univ3First {
  double k, ra, rb;          // loaded with the pool header
  const double2* up;         // (δmax↑, R_2) of this pool
  const double2* dn;         // (δmax↓, R_1)
};

// find_arb_pos (src/cfmms.jl:321-337) on one precomputed (flipped, :289) tick: sub = t.R_1 + t.α,
// load_b() = (δ_max, t.R_2), load_rb() = t.R_2 + t.β.  Returns false when the walk stops (:362, :384).
template <class LoadB, class LoadRb>
__device__ __forceinline__ bool univ3_tick(double k, double sub, double price, bool initial, LoadB load_b,
                                           LoadRb load_rb, double& dsum, double& lsum) {
  double d = __dsub_rn(__dsqrt_rn(__ddiv_rn(k, price)), sub), l;
  if (d <= 0.0) {
    d = 0.0;
    l = 0.0;
  } else {
    const double2 b = load_b();
    if (d >= b.x) {
      d = b.x;
      l = b.y;
    } else {
      l = __dsub_rn(load_rb(), __dsqrt_rn(__dmul_rn(price, k)));
    }
  }
  if (!initial && (d == 0.0 || l == 0.0)) return false;
  dsum = __dadd_rn(dsum, d);
  lsum = __dadd_rn(lsum, l);
  return true;
}

// find_arb!(Δ, Λ, ::UniV3, v), src/cfmms.jl:339-395.  Both walk directions share one loop (the
// direction is data: index step and record half), so a warp whose lanes walk in different
// directions does not execute two loops.  The first visited tick comes from the per-pool record.
// td: this pool's two direction blocks (n_ticks records of 4 doubles each, upper then lower).
__device__ __forceinline__ Trade univ3_arb(const double* __restrict__ td, int n_ticks, const Univ3First& first,
                                           double current_price, int current_tick, double g,
                                           double v1, double v2) {
  Trade t;
  t.d1 = t.d2 = t.l1 = t.l2 = 0.0;
  const double p = __ddiv_rn(v1, v2);
  const double lo = __dmul_rn(g, current_price);
  // no-arb interval :347
  if (lo <= p && p <= __ddiv_rn(current_price, g)) return t;
  const bool up = p < lo;  // :351 "upper pools" (towards lower prices); else :373 lower pools, flipped
  // price = p/γ (:359)  or  1/(γ·p) (:381)
  const double price = __ddiv_rn(up ? p : 1.0, up ? g : __dmul_rn(g, p));
  const int step = up ? 1 : -1;
  const int last = up ? n_ticks : 1;
  const double* rec0 = td + (up ? 0 : 4 * n_ticks);   // this walk's block
  const double* other = td + (up ? 4 * n_ticks : 0);  // the other block: (R_2+β | R_1+α) at [1]
  double dsum = 0.0, lsum = 0.0;
  int idx = current_tick;
  const auto in_range = [&](int i) { return up ? (i <= last) : (i >= last); };
  const auto record = [&](int i) { return reinterpret_cast<const double2*>(rec0 + (size_t)(i - 1) * 4); };
  // The walk is a chain of dependent record loads (tick i+1 is only visited once tick i is fully
  // consumed): the NEXT tick's first sector is requested before this tick's sqrt / div chain
  // starts, so its latency overlaps the arithmetic (most stall samples sat on these loads).  A
  // prefetched record that is never visited costs one 32-byte sector.  (Requesting it only when a
  // two-multiply estimate says the first tick will be consumed was slower despite fewer bytes:
  // the latency matters, the bytes do not.)
  double2 a_next = make_double2(0.0, 0.0), b_next = a_next;
  const auto prefetch = [&](int i) {
    if (in_range(i)) {
      a_next = __ldg(record(i));      // (k, t.R_1 + t.α) of the (flipped) tick
      b_next = __ldg(record(i) + 1);  // (δ_max, t.R_2): same 32-byte sector
    }
  };
  if (in_range(idx)) {
    prefetch(idx + step);
    // is_empty_pool (k == 0): skipped, not terminal (:354-357, :376-379)
    if (first.k != 0.0)
      univ3_tick(
          first.k, up ? first.ra : first.rb, price, true, [&]() { return __ldg(up ? first.up : first.dn); },
          [&]() { return up ? first.rb : first.ra; }, dsum, lsum);
    idx += step;
  }
  for (; in_range(idx); idx += step) {
    const double2 a = a_next, b = b_next;
    prefetch(idx + step);
    if (a.x == 0.0) continue;
    if (!univ3_tick(
            a.x, a.y, price, false, [&]() { return b; },
            [&]() { return __ldg(other + (size_t)(idx - 1) * 4 + 1); },  // t.R_2 + t.β: the other block's record
            dsum, lsum))
      break;
  }
  const double dn = __ddiv_rn(dsum, g);  // pre-fee tendered amount :371, :391
  if (up) {
    t.d1 = dn;
    t.l2 = lsum;
  } else {
    t.d2 = dn;
    t.l1 = lsum;
  }
  return t;
}

}  // namespace cfmm
