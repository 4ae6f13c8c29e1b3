/*
 * cfmm_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the arithmetic on CFMMRouter.jl's dual-decomposition
 * hot path (reference @ 5932e42, v0.3.1).  Every function cites the reference
 * file:line it follows (paths relative to the reference tree).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library; the product path (libcfmm_b200.so)
 * never links or calls it.
 *
 * PARITY PIN.  The reference is Julia and Julia is not available in this image,
 * so the oracle cannot be diffed against a run of the reference.  It is pinned
 * instead on (1) the known-answer tests the reference's own suite holds for
 * this path (test/cfmms.jl:74-86), (2) the reference's optimality predicates
 * (test/cfmms.jl:3-56) restated in tests/, and (3) 50-digit mpmath evaluations
 * of the closed forms (tests/golden/, generator committed).  For
 * ProductTwoCoin and UniV3 the reference uses only IEEE-754 correctly rounded
 * operations (+ - * / sqrt, max) in a fixed order, so a restatement with the
 * same order (this file, compiled with -ffp-contract=off, no fast-math) is
 * bit-identical to the Julia result by construction.  GeometricMeanTwoCoin
 * calls Julia's `^`, which is not correctly rounded (<1 ulp): there the oracle
 * (glibc pow, <1 ulp) can differ from Julia in the last bit -- "parity
 * unpinned at the last ulp" for that type.
 */
#ifndef CFMM_ORACLE_H
#define CFMM_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- per-pool closed forms ------------------------------------------------ */

/* src/cfmms.jl:125-126 (prod_arb_δ/λ), :130-140 (find_arb!) */
void oracle_product_arb(const double R[2], double gamma, const double v[2],
                        double Delta[2], double Lambda[2]);

/* src/cfmms.jl:180-181 (geom_arb_δ/λ), :185-196 (find_arb!) */
void oracle_geomean_arb(const double R[2], const double w[2], double gamma,
                        const double v[2], double Delta[2], double Lambda[2]);

/* src/cfmms.jl:233-235: searchsortedlast(lower_ticks, current_price; rev=true)
 * = number of leading entries with lower_ticks[idx] >= current_price (1-based
 * index of the last such entry; 0 if none). */
int64_t oracle_univ3_current_tick(const double *lower_ticks, int64_t n_ticks,
                                  double current_price);

/* src/cfmms.jl:339-395 with compute_at_tick :294-313, find_arb_pos :321-337,
 * tick_high/low_price :251-259, flip_sides :289. current_tick is 1-based. */
void oracle_univ3_arb(double current_price, int64_t current_tick,
                      const double *lower_ticks, const double *liquidity,
                      int64_t n_ticks, double gamma, const double v[2],
                      double Delta[2], double Lambda[2]);

/* src/cfmms.jl:401-449 (test helper forward_trade): amount received for
 * tendering Delta; used by the UniV3 optimality predicate of test/cfmms.jl:25-56 */
double oracle_univ3_forward_trade(double current_price, int64_t current_tick,
                                  const double *lower_ticks,
                                  const double *liquidity, int64_t n_ticks,
                                  double gamma, const double Delta[2]);

/* compute_at_tick (src/cfmms.jl:294-313): out = {k, alpha, beta, R_1, R_2};
 * idx is 1-based */
void oracle_univ3_tick(double current_price, int64_t current_tick,
                       const double *lower_ticks, const double *liquidity,
                       int64_t n_ticks, int64_t idx, double out[5]);

/* ---- router sweep (src/router.jl:38-42) over flat pool arrays ------------- */
/* R, Delta, Lambda are pool-major [2*m]; Ai is 1-based [2*m] as in Julia.
 * threads <= 1: serial loop; > 1: OpenMP static parallel-for over pools
 * (the analogue of Threads.@threads at router.jl:39). */
void oracle_sweep_product(int64_t m, const double *R, const double *gamma,
                          const int64_t *Ai, const double *v, double *Delta,
                          double *Lambda, int threads);
void oracle_sweep_geomean(int64_t m, const double *R, const double *gamma,
                          const int64_t *Ai, const double *w, const double *v,
                          double *Delta, double *Lambda, int threads);
void oracle_sweep_univ3(int64_t m, const double *current_price,
                        const double *gamma, const int64_t *Ai,
                        const int64_t *tick_off, const double *lower_ticks,
                        const double *liquidity, const double *v,
                        double *Delta, double *Lambda, int threads);

/* ---- router folds (src/router.jl:79-83 and :98-100), serial, pool order --- */
/* acc += sum_i dot(Lambda_i, v[Ai]) - dot(Delta_i, v[Ai]);  G[Ai] += Lambda_i - Delta_i
 * (also netflows!, router.jl:111-119, when G starts at zero).  acc/G are
 * in-out so several pool types can be chained in insertion order. */
void oracle_fold(int64_t m, const int64_t *Ai, const double *Delta,
                 const double *Lambda, const double *v, double *acc, double *G);

/* Same sums in extended precision (long double, Neumaier-compensated): the
 * "true" Psi/acc the atomics-ordered GPU result is compared against.
 * abs_G[j] accumulates sum |Lambda|+|Delta| into token j (error scale). */
void oracle_fold_compensated(int64_t m, const int64_t *Ai, const double *Delta,
                             const double *Lambda, const double *v,
                             long double *acc, long double *G, double *abs_G);

/* ---- CPU timing baselines (bench.py cpu_baseline / --impl reference) ------ */
/* "faithful layout" flavour of the ProductTwoCoin sweep + folds: an array of
 * heap pool objects, each owning heap R[2] / Ai[2] (cfmms.jl:13-17), per-call
 * heap gather of v[Ai] (router.jl:40), dispatch through a function pointer
 * (abstractly-typed Vector{CFMM{T}}, router.jl:6), OpenMP sweep then SERIAL
 * acc and scatter loops (router.jl:79-83, 98-100). */
typedef struct oracle_faithful oracle_faithful;
oracle_faithful *oracle_faithful_create(int64_t n_tokens);
void oracle_faithful_add_product(oracle_faithful *o, int64_t m, const double *R,
                                 const double *gamma, const int64_t *Ai);
void oracle_faithful_add_geomean(oracle_faithful *o, int64_t m, const double *R,
                                 const double *gamma, const int64_t *Ai,
                                 const double *w);
/* one fn+g! evaluation's worth of pool work: sweep, acc fold, G scatter */
double oracle_faithful_sweep(oracle_faithful *o, const double *v, double *G,
                             int threads);
void oracle_faithful_destroy(oracle_faithful *o);

/* SoA flavour: same arithmetic, OpenMP with per-thread Psi then a reduction */
double oracle_soa_sweep_product(int64_t m, const double *R, const double *gamma,
                                const int64_t *Ai, const double *v,
                                int64_t n_tokens, double *G, int threads);

int oracle_max_threads(void);

#ifdef __cplusplus
}
#endif
#endif
