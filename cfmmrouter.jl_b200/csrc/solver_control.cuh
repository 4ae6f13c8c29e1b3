// solver_control.cuh -- the control logic of the projected L-BFGS (solver.cuh), shared by
// cfmm_solve's host loop and the per-row device solves of cfmm_quote_subgraph_orders /
// cfmm_execute_subgraph_orders (subgraph_kernels.cuh).
//
// Everything here acts on scalars: the Gram matrix W = BᵀB of the basis B = [S Y pg] (kSolverK
// columns), the history's age list, the line search's step and values.  The vectors stay where the
// caller keeps them (HBM for cfmm_solve, shared memory for a row).  The comparisons and the order of
// every operation are those of cfmm_solve's loop; on the host they compile to the same arithmetic.
#pragma once
#include <math.h>

#include "solver.cuh"

namespace cfmm {

constexpr double kSolverEps = 2.220446049250313e-16;  // machine epsilon of double

// std::min / std::max semantics ((b < a) ? b : a, (a < b) ? b : a), usable on both sides.
__host__ __device__ inline double lbfgs_min(double a, double b) { return (b < a) ? b : a; }
__host__ __device__ inline double lbfgs_max(double a, double b) { return (a < b) ? b : a; }

// The history of one solve: slots age[0 .. cnt) oldest first, head the slot the next pair goes to.
struct LbfgsHistory {
  int age[kSolverM];
  int cnt, head;
};

// The two-loop recursion in coefficient space over B = [S Y pg]: the direction is d = −B c (clipped
// to the free variables by the caller).  Returns the first trial step: 1, or min(1, 1/|pg|) with an
// empty history (a first step of length <= 1, like L-BFGS-B).
__host__ __device__ inline double lbfgs_direction(const double (&W)[kSolverK][kSolverK], const LbfgsHistory& h,
                                                  double (&c)[kSolverK]) {
  constexpr int M = kSolverM, K = kSolverK;
  for (int j = 0; j < K; ++j) c[j] = 0.0;
  c[K - 1] = 1.0;
  double t_init = 1.0;
  if (h.cnt == 0) {
    const double nrm = sqrt(W[K - 1][K - 1]);
    t_init = nrm > 0.0 ? lbfgs_min(1.0, 1.0 / nrm) : 1.0;
  } else {
    double alpha[M], rho[M];
    for (int a = h.cnt - 1; a >= 0; --a) {
      const int j = h.age[a];
      rho[a] = 1.0 / W[j][M + j];
      double sq = 0.0;
      for (int k = 0; k < K; ++k) sq += W[j][k] * c[k];
      alpha[a] = rho[a] * sq;
      c[M + j] -= alpha[a];
    }
    const int jn = h.age[h.cnt - 1];
    const double gamma = W[jn][M + jn] / W[M + jn][M + jn];
    for (int k = 0; k < K; ++k) c[k] *= gamma;
    for (int a = 0; a < h.cnt; ++a) {
      const int j = h.age[a];
      double yr = 0.0;
      for (int k = 0; k < K; ++k) yr += W[M + j][k] * c[k];
      c[j] += alpha[a] - rho[a] * yr;
    }
  }
  return t_init;
}

// One trial of the Armijo backtracking along the projected path, from f at the current point to
// f_new at P(x + t d); gdx = gᵀ(xt − x), step2 = |xt − x|².  f is a sum of many terms of mixed
// sign: differences below ~8 eps |f| are rounding noise, and near a flat optimum every useful step
// is that small, so the test has that slack.  On kLsRetry, t is the next step to try.
enum LbfgsTrial { kLsAccept, kLsStall, kLsRestart, kLsRetry };

__host__ __device__ inline int lbfgs_trial(double f, double f_new, double gdx, double step2, int cnt, double& t) {
  if (step2 == 0.0) return kLsStall;  // the projected step does not move
  const double noise = 8.0 * kSolverEps * lbfgs_max(lbfgs_max(fabs(f), fabs(f_new)), 1.0);
  if (gdx < 0.0 && f_new <= f + 1e-4 * gdx + noise) return kLsAccept;
  if (!(gdx < 0.0) && cnt > 0) return kLsRestart;  // not a descent direction: restart from −pg
  if (f_new == f_new && f_new < 1e300 && gdx < 0.0) {
    // minimiser of the quadratic through f, the slope gdx (per unit t) and f_new, kept in [0.1 t, 0.5 t]
    const double slope = gdx / t, denom = 2.0 * (f_new - f - gdx);
    double tq = denom > 0.0 ? -slope * t * t / denom : 0.5 * t;
    t = lbfgs_min(0.5 * t, lbfgs_max(0.1 * t, tq));
  } else {
    t *= 0.1;
  }
  return kLsRetry;
}

// After an accepted step stored in slot `slot` (its column pair in W): drop the slot's old pair from
// the age list and append the new one when its curvature is usable.
__host__ __device__ inline void lbfgs_store(const double (&W)[kSolverK][kSolverK], int slot, LbfgsHistory& h) {
  constexpr int M = kSolverM;
  int w = 0;
  for (int a = 0; a < h.cnt; ++a)
    if (h.age[a] != slot) h.age[w++] = h.age[a];
  h.cnt = w;
  const double sy = W[slot][M + slot], yy = W[M + slot][M + slot];
  if (sy > 1e-10 * yy && yy > 0.0) {
    h.age[h.cnt++] = slot;
    h.head = (h.head + 1) % M;
  }
}

// L-BFGS-B's factr test, on two consecutive steps: one short quasi-Newton step (fresh history, a
// bound just hit) is not yet evidence of convergence.  True: stop with status 1.
__host__ __device__ inline bool lbfgs_factr(double f_old, double f, double factr, int& small_steps) {
  if (f_old - f <= factr * kSolverEps * lbfgs_max(lbfgs_max(fabs(f_old), fabs(f)), 1.0)) return ++small_steps >= 2;
  small_steps = 0;
  return false;
}

}  // namespace cfmm
