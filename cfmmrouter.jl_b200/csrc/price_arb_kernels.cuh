// price_arb_kernels.cuh -- arbitrage against external prices over every pool among allowed tokens: one
// dual solve per row (sm_90a; cfmm_quote_price_arbitrage / cfmm_execute_price_arbitrage,
// include/cfmm_b200.h).  Off the sweep path: no sweep kernel reads anything these kernels add.
//
// A row values the call's allowed tokens A (the slots of best_path_kernels.cuh's BestPathGraph, in
// ascending order) at its prices c (a price of 0 leaves the token out) and solves route! with
// LinearNonnegative(c) over the row's pools.  Its setup (pa_setup) is its own; after it, the row runs
// subgraph_kernels.cuh's pool gather, pool ordering, solve (sg_solve with this file's LnRule) and legs.
//   setup   the row's prices into shared memory; T, the priced slots with an active pool to another
//           priced slot; the local tokens (T ascending), the per-slot box c_t + 1e-8, and the pool
//           count of every slot s in T (the pairs {s, u}, u > s in T);
//   solve   cfmm_solve's projected L-BFGS from the box's lower bound, lin = 0, the stop's scale the
//           committed dual value g;
//   legs    split_leg over the pools at the final ν: the legs and, on execute, the transition.
// price_arb_plan_kernel runs the setup only and reports each row's token and pool counts, which size
// the outputs and the workspace.
//
// Inventory rows (cfmm_quote/execute_price_arbitrage_rows, at the end of this file) run the same row
// body over each row's own slot graph (row_graph), with per-token holdings the net may spend and an
// absolute stop beside the relative one (InvRule, InvArbRows).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "subgraph_kernels.cuh"

namespace cfmm {

constexpr int kPriceArbMaxTokens = kSubgraphSlots;  // CFMM_PRICE_ARB_MAX_TOKENS
constexpr double kPriceArbBox = 1e-8;               // LinearNonnegative's lower limit c + 1e-8 (objectives.jl)

// The rows of one call, their options, and their outputs (device arrays; tokens 1-based).  row_orders
// fills the output pointers; received holds each row's profit, and paid is not written.
struct PriceArbRows {
  const double* price;       // [q·nB], row-major, columns in slot order
  const double* min_profit;  // [q] or null
  int max_iter, max_fun;
  double rtol, factr;
  const int64_t* tok_off;  // [q+1] (setup counts, scanned)
  const int64_t* leg_off;  // [q+1]
  double* paid;
  double* received;
  uint8_t* status;
  int32_t* solver_status;
  int32_t* iterations;
  int32_t* fun_evals;
  double* merit;
  int64_t* token;  // [tok_off[q]] or null (with nu, psi)
  double* nu;
  double* psi;
  int64_t* leg_entry;  // [leg_off[q]] or null: (set << 56) | device position
  double* leg_delta;   // [2L] or null (with leg_lambda)
  double* leg_lambda;
};

// Shared state of one row.  ipair stays −1: sg_gather's {s, i} pairs do not exist here.
struct PriceArbSmem {
  int32_t ipair[kSubgraphSlots], cnt[kSubgraphSlots + 1];
  int16_t lidx[kSubgraphSlots];
  uint8_t in[kSubgraphSlots], priced[kSubgraphSlots];
  int32_t ltok[kSubgraphLocal];
  int32_t inc_off[kSubgraphLocal + 1];
  double x[kSubgraphLocal], g[kSubgraphLocal], xt[kSubgraphLocal], gt[kSubgraphLocal], d[kSubgraphLocal],
      pg[kSubgraphLocal], px[kSubgraphLocal], pt[kSubgraphLocal];
  double S[kSolverM][kSubgraphLocal], Y[kSolverM][kSubgraphLocal];
  double W[kSolverK][kSolverK];
  double c[kSolverK];
  double red[kSubgraphWarps];
  double price[kSubgraphLocal], lo[kSubgraphLocal];  // c_t and c_t + 1e-8 in local order
  double gv;  // g at the last evaluation: inside sg_commit, g at the iterate it commits
  unsigned long long mx;
  int32_t n_loc, npool;
};

// The local tokens of T (m.in) and the pool count of every slot (cnt[s], the pools of the pairs {s, u},
// u > s in T, as exclusive offsets), after a barrier that published m.in.  Ends at a barrier.
template <class Smem, class Graph>  // BestPathGraph or RowGraph
__device__ __forceinline__ void pa_local(PairIndexView ix, const Graph& G, Smem& m) {
  const int tid = threadIdx.x, nB = G.nB;
  for (int s = tid; s < nB; s += blockDim.x) {
    int32_t c = 0;
    if (m.in[s]) {
      const int dg = G.deg[s];
      for (int e = 0; e < dg; ++e) {
        const int u = G.nbr[(int64_t)nB * s + e];
        const int32_t k = G.pair[(int64_t)nB * s + e];
        if (u > s && m.in[u]) c += (int32_t)(ix.off[k + 1] - ix.off[k]);
      }
    }
    m.cnt[s] = c;
  }
  __syncthreads();
  if (tid == 0) {
    int loc = 0;
    int32_t tot = 0;
    for (int s = 0; s < nB; ++s) {
      if (m.in[s]) {
        m.lidx[s] = (int16_t)loc;
        m.ltok[loc++] = G.tok[s];
      }
      const int32_t c = m.cnt[s];
      m.cnt[s] = tot;  // exclusive offsets
      tot += c;
    }
    m.cnt[nB] = tot;
    m.n_loc = loc;
    m.npool = tot;
  }
  __syncthreads();
}

// Setup of the row with prices price[0 .. nB) (slot order): T, the local tokens, their prices and box,
// and the pool count of every slot (cnt[s], the pools of the pairs {s, u} for slots u > s in T).
__device__ void pa_setup(PairIndexView ix, const BestPathGraph& G, const uint8_t* __restrict__ gact,
                         const double* __restrict__ price, PriceArbSmem& m) {
  const int tid = threadIdx.x, nB = G.nB;
  for (int s = tid; s < nB; s += blockDim.x) {
    m.ipair[s] = -1;
    m.lidx[s] = -1;
    m.priced[s] = price[s] > 0.0;
  }
  __syncthreads();
  for (int s = tid; s < nB; s += blockDim.x) {
    bool t = false;
    if (m.priced[s]) {
      const int dg = G.deg[s];
      for (int e = 0; e < dg && !t; ++e) t = m.priced[G.nbr[(int64_t)nB * s + e]] && gact[(int64_t)nB * s + e];
    }
    m.in[s] = t;
  }
  __syncthreads();
  pa_local(ix, G, m);
  for (int s = tid; s < nB; s += blockDim.x)
    if (m.in[s]) {
      const double c = price[s];
      m.price[m.lidx[s]] = c;
      m.lo[m.lidx[s]] = __dadd_rn(c, kPriceArbBox);
    }
  __syncthreads();
}

// The rules of a price row, as subgraph_kernels.cuh's SgRule: lin = 0 and a linear value of 0.0; the
// box ν_t >= c_t + 1e-8 (no slot fixed), the start at that bound; m_r = mx / g with g the dual value of
// the committed iterate (0 when mx = 0: nothing trades; +inf when g <= 0 < mx, so the row goes on).
struct LnRule {
  static constexpr bool kOut = false;
  static constexpr bool kBoxStart = true;
  __device__ __forceinline__ double lin_at(const PriceArbSmem&, int) const { return 0.0; }
  __device__ __forceinline__ double value(const PriceArbSmem&) const { return 0.0; }
  __device__ __forceinline__ double lo(const PriceArbSmem& m, int t) const { return m.lo[t]; }
  __device__ __forceinline__ bool fixed(const PriceArbSmem&, int) const { return false; }
  __device__ __forceinline__ int root(const PriceArbSmem&) const { return 0; }
  __device__ __forceinline__ void evaluated(PriceArbSmem& m, double f) const {
    if (threadIdx.x == 0) m.gv = f;  // read after sg_commit's barriers
  }
  __device__ __forceinline__ double merit(const PriceArbSmem& m, double mx) const {
    if (!(mx > 0.0)) return 0.0;
    return m.gv > 0.0 ? __ddiv_rn(mx, m.gv) : __longlong_as_double(0x7ff0000000000000ll);
  }
};

// Per row: the number of tokens the row lists (T) and of its pools.
__global__ void __launch_bounds__(kSubgraphThreads)
    price_arb_plan_kernel(PairIndexView ix, BestPathGraph G, const uint8_t* __restrict__ gact,
                          const double* __restrict__ price, int64_t q, int64_t* __restrict__ ntok,
                          int64_t* __restrict__ npool) {
  __shared__ PriceArbSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    pa_setup(ix, G, gact, price + r * G.nB, m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc;
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Row r on the current state, after setup() (pa_setup, or inv_setup and inv_values) filled m.
// Returns nothing; writes the row's outputs.  EXEC: min_profit decides, and a filled row applies the
// transition of cfmm_apply_trades at its ν to each of its pools.
template <bool EXEC, class Rule, class Graph, class Rows, class Smem, class Setup>
__device__ void price_arb_row(const PathSets* P, PairIndexView ix, const Graph& G, const Rows& R,
                              const SubgraphWork& w, const SplitMoved& mv, int64_t r, Smem& m, Setup setup) {
  __shared__ SgSolveState s;
  __shared__ double s_profit;
  const int tid = threadIdx.x;
  setup();
  const int64_t np = m.npool, n = m.n_loc;
  sg_gather(ix, G, w, m, [](int, auto&) {});
  sg_order_pools(P, w, m, np, n, [&](int32_t t) { return (int32_t)m.lidx[G.slot_of[t]]; });
  double merit;
  const int status = sg_solve(P, w, m, Rule{}, R, n, true, s, merit);
  // the profit Σ_t c_t·Ψ_t in local order, from the first term
  if (tid == 0) {
    double pr = 0.0;
    if (n > 0) {
      pr = __dmul_rn(m.price[0], m.px[0]);
      for (int t = 1; t < n; ++t) pr = __dadd_rn(pr, __dmul_rn(m.price[t], m.px[t]));
    }
    s_profit = pr;
  }
  __syncthreads();
  const double profit = s_profit;
  uint8_t st = 0;  // CFMM_ORDER_FILLED
  if (status != 0)
    st = 5;  // CFMM_ORDER_NOT_CONVERGED
  else if (EXEC && R.min_profit && profit < R.min_profit[r])
    st = 1;  // CFMM_ORDER_LIMIT; an equal min_profit fills
  const bool filled = st == 0;
  sg_legs<EXEC>(P, w, m.x, mv, R, r, np, filled);
  if (R.token) {
    const int64_t o = R.tok_off[r];
    for (int t = tid; t < n; t += blockDim.x) {
      R.token[o + t] = m.ltok[t] + 1;
      R.nu[o + t] = m.x[t];
      R.psi[o + t] = m.px[t];
    }
  }
  if (tid == 0) {
    R.received[r] = filled ? profit : 0.0;
    R.status[r] = st;
    R.solver_status[r] = status;
    R.iterations[r] = s.iter;
    R.fun_evals[r] = s.fev;
    R.merit[r] = merit;
  }
  __syncthreads();  // the next row reuses the shared state and the workspace
}

// Rows rows[0 .. n) (null: 0 .. n), one CTA at a time each; CTA b uses workspace b.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    price_arb_kernel(const PathSets* __restrict__ P, PairIndexView ix, BestPathGraph G,
                     const uint8_t* __restrict__ gact, PriceArbRows R, SubgraphWork w, SplitMoved mv,
                     const int64_t* __restrict__ rows, int64_t n) {
  __shared__ PriceArbSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    const int64_t r = rows ? rows[k] : k;
    price_arb_row<EXEC, LnRule>(P, ix, G, R, wb, mv, r, m, [&] { pa_setup(ix, G, gact, R.price + r * G.nB, m); });
  }
}

// ---- inventory rows (cfmm_quote/execute_price_arbitrage_rows): each row over its own listed tokens L,
// with a price c_t >= 0 and a holding h_t >= 0 per listed token, solving route! with
// cᵀΨ − I(Ψ + h >= 0) over every pool among T.  T is the listed tokens with an active pool to another
// listed token (a price of 0 keeps the token, valued at 0); the pools and the local order are the
// price row's.  The dual is G(ν) = Σ_p π_p(ν) + hᵀν on the price row's box, started at its lower
// bound; P̄ = G − hᵀc = π(ν) + hᵀ(ν − c) >= 0 bounds the profit.  The stop is m_r = mx / P̄ <= rtol or
// mx <= atol, with mx = max_t s_t·|pg_t| and s_t = max(ν_t, c̄), c̄ the least positive price the row
// lists.  A priced token has ν_t > c_t >= c̄, so s_t = ν_t there, as in the price row; a token priced 0
// sits near ν_t = 1e-8, and the floor c̄ keeps its term in token units (a unit of it weighs at least
// the cheapest priced token) instead of letting 1e-8·|pg_t| hide an overdraft of ~1e8·ε units.  A
// row that holds nothing runs LnRule's operations: every listed price > 0 and atol 0 give the price
// row over its list, bit for bit.
//
// Why the fill promise holds (ε = max(rtol·P̄, atol), so s_t·|pg_t| <= ε at the stop): the gradient is
// g_t = h_t + Ψ_t.  A free token has |h_t + Ψ_t| <= ε/s_t; one on its bound has pg_t = 0 only when
// g_t > 0, else |g_t| <= ε/s_t: in both cases Ψ_t >= −h_t − ε/s_t, so no token is overdrawn by more
// than ε/c̄ units.  π is positively homogeneous, so π(ν) = νᵀΨ and P̄ − cᵀΨ = νᵀΨ + hᵀ(ν − c) − cᵀΨ =
// Σ_t (ν_t − c_t)(Ψ_t + h_t).  A free token adds at most (ν_t − c_t)·ε/s_t <= ε; a token on its bound
// adds 1e-8·(Ψ_t + h_t) (ν_t − c_t = 1e-8 up to the rounding of c_t + 1e-8).  So P̄ − cᵀΨ <= |T|·ε +
// Σ_{t on its bound} 1e-8·(Ψ_t + h_t).  P̄ bounds the optimum profit from above (weak duality); cᵀΨ
// exceeds it by at most the overdraft valued at ν, Σ_t (ν_t − c_t)·max(−Ψ_t − h_t, 0) <= |T|·ε.

// The rows of an inventory call: price (PriceArbRows::price) and hold are aligned with the call's
// allow_token ([allow_off[q]]); hold null: every holding 0.
struct InvArbRows : PriceArbRows {
  const double* hold;
  double atol;
};

// An inventory row's shared state: the price row's, with h_t in local order (+0.0 where nothing is
// held), the local tokens with h_t > 0 ascending, and hᵀc over them.  The box c_t + 1e-8 is not
// stored but recomputed (InvRule::lo), which keeps the state within the 48 KB of static shared memory.
struct InvArbSmem {
  int32_t ipair[kSubgraphSlots], cnt[kSubgraphSlots + 1];
  int16_t lidx[kSubgraphSlots];
  uint8_t in[kSubgraphSlots];
  int32_t ltok[kSubgraphLocal];
  int32_t inc_off[kSubgraphLocal + 1];
  double x[kSubgraphLocal], g[kSubgraphLocal], xt[kSubgraphLocal], gt[kSubgraphLocal], d[kSubgraphLocal],
      pg[kSubgraphLocal], px[kSubgraphLocal], pt[kSubgraphLocal];
  double S[kSolverM][kSubgraphLocal], Y[kSolverM][kSubgraphLocal];
  double W[kSolverK][kSolverK];
  double c[kSolverK];
  double red[kSubgraphWarps];
  double price[kSubgraphLocal], h[kSubgraphLocal];  // c_t and h_t in local order
  int16_t held[kSubgraphLocal];
  double gv, hc, cbar;  // cbar: c̄, the least positive price of the row's list
  unsigned long long mx;
  int32_t n_loc, npool, nheld;
};

// Setup of row r over its slot graph G (every slot listed): T (the slots with an active pool to
// another slot), the local tokens and the pool counts.  Ends at a barrier.
__device__ __forceinline__ void inv_setup(PairIndexView ix, const RowGraph& G, const uint8_t* __restrict__ gact,
                                          InvArbSmem& m) {
  const int tid = threadIdx.x, nB = G.nB;
  for (int s = tid; s < nB; s += blockDim.x) {
    m.ipair[s] = -1;
    m.lidx[s] = -1;
    bool t = false;
    const int dg = G.deg[s];
    for (int e = 0; e < dg && !t; ++e) t = gact[(int64_t)nB * s + e];
    m.in[s] = t;
  }
  __syncthreads();
  pa_local(ix, G, m);
}

// Row r's prices and holdings into local order: entry k of the row's list (caller order) goes to
// its slot's local token.  Then the held tokens, hᵀc in local order (the first term alone) and c̄.
__device__ __forceinline__ void inv_values(const RowGraph& G, const RowMasks& M, const InvArbRows& R, int64_t r,
                                           InvArbSmem& m) {
  const int tid = threadIdx.x;
  const int64_t a0 = M.off[r];
  for (int k = tid; k < G.nB; k += blockDim.x) {
    const int l = m.lidx[G.slot_of[(int32_t)(M.tok[a0 + k] - 1)]];
    if (l < 0) continue;
    const double c = R.price[a0 + k], h = R.hold ? R.hold[a0 + k] : 0.0;
    m.price[l] = c;
    m.h[l] = h > 0.0 ? h : 0.0;
  }
  __syncthreads();
  if (tid == 0) {
    int nh = 0;
    double hc = 0.0;
    for (int t = 0; t < m.n_loc; ++t)
      if (m.h[t] > 0.0) {
        const double v = __dmul_rn(m.h[t], m.price[t]);
        hc = nh == 0 ? v : __dadd_rn(hc, v);
        m.held[nh++] = (int16_t)t;
      }
    m.nheld = nh;
    m.hc = hc;
    double cb = __longlong_as_double(0x7ff0000000000000ll);  // the row has a positive price (checked)
    for (int k = 0; k < G.nB; ++k) {
      const double c = R.price[a0 + k];
      if (c > 0.0) cb = fmin(cb, c);
    }
    m.cbar = cb;
  }
  __syncthreads();
}

// The rules of an inventory row: LnRule's box (c_t + 1e-8, the same IEEE addition), start and
// evaluation record, with lin = h, the linear value hᵀν over the held tokens (sg_cta_sum's fixed
// order over them in local order), and m_r = mx / P̄ with P̄ = g − hᵀc (0 when mx = 0; +inf when
// P̄ <= 0 < mx).  With nothing held: LnRule's 0.0 and mx / g.
struct InvRule {
  static constexpr bool kOut = false;
  static constexpr bool kBoxStart = true;
  __device__ __forceinline__ double lin_at(const InvArbSmem& m, int t) const { return m.h[t]; }
  // called by every thread of the CTA (sg_evaluate), so the sum may take the CTA's barriers
  __device__ __forceinline__ double value(InvArbSmem& m) const {
    if (m.nheld == 0) return 0.0;
    double v = 0.0;
    for (int k = threadIdx.x; k < m.nheld; k += blockDim.x) v = __dadd_rn(v, __dmul_rn(m.h[m.held[k]], m.xt[m.held[k]]));
    return sg_cta_sum(v, m);
  }
  __device__ __forceinline__ double lo(const InvArbSmem& m, int t) const { return __dadd_rn(m.price[t], kPriceArbBox); }
  __device__ __forceinline__ bool fixed(const InvArbSmem&, int) const { return false; }
  __device__ __forceinline__ int root(const InvArbSmem&) const { return 0; }
  __device__ __forceinline__ void evaluated(InvArbSmem& m, double f) const {
    if (threadIdx.x == 0) m.gv = f;  // read after sg_commit's barriers
  }
  __device__ __forceinline__ double merit(const InvArbSmem& m, double mx) const {
    if (!(mx > 0.0)) return 0.0;
    const double pb = m.nheld ? __dsub_rn(m.gv, m.hc) : m.gv;
    return pb > 0.0 ? __ddiv_rn(mx, pb) : __longlong_as_double(0x7ff0000000000000ll);
  }
};

// The stop's scale of an inventory row: s_t = max(ν_t, c̄) (ν_t itself wherever c_t > 0).
__device__ __forceinline__ double sg_stop_scale(const InvArbSmem& m, const InvRule&, int t) {
  return fmax(m.x[t], m.cbar);
}

// The absolute stop of inventory rows: mx <= atol at the committed iterate (atol 0: only mx = 0, where
// m_r is 0 already).
template <class Smem>
__device__ __forceinline__ bool sg_atol_met(const Smem& m, const InvArbRows& R) {
  return __longlong_as_double((long long)m.mx) <= R.atol;
}

// Per row: the number of its tokens in T and of its pools.
__global__ void __launch_bounds__(kSubgraphThreads)
    price_arb_rows_plan_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M, int64_t q,
                               int64_t* __restrict__ ntok, int64_t* __restrict__ npool) {
  __shared__ InvArbSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    const RowGraph G = row_graph(P, ix, A, M, r);
    inv_setup(ix, G, rg_act(M), m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc;
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Inventory rows rows[0 .. n) (null: 0 .. n), one CTA at a time each over its own slot graph; CTA b
// uses workspace b.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    price_arb_rows_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M, InvArbRows R,
                          SubgraphWork w, SplitMoved mv, const int64_t* __restrict__ rows, int64_t n) {
  __shared__ InvArbSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    const int64_t r = rows ? rows[k] : k;
    const RowGraph G = row_graph(P, ix, A, M, r);
    price_arb_row<EXEC, InvRule>(P, ix, G, R, wb, mv, r, m, [&] {
      inv_setup(ix, G, rg_act(M), m);
      inv_values(G, M, R, r, m);
    });
  }
}

}  // namespace cfmm
