// subgraph_kernels.cuh -- orders routed over every pool among their allowed tokens: one dual solve
// per row (sm_90a; cfmm_quote_subgraph_swap_orders / cfmm_execute_subgraph_swap_orders, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// The call's allowed tokens are best_path_kernels.cuh's slots (BestPathGraph, built once per call by
// best_path_graph_kernel); subgraph_act_kernel adds, per slot neighbour, whether the pair holds an
// active pool.  One CTA solves one row at a time (a persistent grid strides over the rows):
//   setup   the pairs {j, b}, {i, b} and {j, i}, the component T of i over active pools, the local
//           tokens (0 = i, 1 = j, then T's slots ascending) and the row's pools: every pool of every
//           pair inside T, bitonic-sorted into global insertion order in the CTA's workspace, with a
//           per-token incidence list in that order;
//   solve   cfmm_solve's projected L-BFGS (solver_control.cuh) with every vector in shared memory;
//           an evaluation writes each pool's contributions to the workspace (split_legs at ν taken at
//           the pool's stored tokens), then sums them per token in a fixed warp tree;
//   legs    split_leg over the pools at the final ν: the legs and, on execute, the transition.
// subgraph_kernel solves exact-in rows, subgraph_out_kernel exact-out rows: the same row with the
// linear term, the box, the start's root and the stop's scale of its kind (SgRule), fixed at compile
// time.  subgraph_plan_kernel runs the setup only and reports each row's token and pool counts, which
// size the outputs and the workspace (they do not depend on the kind).
//
// basket_kernels.cuh's rows (limit rows included) and price_arb_kernels.cuh's rows run everything after
// their own setup through this file's helpers, which take the row's shared state and its rules as
// template parameters: the pool gather, the pool ordering, the evaluation, the commit, the L-BFGS
// driver, the legs, and the pair activity, CTA sum, pool view, start and capacity.  The setups stay per kind: running subgraph
// rows through the longer basket setup cost 2.3–2.6 % more kernel time on the headline set (DESIGN §4.5).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "best_path_kernels.cuh"
#include "solver_control.cuh"

namespace cfmm {

constexpr int kSubgraphMaxTokens = 256;                  // CFMM_SUBGRAPH_MAX_TOKENS
constexpr int kSubgraphSlots = kSubgraphMaxTokens + 2;  // a call's slots: a row's B plus its j and i
constexpr int kSubgraphLocal = kSubgraphMaxTokens + 2;  // a row's tokens: i, j and B ∩ T
constexpr int kSubgraphThreads = 256;
constexpr int kSubgraphWarps = kSubgraphThreads / 32;
constexpr double kSubgraphSqrtEps = 1.4901161193847656e-08;  // sqrt(eps), the box of Swap (objectives.jl)

// Per slot neighbour m of slot s (BestPathGraph layout): 1 when the pair holds an active pool.
__device__ __forceinline__ bool subgraph_pair_active(const PathSets* P, PairIndexView ix, int64_t k) {
  for (int64_t e = ix.off[k]; e < ix.off[k + 1]; ++e) {
    const int64_t entry = ix.pool[e];
    const int set = (int)(entry >> kPairSetShift);
    const uint8_t* a = P->s[set].active;
    if (!a || a[entry & kPairPosMask]) return true;
  }
  return false;
}

__global__ void subgraph_act_kernel(const PathSets* __restrict__ P, PairIndexView ix, BestPathGraph G,
                                    uint8_t* __restrict__ act) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)G.nB * G.nB) return;
  const int s = (int)(t / G.nB), m = (int)(t % G.nB);
  if (m < G.deg[s]) act[t] = subgraph_pair_active(P, ix, G.pair[t]) ? 1 : 0;
}

// ---- per-row masks (the *_rows calls): each row's own slots and their graph, built by its CTA

// Slot lookup in a row's slots: its listed tokens (0-based) ascending in tok[0 .. n), bisected; −1
// for a token the row does not list.
struct RowSlotOf {
  const int32_t* tok;
  int n;
  __device__ __forceinline__ int32_t operator[](int32_t t) const {
    int lo = 0, hi = n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (tok[mid] < t)
        lo = mid + 1;
      else
        hi = mid;
    }
    return lo < n && tok[lo] == t ? lo : -1;
  }
};

// One row's slot graph, read through the same members as BestPathGraph: tok and deg in dynamic shared
// memory, nbr and pair (and the activity beside them) in the CTA's part of the call's RowMasks.
struct RowGraph {
  const int32_t* tok;
  RowSlotOf slot_of;
  const int32_t* deg;
  const int16_t* nbr;
  const int32_t* pair;
  int nB;
};

// The per-row masks of a call: row r lists the tokens tok[off[r] .. off[r+1]) (1-based, distinct).
// Each CTA owns cap = bmax² entries of nbr, pair and act (bmax: the call's longest list); the row's
// sorted tokens and degrees live at byte goff of the dynamic shared memory (after the basket rows'
// bk_dyn_bytes).
struct RowMasks {
  const int64_t* off;
  const int64_t* tok;
  int16_t* nbr;
  int32_t* pair;
  uint8_t* act;
  int64_t cap;
  int goff;
};
constexpr int kRowGraphBytes = 2 * kSubgraphSlots * (int)sizeof(int32_t);  // tok and deg

extern __shared__ __align__(8) unsigned char rg_dyn[];

__device__ __forceinline__ const uint8_t* rg_act(const RowMasks& M) { return M.act + M.cap * blockIdx.x; }

// Row r's slot graph, by the whole CTA: its tokens sorted by rank (they are distinct), then one warp
// per slot s: the slots among s's token's neighbours, ascending, with their pair and whether it holds
// an active pool (subgraph_act_kernel's rule), from the adjacency list walked when it is short, else
// bisected per slot (side_pairs' rule).  Ends at a barrier.
__device__ RowGraph row_graph(const PathSets* P, PairIndexView ix, AdjView A, const RowMasks& M, int64_t r) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int32_t* tok = reinterpret_cast<int32_t*>(rg_dyn + M.goff);
  int32_t* deg = tok + kSubgraphSlots;
  const int64_t a0 = M.off[r], c = M.cap * blockIdx.x;
  const int n = (int)(M.off[r + 1] - a0);
  int16_t* nbr = M.nbr + c;
  int32_t* pair = M.pair + c;
  uint8_t* act = M.act + c;
  for (int k = tid; k < n; k += blockDim.x) deg[k] = (int32_t)(M.tok[a0 + k] - 1);  // (staged in deg)
  __syncthreads();
  for (int k = tid; k < n; k += blockDim.x) {
    const int32_t v = deg[k];
    int rank = 0;
    for (int l = 0; l < n; ++l) rank += deg[l] < v;
    tok[rank] = v;
  }
  __syncthreads();
  const RowGraph G{tok, RowSlotOf{tok, n}, deg, nbr, pair, n};
  for (int s = warp; s < n; s += kSubgraphWarps) {
    const int64_t e0 = A.off[tok[s]], e1 = A.off[tok[s] + 1];
    const bool walk = e1 - e0 <= (int64_t)n;
    int cnt = 0;
    for (int64_t b = walk ? e0 : 0; b < (walk ? e1 : (int64_t)n); b += 32) {
      int32_t u = -1;
      int64_t e = -1;
      if (walk) {
        e = b + lane;
        if (e < e1) u = G.slot_of[A.nbr[e]];
      } else if (b + lane < n) {
        e = adj_find(A, e0, e1, tok[b + lane]);
        if (e < e1) u = (int32_t)(b + lane);
      }
      const unsigned in = __ballot_sync(kFull, u >= 0);
      if (u >= 0) {
        const int64_t at = (int64_t)n * s + cnt + __popc(in & ((1u << lane) - 1u));
        nbr[at] = (int16_t)u;
        pair[at] = A.pair[e];
        act[at] = subgraph_pair_active(P, ix, A.pair[e]) ? 1 : 0;
      }
      cnt += __popc(in);
    }
    if (lane == 0) deg[s] = cnt;
  }
  __syncthreads();
  return G;
}

// The rows of one call, their options, and their outputs (device arrays; tokens 1-based).
struct SubgraphRows {
  const int64_t* token_in;
  const int64_t* token_out;
  const double* amount;
  const double* limit;  // null: none
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

// The CTA's workspace: cap (a power of two) pools.
struct SubgraphWork {
  int64_t* ent;
  int64_t* key;
  int32_t* ta;  // local token of the pool's stored token 1
  int32_t* tb;
  int32_t* inc;  // [2·cap] incidence: 2·pool + side
  double* ca;    // Λ₁ − Δ₁ (stored order)
  double* cb;
  int64_t cap;
};

// Shared state of one row.
struct SubgraphSmem {
  int32_t jpair[kSubgraphSlots], ipair[kSubgraphSlots], cnt[kSubgraphSlots + 1];
  int16_t lidx[kSubgraphSlots];
  uint8_t jact[kSubgraphSlots], iact[kSubgraphSlots], in[kSubgraphSlots];
  int32_t ltok[kSubgraphLocal];
  int32_t inc_off[kSubgraphLocal + 1];
  double x[kSubgraphLocal], g[kSubgraphLocal], xt[kSubgraphLocal], gt[kSubgraphLocal], d[kSubgraphLocal],
      pg[kSubgraphLocal], px[kSubgraphLocal], pt[kSubgraphLocal];
  double S[kSolverM][kSubgraphLocal], Y[kSolverM][kSubgraphLocal];
  double W[kSolverK][kSolverK];
  double c[kSolverK];
  double red[kSubgraphWarps];
  unsigned long long mx;
  int32_t direct, n_loc, jin, npool, direct_cnt;
  int32_t jslot, islot;
  int changed;
};

__device__ __forceinline__ bool sg_slot_ok(const SubgraphSmem& m, int s) { return s != m.jslot && s != m.islot; }

// Setup of row (j, i), 0-based: T, the local tokens and the pool count of every slot (cnt[s], the
// pools of the pairs {s, i}, {s, j} when j ∈ T, and {s, u} for slots u > s in T) and of {j, i}.
template <class Graph>  // BestPathGraph or RowGraph
__device__ void sg_setup(const PathSets* P, PairIndexView ix, AdjView A, const Graph& G,
                         const uint8_t* __restrict__ gact, int32_t j, int32_t i, SubgraphSmem& m) {
  const int tid = threadIdx.x, nB = G.nB;
  for (int s = tid; s < nB; s += blockDim.x) {
    m.jpair[s] = m.ipair[s] = -1;
    m.in[s] = 0;
    m.lidx[s] = -1;
  }
  if (tid == 0) {
    m.jslot = G.slot_of[j];
    m.islot = G.slot_of[i];
    m.direct = adj_pair(A, j, i);
    m.jin = m.direct >= 0 && subgraph_pair_active(P, ix, m.direct);
  }
  __syncthreads();
  side_pairs(A, G, j, m.jpair);
  side_pairs(A, G, i, m.ipair);
  __syncthreads();
  for (int s = tid; s < nB; s += blockDim.x) {
    const bool ok = sg_slot_ok(m, s);
    m.jact[s] = ok && m.jpair[s] >= 0 && subgraph_pair_active(P, ix, m.jpair[s]);
    m.iact[s] = ok && m.ipair[s] >= 0 && subgraph_pair_active(P, ix, m.ipair[s]);
    m.in[s] = m.iact[s];
  }
  __syncthreads();
  // the component of i: grow T until no slot joins (every write sets a flag to 1, so the fixed point
  // does not depend on the order)
  while (true) {
    int changed = 0;
    for (int s = tid; s < nB; s += blockDim.x) {
      if (m.in[s] || !sg_slot_ok(m, s)) continue;
      bool join = m.jin && m.jact[s];
      const int dg = G.deg[s];
      for (int e = 0; e < dg && !join; ++e) {
        const int u = G.nbr[(int64_t)nB * s + e];
        join = m.in[u] && gact[(int64_t)nB * s + e];
      }
      if (join) {
        m.in[s] = 1;
        changed = 1;
      }
    }
    if (!m.jin) {
      for (int s = tid; s < nB; s += blockDim.x)
        if (m.in[s] && m.jact[s]) {
          m.jin = 1;  // every writer writes 1
          changed = 1;
        }
    }
    if (!__syncthreads_or(changed)) break;
  }
  // local tokens and pool counts
  for (int s = tid; s < nB; s += blockDim.x) {
    int32_t c = 0;
    if (m.in[s]) {
      const auto pools = [&](int32_t k) { return k >= 0 ? (int32_t)(ix.off[k + 1] - ix.off[k]) : 0; };
      c = pools(m.ipair[s]) + (m.jin ? pools(m.jpair[s]) : 0);
      const int dg = G.deg[s];
      for (int e = 0; e < dg; ++e) {
        const int u = G.nbr[(int64_t)nB * s + e];
        if (u > s && m.in[u]) c += pools(G.pair[(int64_t)nB * s + e]);
      }
    }
    m.cnt[s] = c;
  }
  __syncthreads();
  if (tid == 0) {
    int loc = 2;
    m.ltok[0] = i;
    m.ltok[1] = j;
    for (int s = 0; s < nB; ++s)
      if (m.in[s]) {
        m.lidx[s] = (int16_t)loc;
        m.ltok[loc++] = G.tok[s];
      }
    m.n_loc = loc;
    m.direct_cnt = m.jin && m.direct >= 0 ? (int32_t)(ix.off[m.direct + 1] - ix.off[m.direct]) : 0;
    int32_t tot = m.direct_cnt;
    for (int s = 0; s < nB; ++s) {
      const int32_t c = m.cnt[s];
      m.cnt[s] = tot;  // exclusive offsets after {j, i}'s pools
      tot += c;
    }
    m.cnt[nB] = tot;
    m.npool = tot;
  }
  __syncthreads();
}

template <class Graph>
__device__ __forceinline__ int32_t sg_local(const Graph& G, const SubgraphSmem& m, int32_t t) {
  if (t == m.ltok[0]) return 0;
  if (t == m.ltok[1]) return 1;
  return m.lidx[G.slot_of[t]];
}

// Per row: the number of tokens the row lists (T, j omitted when it is not in T) and of its pools.
__global__ void __launch_bounds__(kSubgraphThreads)
    subgraph_plan_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                         const uint8_t* __restrict__ gact, const int64_t* __restrict__ token_in,
                         const int64_t* __restrict__ token_out, int64_t q, int64_t* __restrict__ ntok,
                         int64_t* __restrict__ npool) {
  __shared__ SubgraphSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    sg_setup(P, ix, A, G, gact, (int32_t)(token_in[r] - 1), (int32_t)(token_out[r] - 1), m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc - (m.jin ? 0 : 1);
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Sum over the CTA of one value per thread, in a fixed order: the xor butterfly 16 … 1 in each warp,
// then the warps' sums in warp order from +0.0.  Every thread gets the result.
template <class Smem>  // SubgraphSmem or BasketSmem (basket_kernels.cuh)
__device__ __forceinline__ double sg_cta_sum(double v, Smem& m) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(kFull, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) m.red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < kSubgraphWarps; ++w) t = __dadd_rn(t, m.red[w]);
  return t;
}

// The pool view of workspace pool e at ν = v (local prices).
__device__ __forceinline__ SplitPool sg_pool(const PathSets* P, const SubgraphWork& w, int64_t e, const double* v) {
  SplitPool sp = split_pool(P, w.ent[e], -1, 1.0);
  sp.v1 = v[w.ta[e]];
  sp.v2 = v[w.tb[e]];
  return sp;
}

__device__ __forceinline__ double sg_lower(int t) { return t == 0 ? 1.0 + kSubgraphSqrtEps : kSubgraphSqrtEps; }

// The box of slot t.  Exact-in: ν_i >= 1 + √eps, ν_t >= √eps otherwise.  Exact-out: ν_j = 1 (slot 1
// is fixed), ν_t >= √eps otherwise, i included.
template <bool OUT>
__device__ __forceinline__ double sg_lo(int t) { return OUT ? kSubgraphSqrtEps : sg_lower(t); }

// The rules of an exact-in (OUT false) or exact-out row, the only part of the solve that depends on the
// row kind (basket_kernels.cuh's BkRule gives the same for basket rows):
//   lin(m, t)     the linear term of slot t's gradient: lin at kLin (amt at j, or −y′ at i), else 0;
//   value(m)      the dual's linear value at ν = xt, lin·ν_kLin;
//   lo(m, t), fixed(m, t)   the box (sg_start's clamp included);
//   kBoxStart     false: the start is sg_start's (true: the box's lower bound, sg_box_start);
//   kOut, root(m) sg_start's root and clamp (exact-out: slot 1, j, fixed at 1);
//   evaluated(m, f)   sees the dual value f of every evaluation (nothing here);
//   merit(m, mx)  m_r from the CTA max mx = max_t ν_t·|pg_t|: mx / (δ·ν_j), or mx / (y·ν_i).
// Every value is the same IEEE operations in the same order as the rule's other uses, so a one-entry
// basket row gives an exact-in row's bits and a one-bought-entry buy row an exact-out row's.
template <bool OUT>
struct SgRule {
  static constexpr bool kOut = OUT;
  static constexpr bool kBoxStart = false;
  static constexpr int kLin = OUT ? 0 : 1;
  double lin, amt;
  __device__ __forceinline__ double lin_at(const SubgraphSmem&, int t) const { return t == kLin ? lin : 0.0; }
  __device__ __forceinline__ double value(const SubgraphSmem& m) const { return __dmul_rn(lin, m.xt[kLin]); }
  __device__ __forceinline__ double lo(const SubgraphSmem&, int t) const { return sg_lo<OUT>(t); }
  __device__ __forceinline__ bool fixed(const SubgraphSmem&, int t) const { return OUT && t == 1; }
  __device__ __forceinline__ int root(const SubgraphSmem&) const { return OUT ? 1 : 0; }
  __device__ __forceinline__ void evaluated(SubgraphSmem&, double) const {}
  __device__ __forceinline__ double merit(const SubgraphSmem& m, double mx) const {
    return __ddiv_rn(mx, __dmul_rn(amt, m.x[OUT ? 0 : 1]));
  }
};

// One evaluation at ν = xt: every pool's contributions, Ψ_t -> pt, gt = lin + Ψ, and the dual's
// value linᵀxt + Σ val (returned to every thread).
template <class Smem, class Rule>
__device__ double sg_evaluate(const PathSets* P, const SubgraphWork& w, Smem& m, const Rule& rule) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t np = m.npool;
  double vs = 0.0;
  for (int64_t e = tid; e < np; e += blockDim.x) {
    const SplitPool sp = sg_pool(P, w, e, m.xt);
    const Trade tr = split_legs(P, sp);
    const double a = __dsub_rn(tr.l1, tr.d1), b = __dsub_rn(tr.l2, tr.d2);
    w.ca[e] = a;
    w.cb[e] = b;
    vs = __dadd_rn(vs, __dadd_rn(__dmul_rn(sp.v1, a), __dmul_rn(sp.v2, b)));
  }
  const double V = sg_cta_sum(vs, m);  // (its syncs also publish ca, cb)
  for (int t = warp; t < m.n_loc; t += kSubgraphWarps) {
    double s = 0.0;
    for (int k = m.inc_off[t] + lane; k < m.inc_off[t + 1]; k += 32) {
      const int32_t v = w.inc[k];
      s = __dadd_rn(s, (v & 1) ? w.cb[v >> 1] : w.ca[v >> 1]);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(kFull, s, o));
    if (lane == 0) {
      m.pt[t] = s;
      m.gt[t] = __dadd_rn(rule.lin_at(m, t), s);
    }
  }
  __syncthreads();
  const double f = __dadd_rn(rule.value(m), V);
  rule.evaluated(m, f);
  return f;
}

// The scale of token t's term in the stop's mx = max_t scale_t·|pg_t|: ν_t, the value at ν of a unit
// of t's projected gradient.  Inventory rows (price_arb_kernels.cuh) floor it.
template <class Smem, class Rule>
__device__ __forceinline__ double sg_stop_scale(const Smem& m, const Rule&, int t) { return m.x[t]; }

// Accept xt: (s, y) into history slot `slot` when store, x <- xt, g <- gt, Ψ, the projected gradient
// and the Gram matrix of [S Y pg] (one warp per entry group, lanes over the tokens, butterfly).
// Returns the rule's m_r.
template <class Smem, class Rule>
__device__ double sg_commit(Smem& m, int slot, bool store, const Rule& rule) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = m.n_loc;
  if (tid == 0) m.mx = 0ull;
  for (int t = tid; t < n; t += blockDim.x) {
    const double xn = m.xt[t], gn = m.gt[t];
    if (store) {
      m.S[slot][t] = __dsub_rn(xn, m.x[t]);
      m.Y[slot][t] = __dsub_rn(gn, m.g[t]);
    }
    m.x[t] = xn;
    m.g[t] = gn;
    m.px[t] = m.pt[t];
    m.pg[t] = rule.fixed(m, t) || (xn <= rule.lo(m, t) && gn > 0.0) ? 0.0 : gn;
  }
  __syncthreads();
  double mx = 0.0;
  for (int t = tid; t < n; t += blockDim.x) mx = fmax(mx, __dmul_rn(sg_stop_scale(m, rule, t), fabs(m.pg[t])));
  for (int o = 16; o >= 1; o >>= 1) mx = fmax(mx, __shfl_xor_sync(kFull, mx, o));
  if (lane == 0) atomicMax(&m.mx, (unsigned long long)__double_as_longlong(mx));  // order-free max
  const auto col = [&](int c, int t) {
    return c < kSolverM ? m.S[c][t] : c < 2 * kSolverM ? m.Y[c - kSolverM][t] : m.pg[t];
  };
  for (int k = warp; k < kSolverK * kSolverK; k += kSubgraphWarps) {
    const int r = k / kSolverK, c = k % kSolverK;
    if (c < r) continue;
    double s = 0.0;
    for (int t = lane; t < n; t += 32) s = fma(col(r, t), col(c, t), s);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(kFull, s, o));
    if (lane == 0) m.W[r][c] = m.W[c][r] = s;
  }
  __syncthreads();
  return rule.merit(m, __longlong_as_double((long long)m.mx));
}

// The start ν⁰: ν_root = 1 (the rule's root: slot 0, i; exact-out: slot 1, j; basket buy rows: i's
// slot); then breadth-first rounds over the active pools: a token not yet priced gets the largest
// r(a → b)·ν_b over its pools to tokens priced in earlier rounds, r the no-trade boundary with a in j's
// role (the arbitrage scan's rate).  A token is priced once, so gaining cycles cannot inflate the
// start.  Then clamped to the rule's box (kOut: the root fixed at 1; every other slot >= lo(m, t)).
// Into xt.
template <class Smem, class Rule>
__device__ void sg_start(const PathSets* P, const SubgraphWork& w, Smem& m, const Rule& rule) {
  constexpr bool OUT = Rule::kOut;
  const int tid = threadIdx.x, n = m.n_loc, root = rule.root(m);
  for (int t = tid; t < n; t += blockDim.x) m.x[t] = m.xt[t] = t == root ? 1.0 : 0.0;
  __syncthreads();
  unsigned long long* nxt = reinterpret_cast<unsigned long long*>(m.xt);
  for (int round = 1; round < n; ++round) {
    int changed = 0;
    for (int64_t e = tid; e < m.npool; e += blockDim.x) {
      SplitPool sp = split_pool(P, w.ent[e], -1, 1.0);
      if (!sp.active) continue;
      for (int side = 0; side < 2; ++side) {
        const int32_t a = side ? w.tb[e] : w.ta[e], b = side ? w.ta[e] : w.tb[e];
        if (m.x[a] != 0.0 || !(m.x[b] > 0.0)) continue;  // a is priced once, from tokens priced before
        sp.x_is_j = side == 0;
        const double c = __dmul_rn(split_boundary(P, sp), m.x[b]);
        if (c > 0.0 && c < kPathInf) {
          atomicMax(nxt + a, (unsigned long long)__double_as_longlong(c));  // order-free max
          changed = 1;
        }
      }
    }
    const bool more = __syncthreads_or(changed);
    for (int t = tid; t < n; t += blockDim.x) m.x[t] = m.xt[t];
    __syncthreads();
    if (!more) break;
  }
  for (int t = tid; t < n; t += blockDim.x) m.xt[t] = OUT && t == root ? 1.0 : fmax(m.x[t], rule.lo(m, t));
  __syncthreads();
}

// The start of a rule with kBoxStart: every slot at its lower bound.  Into x and xt.
template <class Smem, class Rule>
__device__ __forceinline__ void sg_box_start(Smem& m, const Rule& rule) {
  for (int t = threadIdx.x; t < m.n_loc; t += blockDim.x) m.x[t] = m.xt[t] = rule.lo(m, t);
  __syncthreads();
}

// What workspace pool e could ever pay out of the token at local slot `slot` (exact-out rows: i,
// slot 0): 0 unless it is active and holds that token; a two-coin pool's reserve of it; a UniV3
// pool's f(DBL_MAX) for a tender of its other token, the walk to the end of its ladder
// (swap_crossing's unreachable test).
__device__ __forceinline__ double sg_capacity(const PathSets* P, const SubgraphWork& w, int64_t e, int32_t slot = 0) {
  const bool a = w.ta[e] == slot;
  if (!a && w.tb[e] != slot) return 0.0;
  const SplitPool sp = split_pool(P, w.ent[e], -1, 1.0);
  if (!sp.active) return 0.0;
  const SwapSet& S = P->s[sp.k];
  if ((sp.k >> 1) < 2) {
    const double2 R = S.R[sp.p];
    return a ? R.x : R.y;
  }
  return swap_pool<2>(S, sp.p).f(__longlong_as_double(kSwapOrdMax), !a);
}

// CTA b's workspace: workspace b of w.
__device__ __forceinline__ SubgraphWork sg_cta_work(const SubgraphWork& w) {
  const int64_t c = w.cap * blockIdx.x;
  SubgraphWork wb = w;
  wb.ent += c;
  wb.key += c;
  wb.ta += c;
  wb.tb += c;
  wb.inc += 2 * c;
  wb.ca += c;
  wb.cb += c;
  return wb;
}

// The pools of every slot s in T into the workspace at the offset the setup counted (cnt[s]): {s, i},
// then the row kind's side pairs of s (side(s, put)), then {s, u} for the slots u > s in T.  Then a
// barrier, which also publishes the row's leading pools.
template <class Smem, class Side, class Graph>
__device__ __forceinline__ void sg_gather(PairIndexView ix, const Graph& G, const SubgraphWork& w,
                                          const Smem& m, Side side) {
  for (int s = threadIdx.x; s < G.nB; s += blockDim.x) {
    if (!m.in[s]) continue;
    int64_t o = m.cnt[s];
    const auto put = [&](int64_t k) {
      if (k < 0) return;
      for (int64_t e = ix.off[k]; e < ix.off[k + 1]; ++e) w.ent[o++] = ix.pool[e];
    };
    put(m.ipair[s]);
    side(s, put);
    const int dg = G.deg[s];
    for (int e = 0; e < dg; ++e) {
      const int u = G.nbr[(int64_t)G.nB * s + e];
      if (u > s && m.in[u]) put(G.pair[(int64_t)G.nB * s + e]);
    }
  }
  __syncthreads();
}

// The row's np pools into global insertion order (a bitonic sort on (global index, entry), padded to a
// power of two), each pool's stored tokens as local slots (local(t), t 0-based), and for each of the n
// local tokens an incidence list in pool order (one warp per token, a ballot per 32 pools: count, then
// fill).
template <class Smem, class Local>
__device__ __forceinline__ void sg_order_pools(const PathSets* P, const SubgraphWork& w, Smem& m, int64_t np,
                                               int64_t n, Local local) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int64_t p2 = 1;
  while (p2 < np) p2 <<= 1;
  for (int64_t e = tid; e < p2; e += blockDim.x) {
    if (e < np) {
      const int64_t en = w.ent[e];
      const int k = (int)(en >> kPairSetShift);
      w.key[e] = P->s[k].gidx[en & kPairPosMask] & ~(1ll << 62);
    } else {
      w.key[e] = INT64_MAX;
      w.ent[e] = -1;
    }
  }
  __syncthreads();
  for (int64_t k = 2; k <= p2; k <<= 1)
    for (int64_t jj = k >> 1; jj > 0; jj >>= 1) {
      for (int64_t e = tid; e < p2; e += blockDim.x) {
        const int64_t o = e ^ jj;
        if (o > e) {
          const bool up = (e & k) == 0;
          const int64_t ke = w.key[e], ko = w.key[o];
          if (up ? ke > ko : ke < ko) {
            w.key[e] = ko;
            w.key[o] = ke;
            const int64_t t = w.ent[e];
            w.ent[e] = w.ent[o];
            w.ent[o] = t;
          }
        }
      }
      __syncthreads();
    }
  for (int64_t e = tid; e < np; e += blockDim.x) {
    const int64_t en = w.ent[e];
    const int k = (int)(en >> kPairSetShift);
    const int2 a = P->Ai[k][en & kPairPosMask];
    w.ta[e] = local(a.x);
    w.tb[e] = local(a.y);
  }
  __syncthreads();
  for (int t = warp; t < n; t += kSubgraphWarps) {
    int c = 0;
    for (int64_t b = 0; b < np; b += 32) {
      const int64_t e = b + lane;
      c += __popc(__ballot_sync(kFull, e < np && (w.ta[e] == t || w.tb[e] == t)));
    }
    if (lane == 0) m.inc_off[t + 1] = c;
  }
  __syncthreads();
  if (tid == 0) {
    m.inc_off[0] = 0;
    for (int t = 0; t < n; ++t) m.inc_off[t + 1] += m.inc_off[t];
  }
  __syncthreads();
  for (int t = warp; t < n; t += kSubgraphWarps) {
    int c = m.inc_off[t];
    for (int64_t b = 0; b < np; b += 32) {
      const int64_t e = b + lane;
      const bool ha = e < np && w.ta[e] == t, hb = e < np && w.tb[e] == t;
      const unsigned hit = __ballot_sync(kFull, ha || hb);
      if (ha || hb) w.inc[c + __popc(hit & ((1u << lane) - 1u))] = (int32_t)(2 * e + (hb ? 1 : 0));
      c += __popc(hit);
    }
  }
  __syncthreads();
}

// The absolute floor beside the relative stop: whether the committed mx = max_t ν_t·|pg_t| (m.mx) is at
// most the rows' atol.  Only rows that carry an atol have one (price_arb_kernels.cuh's InvArbRows).
template <class Smem, class Rows>
__device__ __forceinline__ bool sg_atol_met(const Smem&, const Rows&) { return false; }

// The solve's CTA-wide state: thread 0 decides, every thread reads after a barrier.
struct SgSolveState {
  LbfgsHistory hist;
  double f, t, merit;
  int state, status, iter, fev, small;
};

// cfmm_solve's projected L-BFGS (solver_control.cuh) on the row's dual over its n local tokens, every
// vector in shared memory, from sg_start (kBoxStart: sg_box_start) when solve (else nothing runs).
// Returns the solver status (−1: no solve) and sets merit to the last m_r; s keeps the iteration and
// evaluation counts.
template <class Smem, class Rule, class Rows>
__device__ __forceinline__ int sg_solve(const PathSets* P, const SubgraphWork& w, Smem& m, const Rule& rule,
                                        const Rows& R, int64_t n, bool solve, SgSolveState& s, double& merit) {
  const int tid = threadIdx.x;
  double f = 0.0;
  int status = -1;
  merit = 0.0;
  if (tid == 0) {
    s.iter = s.fev = s.small = 0;
    s.hist.cnt = s.hist.head = 0;
  }
  if (!solve) return status;
  for (int t = tid; t < n; t += blockDim.x)  // an empty history, as cfmm_solve's zeroed one
    for (int a = 0; a < kSolverM; ++a) m.S[a][t] = m.Y[a][t] = 0.0;
  if constexpr (Rule::kBoxStart)
    sg_box_start(m, rule);
  else
    sg_start(P, w, m, rule);
  f = sg_evaluate(P, w, m, rule);
  merit = sg_commit(m, 0, false, rule);
  if (tid == 0) {
    s.fev = 1;
    s.f = f;
    s.merit = merit;
  }
  __syncthreads();
  while (true) {
    __syncthreads();  // every thread has read the last decision
    // state: 0 run, 1 stop
    if (tid == 0) {
      s.state = 0;
      if (!(s.f == s.f)) s.status = 5, s.state = 1;
      else if (s.merit <= R.rtol || sg_atol_met(m, R)) s.status = 0, s.state = 1;
      else if (s.iter >= R.max_iter) s.status = 2, s.state = 1;
      else if (s.fev >= R.max_fun) s.status = 3, s.state = 1;
      else s.t = lbfgs_direction(m.W, s.hist, m.c);
    }
    __syncthreads();
    if (s.state) break;
    for (int t = tid; t < n; t += blockDim.x) {
      double v = __dmul_rn(m.c[kSolverK - 1], m.pg[t]);
#pragma unroll
      for (int a = 0; a < kSolverM; ++a) {
        v = fma(m.c[a], m.S[a][t], v);
        v = fma(m.c[kSolverM + a], m.Y[a][t], v);
      }
      m.d[t] = rule.fixed(m, t) || (m.x[t] <= rule.lo(m, t) && m.g[t] > 0.0) ? 0.0 : -v;
    }
    __syncthreads();
    int dec = kLsRetry;
    double f_new = s.f;
    for (int ls = 0; ls < 30 && s.fev < R.max_fun; ++ls) {
      const double t = s.t;
      double gd = 0.0, st2 = 0.0;
      for (int k = tid; k < n; k += blockDim.x) {
        const double y = rule.fixed(m, k) ? 1.0 : fmax(fma(t, m.d[k], m.x[k]), rule.lo(m, k));
        m.xt[k] = y;
        const double dx = __dsub_rn(y, m.x[k]);
        gd = fma(m.g[k], dx, gd);
        st2 = fma(dx, dx, st2);
      }
      const double gdx = sg_cta_sum(gd, m), step2 = sg_cta_sum(st2, m);
      f_new = sg_evaluate(P, w, m, rule);
      if (tid == 0) {
        ++s.fev;
        double tn = s.t;
        s.state = lbfgs_trial(s.f, f_new, gdx, step2, s.hist.cnt, tn);
        s.t = tn;
      }
      __syncthreads();
      dec = s.state;
      __syncthreads();
      if (dec != kLsRetry) break;
    }
    if (dec != kLsAccept) {
      if (tid == 0) {
        if (s.hist.cnt > 0 && dec != kLsStall) {
          s.hist.cnt = 0;  // drop the history and retry with steepest descent
          s.state = 0;
        } else {
          s.status = dec == kLsStall ? 1 : 4;
          s.state = 1;
        }
      }
      __syncthreads();
      if (s.state) break;
      continue;
    }
    const int slot = s.hist.head;
    const double mr = sg_commit(m, slot, true, rule);
    if (tid == 0) {
      lbfgs_store(m.W, slot, s.hist);
      ++s.iter;
      const double f_old = s.f;
      s.f = f_new;
      s.merit = mr;
      s.state = lbfgs_factr(f_old, f_new, R.factr, s.small) ? 1 : 0;
      if (s.state) s.status = 1;
    }
    __syncthreads();
    if (s.state) break;
  }
  merit = s.merit;
  return s.status;
}

// The legs of the row's np pools at ν = x into leg_off[r] .. (and, filled on execute, the transition).
template <bool EXEC, class Rows>
__device__ __forceinline__ void sg_legs(const PathSets* P, const SubgraphWork& w, const double* x, const SplitMoved& mv,
                                        const Rows& R, int64_t r, int64_t np, bool filled) {
  const int64_t l0 = R.leg_off[r];
  for (int64_t e = threadIdx.x; e < np; e += blockDim.x) {
    if (R.leg_entry) R.leg_entry[l0 + e] = w.ent[e];
    split_leg<EXEC>(P, filled, [&] { return sg_pool(P, w, e, x); }, mv, R.leg_delta, R.leg_lambda, l0 + e);
  }
}

// Row r on the current state.  Returns nothing; writes the row's outputs.  EXEC: the limit decides,
// and a filled row applies the transition of cfmm_apply_trades at its ν to each of its pools.  OUT:
// the row buys y = amount of i; its dual has lin = −y′ at i, y′ = y·(1 + rtol) rounded up, and ν_j
// fixed at 1; it is unreachable when y is at least what its pools holding i could pay out.
template <bool EXEC, bool OUT, class Graph>
__device__ void subgraph_row(const PathSets* P, PairIndexView ix, AdjView A, const Graph& G,
                             const uint8_t* gact, const SubgraphRows& R, const SubgraphWork& w, const SplitMoved& mv,
                             int64_t r, SubgraphSmem& m) {
  __shared__ SgSolveState s;
  const int tid = threadIdx.x;
  const int32_t j = (int32_t)(R.token_in[r] - 1), i = (int32_t)(R.token_out[r] - 1);
  const double amt = R.amount[r];
  const SgRule<OUT> rule{OUT ? -__fma_ru(amt, R.rtol, amt) : amt, amt};
  sg_setup(P, ix, A, G, gact, j, i, m);
  const int64_t np = m.npool, n = m.n_loc;
  // the pools: {j, i} first, then each slot's, at the offsets the setup counted
  if (tid == 0 && m.direct_cnt > 0) {
    for (int64_t e = ix.off[m.direct]; e < ix.off[m.direct + 1]; ++e) w.ent[e - ix.off[m.direct]] = ix.pool[e];
  }
  sg_gather(ix, G, w, m, [&](int s, auto& put) {
    if (m.jin) put(m.jpair[s]);
  });
  sg_order_pools(P, w, m, np, n, [&](int32_t t) { return sg_local(G, m, t); });
  // exact-out: the capacity of i over the row's pools, once, before any solve
  bool short_cap = false;
  if constexpr (OUT) {
    if (m.jin && amt > 0.0) {
      double c = 0.0;
      for (int64_t e = tid; e < np; e += blockDim.x) c = __dadd_rn(c, sg_capacity(P, w, e));
      short_cap = amt >= sg_cta_sum(c, m);
    }
  }
  const bool solve = m.jin && amt > 0.0 && !short_cap;
  double merit;
  const int status = sg_solve(P, w, m, rule, R, n, solve, s, merit);
  // status, the limit, the legs (and the transition on execute)
  const double received = solve ? m.px[0] : 0.0, paid = solve ? __dsub_rn(0.0, m.px[1]) : 0.0;
  uint8_t st = 0;  // CFMM_ORDER_FILLED (amount 0: zeros, no solve)
  if (amt > 0.0) {
    if (!m.jin || short_cap)
      st = 2;  // CFMM_ORDER_UNREACHABLE
    else if (status != 0 || (OUT && !(received >= amt)))
      st = 5;  // CFMM_ORDER_NOT_CONVERGED (exact-out: also a converged row short of y)
    else if (EXEC && R.limit && (OUT ? paid > R.limit[r] : received < R.limit[r]))
      st = 1;  // CFMM_ORDER_LIMIT; an equal limit fills
  }
  const bool filled = st == 0 && solve;
  sg_legs<EXEC>(P, w, m.x, mv, R, r, np, filled);
  if (R.token) {
    int64_t o = R.tok_off[r];
    for (int t = tid; t < n; t += blockDim.x) {
      if (t == 1 && !m.jin) continue;
      const int64_t at = o + (t >= 2 && !m.jin ? t - 1 : t);
      R.token[at] = m.ltok[t] + 1;
      R.nu[at] = solve ? m.x[t] : 0.0;
      R.psi[at] = solve ? m.px[t] : 0.0;
    }
  }
  if (tid == 0) {
    R.paid[r] = filled ? paid : 0.0;
    R.received[r] = filled ? received : 0.0;
    R.status[r] = st;
    R.solver_status[r] = status;
    R.iterations[r] = solve ? s.iter : 0;
    R.fun_evals[r] = solve ? s.fev : 0;
    R.merit[r] = solve ? merit : 0.0;
  }
  __syncthreads();  // the next row reuses the shared state and the workspace
}

// Exact-in rows rows[0 .. n) (null: 0 .. n), one CTA at a time each; CTA b uses workspace b.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    subgraph_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                    const uint8_t* __restrict__ gact, SubgraphRows R, SubgraphWork w, SplitMoved mv,
                    const int64_t* __restrict__ rows, int64_t n) {
  __shared__ SubgraphSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x)
    subgraph_row<EXEC, false>(P, ix, A, G, gact, R, wb, mv, rows ? rows[k] : k, m);
}

// Exact-out rows rows[0 .. n), as subgraph_kernel.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    subgraph_out_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                        const uint8_t* __restrict__ gact, SubgraphRows R, SubgraphWork w, SplitMoved mv,
                        const int64_t* __restrict__ rows, int64_t n) {
  __shared__ SubgraphSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x)
    subgraph_row<EXEC, true>(P, ix, A, G, gact, R, wb, mv, rows ? rows[k] : k, m);
}

// Per-row masks: subgraph_plan_kernel with each row's own slot graph.
__global__ void __launch_bounds__(kSubgraphThreads)
    subgraph_rows_plan_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M,
                              const int64_t* __restrict__ token_in, const int64_t* __restrict__ token_out, int64_t q,
                              int64_t* __restrict__ ntok, int64_t* __restrict__ npool) {
  __shared__ SubgraphSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    const RowGraph G = row_graph(P, ix, A, M, r);
    sg_setup(P, ix, A, G, rg_act(M), (int32_t)(token_in[r] - 1), (int32_t)(token_out[r] - 1), m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc - (m.jin ? 0 : 1);
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Per-row masks: exact-in (OUT false) or exact-out rows rows[0 .. n) (null: 0 .. n), as
// subgraph_kernel / subgraph_out_kernel, each over its own slot graph.
template <bool EXEC, bool OUT>
__global__ void __launch_bounds__(kSubgraphThreads)
    subgraph_rows_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M, SubgraphRows R,
                         SubgraphWork w, SplitMoved mv, const int64_t* __restrict__ rows, int64_t n) {
  __shared__ SubgraphSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    const int64_t r = rows ? rows[k] : k;
    const RowGraph G = row_graph(P, ix, A, M, r);
    subgraph_row<EXEC, OUT>(P, ix, A, G, rg_act(M), R, wb, mv, r, m);
  }
}

}  // namespace cfmm
