// basket_kernels.cuh -- token baskets liquidated over every pool among their allowed tokens: one dual
// solve per row (sm_90a; cfmm_quote_basket_orders / cfmm_execute_basket_orders, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// A row sells a basket of K <= kBasketMaxTokens tokens b_0 .. b_{K-1} for i: route! with
// BasketLiquidation(i, Δin) over the row's pools.  It is subgraph_kernels.cuh's row with the one side
// token j generalised to K basket tokens.  Its setup (bk_setup) is its own; after it, the row runs
// that file's pool gather, pool ordering, solve (sg_solve with this file's BkRule) and legs, and
// subgraph orders keep their own row kernel and setup (DESIGN §4.5).
//   setup   the pairs {b_k, s} and {i, s} for every slot s, {b_k, i} and {b_k, b_l}; the component T
//           of i over active pools; the local tokens (0 = i, then the basket tokens in T in basket
//           order, then T's slots ascending) and the row's pools: every pool of every pair inside T,
//           bitonic-sorted into global insertion order in the CTA's workspace, with a per-token
//           incidence list in that order;
//   solve   cfmm_solve's projected L-BFGS (solver_control.cuh) with every vector in shared memory;
//           the gradient is (δ_k at b_k) + Ψ and the dual value and the stop's denominator use
//           V = Σ_k δ_k·ν_k, added in basket order from the first term (one entry: δ·ν_j's bits);
//   legs    split_leg over the pools at the final ν: the legs and, on execute, the transition.
// The basket tokens' slot pairs ({b_k, s} and its activity, K·nB entries each) live in dynamic shared
// memory (bk_dyn_bytes).  basket_plan_kernel runs the setup only and reports each row's token and pool
// counts, which size the outputs and the workspace.
//
// basket_buy_kernel runs buy rows: rows whose entries include at least one bought entry (kind
// CFMM_SWAP_EXACT_OUT: buy y_l of b_l).  It is the same row with BUY set at compile time: the local
// order is the bought entries, then i, then the sold entries, then B ∩ T; lin is δ_k at sold and
// −y′_l = −y_l·(1 + rtol) (rounded up) at bought entries; ν_i is fixed at 1 and every other slot has
// ν_t >= √eps; the start prices from i's slot; the stop adds a term per bought entry; and a bought
// entry's capacity is checked before the solve (sg_capacity at its slot).  One bought entry and no
// sold entries give subgraph_out_kernel's outputs bit for bit.
//
// basket_limit_kernel runs limit rows (cfmm_quote_limit_orders / cfmm_execute_limit_orders): a basket
// row whose entries carry limit prices c_k (units of i per unit of b_k).  It is the basket row with LIM
// set at compile time: the box of entry k in T is ν_k >= fmax(c_k, √eps) (LimRule's per-slot lo, which
// also clamps the start), and an entry outside T with c_k > 0 is dropped rather than making the row
// unreachable.  Every c_k = 0 gives basket_kernel's outputs bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "subgraph_kernels.cuh"

namespace cfmm {

constexpr int kBasketMaxTokens = 16;  // CFMM_BASKET_MAX_TOKENS
constexpr uint8_t kBasketBought = 1;  // CFMM_SWAP_EXACT_OUT, the kind of a bought entry

// The rows of one call, their options, and their outputs (device arrays; tokens 1-based).
struct BasketRows {
  const int64_t* token_out;
  const int64_t* basket_off;  // [q+1]
  const int64_t* basket_token;
  const double* basket_amount;
  const double* limit;  // null: none
  int max_iter, max_fun;
  double rtol, factr;
  const int64_t* tok_off;  // [q+1] (setup counts, scanned)
  const int64_t* leg_off;  // [q+1]
  double* paid;            // [basket_off[q]]
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

// The rows of a limit call: the basket rows', plus each entry's limit price.
struct LimitRows : BasketRows {
  const double* limit_price;  // [basket_off[q]]: c_k, the least i per unit of b_k
};

// Shared state of one row.  kpair[k][l] is the pair {b_k, b_l}, kpair[k][k] the pair {b_k, i};
// kact the same pairs' activity.
struct BasketSmem {
  int32_t ipair[kSubgraphSlots], cnt[kSubgraphSlots + 1];
  int16_t lidx[kSubgraphSlots];
  uint8_t iact[kSubgraphSlots], in[kSubgraphSlots], side[kSubgraphSlots];
  int32_t ltok[kSubgraphLocal];
  int32_t inc_off[kSubgraphLocal + 1];
  double x[kSubgraphLocal], g[kSubgraphLocal], xt[kSubgraphLocal], gt[kSubgraphLocal], d[kSubgraphLocal],
      pg[kSubgraphLocal], px[kSubgraphLocal], pt[kSubgraphLocal];
  double S[kSolverM][kSubgraphLocal], Y[kSolverM][kSubgraphLocal];
  double W[kSolverK][kSolverK];
  double c[kSolverK];
  double red[kSubgraphWarps];
  double bamt[kBasketMaxTokens];  // δ of the basket tokens in T, in local order 1 .. nin
  int32_t btok[kBasketMaxTokens];
  int32_t kpair[kBasketMaxTokens][kBasketMaxTokens];
  uint8_t kact[kBasketMaxTokens][kBasketMaxTokens];
  uint8_t bin[kBasketMaxTokens];
  int8_t bloc[kBasketMaxTokens];  // local index of b_k, −1 outside T
  unsigned long long mx;
  int32_t nK, nin, n_loc, npool, basket_cnt;
  int changed;
};

// A buy row's shared state: the basket row's, plus the entries' kinds (in the caller's order, staged by
// basket_buy_kernel), lin per entry and the count of bought entries in T (their local slots
// 0 .. nout − 1; i's slot is nout).  bamt and blin are indexed by entry in local order, i skipped.
struct BasketBuySmem : BasketSmem {
  double blin[kBasketMaxTokens];
  uint8_t bkind[kBasketMaxTokens];
  int32_t nout;
};
template <bool BUY>
using BkSmem = std::conditional_t<BUY, BasketBuySmem, BasketSmem>;

// A limit row's shared state: the basket row's, plus the lower bound of every local slot (LimRule).
struct BasketLimitSmem : BasketSmem {
  double lo[kSubgraphLocal];
};

// The local slot of entry k (in local order, i skipped), and i's slot.
template <bool BUY>
__device__ __forceinline__ int bk_slot(const BkSmem<BUY>& m, int k) {
  if constexpr (BUY)
    return k < m.nout ? k : k + 1;
  else
    return k + 1;
}
template <bool BUY>
__device__ __forceinline__ int bk_root(const BkSmem<BUY>& m) {
  if constexpr (BUY)
    return m.nout;
  else
    return 0;
}
// The box of slot t: basket rows that of Swap (sg_lower); buy rows ν_i = 1 (bk_fixed) and ν_t >= √eps.
template <bool BUY>
__device__ __forceinline__ double bk_lo(int t) { return BUY ? kSubgraphSqrtEps : sg_lower(t); }
template <bool BUY>
__device__ __forceinline__ bool bk_fixed(const BkSmem<BUY>& m, int t) { return BUY && t == bk_root<BUY>(m); }

// The dynamic shared memory of a call whose longest basket has K entries: {b_k, s} and its activity.
__host__ __device__ __forceinline__ size_t bk_dyn_bytes(int K, int nB) {
  return ((size_t)K * (size_t)nB * 5 + 7) & ~(size_t)7;
}
extern __shared__ __align__(8) unsigned char bk_dyn[];

// Setup of the row trading btok[0 .. K) (1-based) for i (0-based): T, the local tokens and the pool
// count of every slot (cnt[s], the pools of the pairs {s, i}, {s, b_k} for b_k ∈ T, and {s, u} for
// slots u > s in T) and of the pairs among i and the basket tokens in T (basket_cnt).  BUY: the local
// order puts the bought entries (m.bkind) before i; the counts are the same.
template <bool BUY, class Graph>  // BestPathGraph or RowGraph
__device__ void bk_setup(const PathSets* P, PairIndexView ix, AdjView A, const Graph& G,
                         const uint8_t* __restrict__ gact, const int64_t* __restrict__ btok, int K, int32_t i,
                         BkSmem<BUY>& m) {
  const int tid = threadIdx.x, nB = G.nB;
  int32_t* bpair = reinterpret_cast<int32_t*>(bk_dyn);  // [K][nB]
  uint8_t* bact = bk_dyn + (size_t)4 * K * nB;          // [K][nB]
  for (int s = tid; s < nB; s += blockDim.x) {
    m.ipair[s] = -1;
    m.in[s] = 0;
    m.side[s] = 0;
    m.lidx[s] = -1;
  }
  for (int e = tid; e < K * nB; e += blockDim.x) bpair[e] = -1;
  if (tid < K) m.btok[tid] = (int32_t)(btok[tid] - 1);
  if (tid == 0) m.nK = K;
  __syncthreads();
  // the slots of i and of the basket tokens hold no B token; the pairs among them
  if (tid <= K) {
    const int32_t t = tid < K ? m.btok[tid] : i;
    const int32_t s = G.slot_of[t];
    if (s >= 0) m.side[s] = 1;
  }
  for (int e = tid; e < K * K; e += blockDim.x) {
    const int k = e / K, l = e % K;
    if (l < k) continue;
    const int32_t p = adj_pair(A, m.btok[k], l == k ? i : m.btok[l]);
    const uint8_t a = p >= 0 && subgraph_pair_active(P, ix, p);
    m.kpair[k][l] = m.kpair[l][k] = p;
    m.kact[k][l] = m.kact[l][k] = a;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k) side_pairs(A, G, m.btok[k], bpair + (size_t)k * nB);
  side_pairs(A, G, i, m.ipair);
  __syncthreads();
  for (int s = tid; s < nB; s += blockDim.x) {
    const bool ok = !m.side[s];
    m.iact[s] = ok && m.ipair[s] >= 0 && subgraph_pair_active(P, ix, m.ipair[s]);
    m.in[s] = m.iact[s];
  }
  for (int e = tid; e < K * nB; e += blockDim.x)
    bact[e] = !m.side[e % nB] && bpair[e] >= 0 && subgraph_pair_active(P, ix, bpair[e]);
  if (tid < K) m.bin[tid] = m.kact[tid][tid];
  __syncthreads();
  // the component of i: grow T until no slot or basket token joins (every write sets a flag to 1, so
  // the fixed point does not depend on the order)
  while (true) {
    int changed = 0;
    for (int s = tid; s < nB; s += blockDim.x) {
      if (m.in[s] || m.side[s]) continue;
      bool join = false;
      for (int k = 0; k < K && !join; ++k) join = m.bin[k] && bact[(size_t)k * nB + s];
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
    for (int e = tid; e < K * nB; e += blockDim.x) {
      const int k = e / nB;
      if (!m.bin[k] && m.in[e % nB] && bact[e]) {
        m.bin[k] = 1;  // every writer writes 1
        changed = 1;
      }
    }
    for (int e = tid; e < K * K; e += blockDim.x) {
      const int k = e / K, l = e % K;
      if (l != k && !m.bin[k] && m.bin[l] && m.kact[k][l]) {
        m.bin[k] = 1;
        changed = 1;
      }
    }
    if (!__syncthreads_or(changed)) break;
  }
  // local tokens and pool counts
  const auto pools = [&](int32_t k) { return k >= 0 ? (int32_t)(ix.off[k + 1] - ix.off[k]) : 0; };
  for (int s = tid; s < nB; s += blockDim.x) {
    int32_t c = 0;
    if (m.in[s]) {
      c = pools(m.ipair[s]);
      for (int k = 0; k < K; ++k)
        if (m.bin[k]) c += pools(bpair[(size_t)k * nB + s]);
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
    int loc = 1;
    int32_t tot = 0;
    if constexpr (BUY) {
      // the bought entries in T in the caller's order, then i, then the sold entries in T
      loc = 0;
      for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1) {
          m.nout = loc;
          m.ltok[loc++] = i;
        }
        for (int k = 0; k < K; ++k) {
          if (pass == 0) m.bloc[k] = -1;
          if (!m.bin[k] || (m.bkind[k] == kBasketBought) != (pass == 0)) continue;
          m.bloc[k] = (int8_t)loc;
          m.ltok[loc++] = m.btok[k];
          for (int l = k; l < K; ++l)
            if (m.bin[l]) tot += pools(m.kpair[k][l]);
        }
      }
    } else {
      m.ltok[0] = i;
      for (int k = 0; k < K; ++k) {
        m.bloc[k] = -1;
        if (!m.bin[k]) continue;
        m.bloc[k] = (int8_t)loc;
        m.ltok[loc++] = m.btok[k];
        for (int l = k; l < K; ++l)
          if (m.bin[l]) tot += pools(m.kpair[k][l]);
      }
    }
    m.nin = loc - 1;
    for (int s = 0; s < nB; ++s)
      if (m.in[s]) {
        m.lidx[s] = (int16_t)loc;
        m.ltok[loc++] = G.tok[s];
      }
    m.n_loc = loc;
    m.basket_cnt = tot;
    for (int s = 0; s < nB; ++s) {
      const int32_t c = m.cnt[s];
      m.cnt[s] = tot;  // exclusive offsets after the pools among i and the basket
      tot += c;
    }
    m.cnt[nB] = tot;
    m.npool = tot;
  }
  __syncthreads();
}

template <bool BUY, class Graph>
__device__ __forceinline__ int32_t bk_local(const Graph& G, const BkSmem<BUY>& m, int32_t t) {
  if constexpr (BUY) {
    for (int k = 0; k <= m.nin; ++k)  // i and the entries in T
      if (t == m.ltok[k]) return k;
  } else {
    if (t == m.ltok[0]) return 0;
    for (int k = 1; k <= m.nin; ++k)
      if (t == m.ltok[k]) return k;
  }
  return m.lidx[G.slot_of[t]];
}

// Per row: the number of tokens the row lists (T) and of its pools.
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_plan_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                       const uint8_t* __restrict__ gact, const int64_t* __restrict__ basket_off,
                       const int64_t* __restrict__ basket_token, const int64_t* __restrict__ token_out, int64_t q,
                       int64_t* __restrict__ ntok, int64_t* __restrict__ npool) {
  __shared__ BasketSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    const int64_t b0 = basket_off[r];
    bk_setup<false>(P, ix, A, G, gact, basket_token + b0, (int)(basket_off[r + 1] - b0), (int32_t)(token_out[r] - 1),
                    m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc;
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Σ_k c_k·v_k over the entries in T, in local order (the first term alone, not 0.0 + it).  c = bamt:
// V (basket rows: δ in basket order); c = blin: a buy row's linear term.
template <bool BUY>
__device__ __forceinline__ double bk_value(const BkSmem<BUY>& m, const double* c, const double* v) {
  double s = __dmul_rn(c[0], v[bk_slot<BUY>(m, 0)]);
  for (int k = 1; k < m.nin; ++k) s = __dadd_rn(s, __dmul_rn(c[k], v[bk_slot<BUY>(m, k)]));
  return s;
}

// The rules of a basket row (BUY false) or a buy row, as subgraph_kernels.cuh's SgRule: lin is δ_k at
// the basket tokens (buy rows: blin, δ_k at sold and −y′_l at bought entries), the dual's linear value
// bk_value over bamt (blin); the box is Swap's (buy rows: ν_i = 1 and ν_t >= √eps), the start's root
// is i's slot; m_r = mx / V, V = Σ_k amount_k·ν_k (y, not y′, at bought entries), and a buy row's m_r
// is at least ν_l·|pg_l| / (y_l·ν_l) for every bought entry with y_l > 0.
template <bool BUY>
struct BkRule {
  static constexpr bool kOut = BUY;
  static constexpr bool kBoxStart = false;
  __device__ __forceinline__ double lin_at(const BkSmem<BUY>& m, int t) const {
    if constexpr (BUY)
      return t == m.nout || t > m.nin ? 0.0 : m.blin[t < m.nout ? t : t - 1];
    else
      return t >= 1 && t <= m.nin ? m.bamt[t - 1] : 0.0;
  }
  __device__ __forceinline__ double value(const BkSmem<BUY>& m) const {
    if constexpr (BUY)
      return bk_value<BUY>(m, m.blin, m.xt);
    else
      return bk_value<BUY>(m, m.bamt, m.xt);
  }
  __device__ __forceinline__ double lo(const BkSmem<BUY>&, int t) const { return bk_lo<BUY>(t); }
  __device__ __forceinline__ bool fixed(const BkSmem<BUY>& m, int t) const { return bk_fixed<BUY>(m, t); }
  __device__ __forceinline__ int root(const BkSmem<BUY>& m) const { return bk_root<BUY>(m); }
  __device__ __forceinline__ void evaluated(BkSmem<BUY>&, double) const {}
  __device__ __forceinline__ double merit(const BkSmem<BUY>& m, double mx) const {
    double mr = __ddiv_rn(mx, bk_value<BUY>(m, m.bamt, m.x));
    if constexpr (BUY) {
      for (int l = 0; l < m.nout; ++l)
        if (m.bamt[l] > 0.0)
          mr = fmax(mr, __ddiv_rn(__dmul_rn(m.x[l], fabs(m.pg[l])), __dmul_rn(m.bamt[l], m.x[l])));
    }
    return mr;
  }
};

// The rules of a limit row: the basket row's (BkRule<false>), with the box read per slot from m.lo:
// ν_i >= 1 + √eps, ν_k >= fmax(c_k, √eps) at the entries in T, ν_t >= √eps elsewhere.
struct LimRule : BkRule<false> {
  __device__ __forceinline__ double lo(const BasketLimitSmem& m, int t) const { return m.lo[t]; }
};

template <bool BUY, bool LIM>
using BkRowSmem = std::conditional_t<LIM, BasketLimitSmem, BkSmem<BUY>>;
template <bool LIM>
using BkRows = std::conditional_t<LIM, LimitRows, BasketRows>;

// Row r on the current state.  Returns nothing; writes the row's outputs.  EXEC: the limit decides,
// and a filled row applies the transition of cfmm_apply_trades at its ν to each of its pools.  BUY:
// a buy row (its entries' kinds in m.bkind): the dual has lin = δ_k at sold and −y′_l at bought
// entries and ν_i fixed at 1; a bought entry with y_l at least what the row's pools holding b_l could
// pay out makes the row unreachable, and a row fills only when every bought entry with y_l > 0
// receives at least y_l.  LIM: a limit row (R.limit_price): the box of entry k in T is
// ν_k >= fmax(c_k, √eps), and an entry outside T with c_k > 0 is dropped (paid 0).
template <bool EXEC, bool BUY = false, bool LIM = false, class Graph>
__device__ void basket_row(const PathSets* P, PairIndexView ix, AdjView A, const Graph& G,
                             const uint8_t* gact, const BkRows<LIM>& R, const SubgraphWork& w, const SplitMoved& mv,
                             int64_t r, BkRowSmem<BUY, LIM>& m) {
  __shared__ SgSolveState s;
  __shared__ int s_any, s_unreach;
  const int tid = threadIdx.x;
  const int64_t b0 = R.basket_off[r];
  bk_setup<BUY>(P, ix, A, G, gact, R.basket_token + b0, (int)(R.basket_off[r + 1] - b0),
                (int32_t)(R.token_out[r] - 1), m);
  const int64_t np = m.npool, n = m.n_loc;
  // the amounts of the basket tokens in T; a positive amount outside T makes the row unreachable
  if constexpr (LIM) {
    // Swap's box, then each entry in T raised to its limit; an entry outside T with c_k > 0 cannot
    // fill at any price and is dropped, one with c_k = 0 follows the basket rule
    for (int t = tid; t < n; t += blockDim.x) m.lo[t] = sg_lower(t);
    __syncthreads();
    if (tid == 0) {
      int any = 0, unreach = 0;
      for (int k = 0; k < m.nK; ++k) {
        const double a = R.basket_amount[b0 + k], c = R.limit_price[b0 + k];
        if (m.bloc[k] >= 0) {
          m.bamt[m.bloc[k] - 1] = a;
          m.lo[m.bloc[k]] = fmax(c, kSubgraphSqrtEps);
          any |= a > 0.0;
        } else if (c == 0.0) {
          any |= a > 0.0;
          unreach |= a > 0.0;
        }
      }
      s_any = any;
      s_unreach = unreach;
    }
  } else if constexpr (BUY) {
    // bamt and blin by entry in local order (i skipped): δ and δ at sold, y and −y′ at bought entries
    if (tid == 0) {
      int any = 0, unreach = 0;
      for (int k = 0; k < m.nK; ++k) {
        const double a = R.basket_amount[b0 + k];
        any |= a > 0.0;
        if (m.bloc[k] >= 0) {
          const int e = m.bloc[k] < m.nout ? m.bloc[k] : m.bloc[k] - 1;
          m.bamt[e] = a;
          m.blin[e] = m.bkind[k] == kBasketBought ? -__fma_ru(a, R.rtol, a) : a;
        } else {
          unreach |= a > 0.0;
        }
      }
      s_any = any;
      s_unreach = unreach;
    }
  } else {
    if (tid == 0) {
      int any = 0, unreach = 0;
      for (int k = 0; k < m.nK; ++k) {
        const double a = R.basket_amount[b0 + k];
        any |= a > 0.0;
        if (m.bloc[k] >= 0)
          m.bamt[m.bloc[k] - 1] = a;
        else
          unreach |= a > 0.0;
      }
      s_any = any;
      s_unreach = unreach;
    }
  }
  // the pools: those among i and the basket first, then each slot's, at the offsets the setup counted
  if (tid == 0 && m.basket_cnt > 0) {
    int64_t o = 0;
    for (int k = 0; k < m.nK; ++k)
      for (int l = k; l < m.nK; ++l) {
        const int64_t p = m.kpair[k][l];
        if (!m.bin[k] || !m.bin[l] || p < 0) continue;
        for (int64_t e = ix.off[p]; e < ix.off[p + 1]; ++e) w.ent[o++] = ix.pool[e];
      }
  }
  const int32_t* bpair = reinterpret_cast<const int32_t*>(bk_dyn);
  sg_gather(ix, G, w, m, [&](int s, auto& put) {
    for (int k = 0; k < m.nK; ++k)
      if (m.bin[k]) put(bpair[(size_t)k * G.nB + s]);
  });
  sg_order_pools(P, w, m, np, n, [&](int32_t t) { return bk_local<BUY>(G, m, t); });
  // buy rows: the capacity of each bought entry over the row's pools, once, before any solve; a
  // shortfall makes the row unreachable
  if constexpr (BUY) {
    if (s_any && !s_unreach) {
      bool short_cap = false;
      for (int l = 0; l < m.nout; ++l) {
        const double y = m.bamt[l];
        if (!(y > 0.0)) continue;
        double c = 0.0;
        for (int64_t e = tid; e < np; e += blockDim.x) c = __dadd_rn(c, sg_capacity(P, w, e, l));
        short_cap |= y >= sg_cta_sum(c, m);
      }
      if (tid == 0 && short_cap) s_unreach = 1;
      __syncthreads();
    }
  }
  const bool any = s_any, solve = any && !s_unreach;
  double merit;
  const int status = sg_solve(P, w, m, std::conditional_t<LIM, LimRule, BkRule<BUY>>{}, R, n, solve, s, merit);
  // status, the limit, the legs (and the transition on execute)
  const double received = solve ? m.px[bk_root<BUY>(m)] : 0.0;
  uint8_t st = 0;  // CFMM_ORDER_FILLED (amounts all 0: zeros, no solve)
  if (any) {
    if (s_unreach)
      st = 2;  // CFMM_ORDER_UNREACHABLE
    else if (status != 0)
      st = 5;  // CFMM_ORDER_NOT_CONVERGED
    else if (EXEC && R.limit && received < R.limit[r])
      st = 1;  // CFMM_ORDER_LIMIT; an equal limit fills (buy rows: received may be negative)
  }
  if constexpr (BUY) {
    // a converged buy row short of a bought y_l > 0 is not converged, whatever its limit
    if (solve && status == 0)
      for (int l = 0; l < m.nout; ++l)
        if (m.bamt[l] > 0.0 && !(m.px[l] >= m.bamt[l])) st = 5;
  }
  const bool filled = st == 0 && solve;
  sg_legs<EXEC>(P, w, m.x, mv, R, r, np, filled);
  if (R.token) {
    const int64_t o = R.tok_off[r];
    for (int t = tid; t < n; t += blockDim.x) {
      R.token[o + t] = m.ltok[t] + 1;
      R.nu[o + t] = solve ? m.x[t] : 0.0;
      R.psi[o + t] = solve ? m.px[t] : 0.0;
    }
  }
  if (tid < m.nK) {
    const int b = m.bloc[tid];
    R.paid[b0 + tid] = filled && b >= 0 ? __dsub_rn(0.0, m.px[b]) : 0.0;
  }
  if (tid == 0) {
    R.received[r] = filled ? received : 0.0;
    R.status[r] = st;
    R.solver_status[r] = status;
    R.iterations[r] = solve ? s.iter : 0;
    R.fun_evals[r] = solve ? s.fev : 0;
    R.merit[r] = solve ? merit : 0.0;
  }
  __syncthreads();  // the next row reuses the shared state and the workspace
}

// Sell-only rows rows[0 .. n) (null: 0 .. n), one CTA at a time each; CTA b uses workspace b.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                    const uint8_t* __restrict__ gact, BasketRows R, SubgraphWork w, SplitMoved mv,
                    const int64_t* __restrict__ rows, int64_t n) {
  __shared__ BasketSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x)
    basket_row<EXEC>(P, ix, A, G, gact, R, wb, mv, rows ? rows[k] : k, m);
}

// Buy rows rows[0 .. n), as basket_kernel; kind [basket_off[q]] holds every entry's kind.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_buy_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                      const uint8_t* __restrict__ gact, BasketRows R, const uint8_t* __restrict__ kind, SubgraphWork w,
                      SplitMoved mv, const int64_t* __restrict__ rows, int64_t n) {
  __shared__ BasketBuySmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    const int64_t r = rows[k], b0 = R.basket_off[r];
    // (the previous row ended at a barrier, and the setup's barriers publish these before any read)
    if (threadIdx.x < R.basket_off[r + 1] - b0) m.bkind[threadIdx.x] = kind[b0 + threadIdx.x];
    basket_row<EXEC, true>(P, ix, A, G, gact, R, wb, mv, r, m);
  }
}

// Limit rows rows[0 .. n) (null: 0 .. n), as basket_kernel.
template <bool EXEC>
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_limit_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                        const uint8_t* __restrict__ gact, LimitRows R, SubgraphWork w, SplitMoved mv,
                        const int64_t* __restrict__ rows, int64_t n) {
  __shared__ BasketLimitSmem m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x)
    basket_row<EXEC, false, true>(P, ix, A, G, gact, R, wb, mv, rows ? rows[k] : k, m);
}

// Per-row masks: basket_plan_kernel with each row's own slot graph.
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_rows_plan_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M,
                            const int64_t* __restrict__ basket_off, const int64_t* __restrict__ basket_token,
                            const int64_t* __restrict__ token_out, int64_t q, int64_t* __restrict__ ntok,
                            int64_t* __restrict__ npool) {
  __shared__ BasketSmem m;
  for (int64_t r = blockIdx.x; r < q; r += gridDim.x) {
    const int64_t b0 = basket_off[r];
    const RowGraph G = row_graph(P, ix, A, M, r);
    bk_setup<false>(P, ix, A, G, rg_act(M), basket_token + b0, (int)(basket_off[r + 1] - b0),
                    (int32_t)(token_out[r] - 1), m);
    if (threadIdx.x == 0) {
      ntok[r] = m.n_loc;
      npool[r] = m.npool;
    }
    __syncthreads();
  }
}

// Per-row masks: sell-only (BUY and LIM false), buy (BUY; kind as basket_buy_kernel's) or limit (LIM)
// rows rows[0 .. n) (null: 0 .. n), as basket_kernel / basket_buy_kernel / basket_limit_kernel, each
// over its own slot graph.
template <bool EXEC, bool BUY, bool LIM>
__global__ void __launch_bounds__(kSubgraphThreads)
    basket_rows_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, RowMasks M, BkRows<LIM> R,
                       const uint8_t* __restrict__ kind, SubgraphWork w, SplitMoved mv,
                       const int64_t* __restrict__ rows, int64_t n) {
  __shared__ BkRowSmem<BUY, LIM> m;
  const SubgraphWork wb = sg_cta_work(w);
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    const int64_t r = rows ? rows[k] : k;
    if constexpr (BUY) {
      const int64_t b0 = R.basket_off[r];
      if (threadIdx.x < R.basket_off[r + 1] - b0) m.bkind[threadIdx.x] = kind[b0 + threadIdx.x];
    }
    const RowGraph G = row_graph(P, ix, A, M, r);
    basket_row<EXEC, BUY, LIM>(P, ix, A, G, rg_act(M), R, wb, mv, r, m);
  }
}

}  // namespace cfmm
