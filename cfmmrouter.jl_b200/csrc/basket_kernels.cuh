// basket_kernels.cuh -- token baskets liquidated over every pool among their allowed tokens: one dual
// solve per row (sm_90a; cfmm_quote_basket_orders / cfmm_execute_basket_orders, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// A row sells a basket of K <= kBasketMaxTokens tokens b_0 .. b_{K-1} for i: route! with
// BasketLiquidation(i, Δin) over the row's pools.  It is subgraph_kernels.cuh's row with the one side
// token j generalised to K basket tokens, and shares that file's pair activity (subgraph_act_kernel),
// workspace, side pairs, CTA sum, pool view and start; subgraph orders keep their own row kernel.
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

// The pair {a, b} from a's adjacency list (bisected), −1 when there is none.
__device__ __forceinline__ int32_t bk_pair(AdjView A, int32_t a, int32_t b) {
  int64_t lo = A.off[a], hi = A.off[a + 1];
  const int64_t a1 = hi;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (A.nbr[mid] < b)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < a1 && A.nbr[lo] == b ? A.pair[lo] : -1;
}

// Setup of the row trading btok[0 .. K) (1-based) for i (0-based): T, the local tokens and the pool
// count of every slot (cnt[s], the pools of the pairs {s, i}, {s, b_k} for b_k ∈ T, and {s, u} for
// slots u > s in T) and of the pairs among i and the basket tokens in T (basket_cnt).  BUY: the local
// order puts the bought entries (m.bkind) before i; the counts are the same.
template <bool BUY>
__device__ void bk_setup(const PathSets* P, PairIndexView ix, AdjView A, const BestPathGraph& G,
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
    const int32_t p = bk_pair(A, m.btok[k], l == k ? i : m.btok[l]);
    const uint8_t a = p >= 0 && subgraph_pair_active(P, ix, p);
    m.kpair[k][l] = m.kpair[l][k] = p;
    m.kact[k][l] = m.kact[l][k] = a;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k) sg_side_pairs(A, G, m.btok[k], bpair + (size_t)k * nB);
  sg_side_pairs(A, G, i, m.ipair);
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

template <bool BUY>
__device__ __forceinline__ int32_t bk_local(const BestPathGraph& G, const BkSmem<BUY>& m, int32_t t) {
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

// One evaluation at ν = xt: every pool's contributions, Ψ_t -> pt, gt = lin + Ψ, and the dual's
// value linᵀxt + Σ val (returned to every thread).
template <bool BUY>
__device__ double bk_evaluate(const PathSets* P, const SubgraphWork& w, BkSmem<BUY>& m) {
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
      if constexpr (BUY)
        m.gt[t] = __dadd_rn(t == m.nout || t > m.nin ? 0.0 : m.blin[t < m.nout ? t : t - 1], s);
      else
        m.gt[t] = __dadd_rn(t >= 1 && t <= m.nin ? m.bamt[t - 1] : 0.0, s);
    }
  }
  __syncthreads();
  if constexpr (BUY)
    return __dadd_rn(bk_value<BUY>(m, m.blin, m.xt), V);
  else
    return __dadd_rn(bk_value<BUY>(m, m.bamt, m.xt), V);
}

// Accept xt: (s, y) into history slot `slot` when store, x <- xt, g <- gt, Ψ, the projected gradient
// and the Gram matrix of [S Y pg] (one warp per entry group, lanes over the tokens, butterfly).
// Returns m_r = max_t ν_t·|pg_t| / V, V = Σ_k amount_k·ν_k (y, not y′, at bought entries); a buy
// row's m_r is at least ν_l·|pg_l| / (y_l·ν_l) for every bought entry with y_l > 0.
template <bool BUY>
__device__ double bk_commit(BkSmem<BUY>& m, int slot, bool store) {
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
    m.pg[t] = bk_fixed<BUY>(m, t) || (xn <= bk_lo<BUY>(t) && gn > 0.0) ? 0.0 : gn;
  }
  __syncthreads();
  double mx = 0.0;
  for (int t = tid; t < n; t += blockDim.x) mx = fmax(mx, __dmul_rn(m.x[t], fabs(m.pg[t])));
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
  double mr = __ddiv_rn(__longlong_as_double((long long)m.mx), bk_value<BUY>(m, m.bamt, m.x));
  if constexpr (BUY) {
    for (int l = 0; l < m.nout; ++l)
      if (m.bamt[l] > 0.0)
        mr = fmax(mr, __ddiv_rn(__dmul_rn(m.x[l], fabs(m.pg[l])), __dmul_rn(m.bamt[l], m.x[l])));
  }
  return mr;
}

// Row r on the current state.  Returns nothing; writes the row's outputs.  EXEC: the limit decides,
// and a filled row applies the transition of cfmm_apply_trades at its ν to each of its pools.  BUY:
// a buy row (its entries' kinds in m.bkind): the dual has lin = δ_k at sold and −y′_l at bought
// entries and ν_i fixed at 1; a bought entry with y_l at least what the row's pools holding b_l could
// pay out makes the row unreachable, and a row fills only when every bought entry with y_l > 0
// receives at least y_l.
template <bool EXEC, bool BUY = false>
__device__ void basket_row(const PathSets* P, PairIndexView ix, AdjView A, const BestPathGraph& G,
                             const uint8_t* gact, const BasketRows& R, const SubgraphWork& w, const SplitMoved& mv,
                             int64_t r, BkSmem<BUY>& m) {
  __shared__ LbfgsHistory hist;
  __shared__ double s_f, s_t, s_merit;
  __shared__ int s_state, s_status, s_iter, s_fev, s_small, s_any, s_unreach;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t b0 = R.basket_off[r];
  bk_setup<BUY>(P, ix, A, G, gact, R.basket_token + b0, (int)(R.basket_off[r + 1] - b0),
                (int32_t)(R.token_out[r] - 1), m);
  const int64_t np = m.npool, n = m.n_loc;
  // the amounts of the basket tokens in T; a positive amount outside T makes the row unreachable
  if constexpr (BUY) {
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
  for (int s = tid; s < G.nB; s += blockDim.x) {
    if (!m.in[s]) continue;
    int64_t o = m.cnt[s];
    const auto put = [&](int64_t k) {
      if (k < 0) return;
      for (int64_t e = ix.off[k]; e < ix.off[k + 1]; ++e) w.ent[o++] = ix.pool[e];
    };
    put(m.ipair[s]);
    for (int k = 0; k < m.nK; ++k)
      if (m.bin[k]) put(bpair[(size_t)k * G.nB + s]);
    const int dg = G.deg[s];
    for (int e = 0; e < dg; ++e) {
      const int u = G.nbr[(int64_t)G.nB * s + e];
      if (u > s && m.in[u]) put(G.pair[(int64_t)G.nB * s + e]);
    }
  }
  __syncthreads();
  // global insertion order: a bitonic sort on (global index, entry), padded to a power of two
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
    w.ta[e] = bk_local<BUY>(G, m, a.x);
    w.tb[e] = bk_local<BUY>(G, m, a.y);
  }
  __syncthreads();
  // incidence lists in pool order: one warp per token, a ballot per 32 pools (count, then fill)
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
  // the solve
  const bool any = s_any, solve = any && !s_unreach;
  double f = 0.0, merit = 0.0;
  int status = -1;
  if (tid == 0) {
    s_iter = s_fev = s_small = 0;
    hist.cnt = hist.head = 0;
  }
  if (solve) {
    for (int t = tid; t < n; t += blockDim.x)  // an empty history, as cfmm_solve's zeroed one
      for (int a = 0; a < kSolverM; ++a) m.S[a][t] = m.Y[a][t] = 0.0;
    if constexpr (BUY)
      sg_start<BasketBuySmem, true>(P, w, m, bk_root<BUY>(m));
    else
      sg_start(P, w, m);
    f = bk_evaluate<BUY>(P, w, m);
    merit = bk_commit<BUY>(m, 0, false);
    if (tid == 0) {
      s_fev = 1;
      s_f = f;
      s_merit = merit;
    }
    __syncthreads();
    while (true) {
      __syncthreads();  // every thread has read the last decision
      // state: 0 run, 1 stop
      if (tid == 0) {
        s_state = 0;
        if (!(s_f == s_f)) s_status = 5, s_state = 1;
        else if (s_merit <= R.rtol) s_status = 0, s_state = 1;
        else if (s_iter >= R.max_iter) s_status = 2, s_state = 1;
        else if (s_fev >= R.max_fun) s_status = 3, s_state = 1;
        else s_t = lbfgs_direction(m.W, hist, m.c);
      }
      __syncthreads();
      if (s_state) break;
      for (int t = tid; t < n; t += blockDim.x) {
        double v = __dmul_rn(m.c[kSolverK - 1], m.pg[t]);
#pragma unroll
        for (int a = 0; a < kSolverM; ++a) {
          v = fma(m.c[a], m.S[a][t], v);
          v = fma(m.c[kSolverM + a], m.Y[a][t], v);
        }
        m.d[t] = bk_fixed<BUY>(m, t) || (m.x[t] <= bk_lo<BUY>(t) && m.g[t] > 0.0) ? 0.0 : -v;
      }
      __syncthreads();
      int dec = kLsRetry;
      double f_new = s_f;
      for (int ls = 0; ls < 30 && s_fev < R.max_fun; ++ls) {
        const double t = s_t;
        double gd = 0.0, st2 = 0.0;
        for (int k = tid; k < n; k += blockDim.x) {
          const double y = bk_fixed<BUY>(m, k) ? 1.0 : fmax(fma(t, m.d[k], m.x[k]), bk_lo<BUY>(k));
          m.xt[k] = y;
          const double dx = __dsub_rn(y, m.x[k]);
          gd = fma(m.g[k], dx, gd);
          st2 = fma(dx, dx, st2);
        }
        const double gdx = sg_cta_sum(gd, m), step2 = sg_cta_sum(st2, m);
        f_new = bk_evaluate<BUY>(P, w, m);
        if (tid == 0) {
          ++s_fev;
          double tn = s_t;
          s_state = lbfgs_trial(s_f, f_new, gdx, step2, hist.cnt, tn);
          s_t = tn;
        }
        __syncthreads();
        dec = s_state;
        __syncthreads();
        if (dec != kLsRetry) break;
      }
      if (dec != kLsAccept) {
        if (tid == 0) {
          if (hist.cnt > 0 && dec != kLsStall) {
            hist.cnt = 0;  // drop the history and retry with steepest descent
            s_state = 0;
          } else {
            s_status = dec == kLsStall ? 1 : 4;
            s_state = 1;
          }
        }
        __syncthreads();
        if (s_state) break;
        continue;
      }
      const int slot = hist.head;
      const double mr = bk_commit<BUY>(m, slot, true);
      if (tid == 0) {
        lbfgs_store(m.W, slot, hist);
        ++s_iter;
        const double f_old = s_f;
        s_f = f_new;
        s_merit = mr;
        s_state = lbfgs_factr(f_old, f_new, R.factr, s_small) ? 1 : 0;
        if (s_state) s_status = 1;
      }
      __syncthreads();
      if (s_state) break;
    }
    status = s_status;
    merit = s_merit;
  }
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
  const int64_t l0 = R.leg_off[r];
  for (int64_t e = tid; e < np; e += blockDim.x) {
    if (R.leg_entry) R.leg_entry[l0 + e] = w.ent[e];
    split_leg<EXEC>(P, filled, [&] { return sg_pool(P, w, e, m.x); }, mv, R.leg_delta, R.leg_lambda, l0 + e);
  }
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
    R.iterations[r] = solve ? s_iter : 0;
    R.fun_evals[r] = solve ? s_fev : 0;
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
  const int64_t c = w.cap * blockIdx.x;
  SubgraphWork wb = w;
  wb.ent += c;
  wb.key += c;
  wb.ta += c;
  wb.tb += c;
  wb.inc += 2 * c;
  wb.ca += c;
  wb.cb += c;
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

}  // namespace cfmm
