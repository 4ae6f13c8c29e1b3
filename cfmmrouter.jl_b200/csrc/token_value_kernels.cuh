// token_value_kernels.cuh -- the token values of cfmm_quote_token_values (sm_90a, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// One root per row, every token a destination: a single-source dynamic programme over "at most h
// hops", run level by level as pool-parallel passes over the six pool sets (no pair index).  A group
// of up to kTvMaxGroup rows shares each pass; every array of the group is per row except the
// frontier masks, whose bit r belongs to row r alone, so a row's bits do not depend on its group.
//
//   tv_init_kernel      per token: the group's level-0 values, the root in the frontier
//   tv_relax_kernel     per pool position, level h: for each row whose frontier (the tokens that
//                       changed at level h−1) holds one of the pool's tokens, the hop's quote
//                       (path_hop_f / path_hop_exact_out, cfmm_quote_swaps / _exact_out bit for bit),
//                       kept when it beats the target's level h−1 value and merged into the target's
//                       slot with a 16-byte compare-and-swap on the rank key below
//   tv_finalize_kernel  per token, level h: the slot's winner becomes the value and the level-h
//                       predecessor (neighbour token, global insertion index), the slot is cleared,
//                       the next frontier mask and the per-row change counts are written
//   tv_rebuild_kernel   per (row, token): the walk back through the predecessors for hops and the
//                       repeated-pool check
//   tv_path_kernel      per requested (row, token): the walk in path order, priced by path_run (the
//                       code of cfmm_quote_paths)
// A level whose previous level changed no token of any row of the group returns at once, so a call
// launches a fixed number of kernels and stops early without a host round trip.
// cfmm_quote_token_values_net adds tv_select_kernel after each finalize (the best level net of a
// per-hop cost, per row and token), and tv_rebuild_kernel / tv_path_kernel walk from the selected
// level.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "best_path_kernels.cuh"

namespace cfmm {

constexpr int kTvMaxGroup = 64;       // rows per pass: one bit each in a frontier mask
constexpr int kTvThreads = 256;
constexpr int kTvMaxHops = 8;        // CFMM_PATH_MAX_HOPS
constexpr uint8_t kTvNever = 0xff;    // lvl of a token the row never reached
constexpr uint64_t kTvNoPred = ~0ull; // pred of a token that did not change at that level

// The rank key of a candidate, as one unsigned 128-bit number where larger ranks first: the high
// word is the amount's bits (exact-in; positive doubles order as their bits) or their complement
// (exact-out: the smaller amount first), the low word the complement of (neighbour token << 32 |
// global insertion index), so the smaller neighbour and then the earlier pool win a tie.  0 is the
// empty slot: no candidate maps to it (exact-in amounts are > 0, exact-out amounts finite).
__device__ __forceinline__ unsigned __int128 tv_key(double c, bool out, uint32_t nbr, uint32_t gi) {
  const uint64_t b = (uint64_t)__double_as_longlong(c);
  const uint64_t lo = ~(((uint64_t)nbr << 32) | gi);
  return ((unsigned __int128)(out ? ~b : b) << 64) | lo;
}

// The larger of *slot and v into *slot.  The first guess is the empty slot, so the slot is only
// ever read through the compare-and-swap (a plain 16-byte load could pair halves of two writes).
__device__ __forceinline__ void tv_merge(unsigned __int128* slot, unsigned __int128 v) {
  unsigned __int128 old = 0;
  while (true) {
    const unsigned __int128 seen = atomicCAS(slot, old, v);
    if (seen == old || seen >= v) return;
    old = seen;
  }
}

// The device positions of the six sets as one range: set k holds start[k] .. start[k+1).
struct TvSets {
  int64_t start[kPathSets + 1];
};

// The group's rows (pointers at the group's first row) and workspace, n = n_tokens, H = max_hops.
struct TvWork {
  const int64_t* root;     // [G] 1-based
  const uint8_t* kind;     // [G]
  const double* amount;    // [G]
  const uint8_t* allowed;  // [n] or null
  int G, H;
  int64_t n;
  double* val;             // [G][n]  the value at the last level run
  unsigned __int128* best; // [G][n]  the merge slots of the level being run
  uint8_t* lvl;            // [G][n]  the level a token last changed at (kTvNever: unreached)
  uint64_t* pred;          // [G][H][n]  (neighbour << 32 | global insertion index) at level h+1
  uint64_t* fmask;         // [2][n]  frontier masks, level h at h & 1
  int32_t* cnt;            // [G][H+1]  tokens changed per row and level
  int32_t* tot;            // [H+1]  summed over the group
};

__device__ __forceinline__ bool tv_out(const TvWork& W, int r) { return W.kind[r] != 0; }

__global__ void tv_init_kernel(TvWork W) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) {
    for (int r = 0; r < W.G; ++r)
      for (int h = 0; h <= W.H; ++h) W.cnt[r * (W.H + 1) + h] = h == 0;
    for (int h = 0; h <= W.H; ++h) W.tot[h] = h == 0 ? W.G : 0;
  }
  if (t >= W.n) return;
  uint64_t mask = 0;
  for (int r = 0; r < W.G; ++r) {
    const int64_t i = (int64_t)r * W.n + t;
    const bool is_root = W.root[r] - 1 == t;
    W.val[i] = is_root ? W.amount[r] : (tv_out(W, r) ? kPathInf : 0.0);
    W.lvl[i] = is_root ? 0 : kTvNever;
    W.best[i] = 0;
    mask |= (uint64_t)is_root << r;
  }
  W.fmask[t] = mask;
}

// Level h over every pool position of the six sets.  Exact-in: the frontier token u tenders a(u)
// and the other token t receives f(a(u)).  Exact-out: the frontier token v is wanted, c(v) of it,
// and the other token u tenders x*(c(v)).  Either way the frontier token is the neighbour in the
// rank key and the other token the target.
__global__ void __launch_bounds__(kTvThreads) tv_relax_kernel(const PathSets* __restrict__ P, TvSets S, TvWork W,
                                                               int h) {
  if (W.tot[h - 1] == 0) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int k = 0;
  while (k < kPathSets && i >= S.start[k + 1]) ++k;
  if (k == kPathSets) return;
  const int64_t p = i - S.start[k];
  const SwapSet& s = P->s[k];
  const int64_t g = s.gidx[p];
  if (g < 0 || (s.active && !s.active[p])) return;  // padding, retired
  const int2 a = P->Ai[k][p];
  const uint64_t* fm = W.fmask + (size_t)((h - 1) & 1) * W.n;
  const uint64_t ma = fm[a.x], mb = fm[a.y];
  if (!(ma | mb)) return;
  const bool sw = (k >> 1) < 2 && ((g >> 62) & 1);
  const uint32_t gi = (uint32_t)(g & ~(1ll << 62));
  for (int side = 0; side < 2; ++side) {
    const int32_t src = side ? a.y : a.x, dst = side ? a.x : a.y;
    uint64_t m = side ? mb : ma;
    if (!m || (W.allowed && !W.allowed[dst])) continue;
    // the ingest token 1 of the pool is a.x unless it is stored exchanged
    const bool src_tok1 = (side == 0) != sw;
    while (m) {
      const int r = __ffsll((long long)m) - 1;
      m &= m - 1;
      if (W.root[r] - 1 == dst) continue;
      const bool out = tv_out(W, r);
      const double vs = W.val[(int64_t)r * W.n + src], vt = W.val[(int64_t)r * W.n + dst];
      double c;
      if (!out) {
        c = path_hop_f(P, k, p, vs, src_tok1);
        if (!(c > vt)) continue;  // NaN, nothing out, or no better than level h−1
      } else {
        c = path_hop_exact_out(P, k, p, vs, !src_tok1);
        if (!(c < vt)) continue;  // NaN, unreachable, or no better than level h−1
      }
      tv_merge(W.best + (int64_t)r * W.n + dst, tv_key(c, out, (uint32_t)src, gi));
    }
  }
}

__global__ void __launch_bounds__(kTvThreads) tv_finalize_kernel(TvWork W, int h) {
  __shared__ int32_t changed[kTvMaxGroup];
  if (W.tot[h - 1] == 0) return;
  for (int r = threadIdx.x; r < W.G; r += blockDim.x) changed[r] = 0;
  __syncthreads();
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < W.n) {
    uint64_t mask = 0;
    for (int r = 0; r < W.G; ++r) {
      const int64_t i = (int64_t)r * W.n + t;
      const unsigned __int128 b = W.best[i];
      uint64_t pr = kTvNoPred;
      if (b != 0) {  // every merged candidate beat level h−1
        const uint64_t hi = (uint64_t)(b >> 64);
        W.val[i] = __longlong_as_double((long long)(tv_out(W, r) ? ~hi : hi));
        W.lvl[i] = (uint8_t)h;
        W.best[i] = 0;
        pr = ~(uint64_t)b;
        mask |= 1ull << r;
        atomicAdd_block(changed + r, 1);
      }
      W.pred[((int64_t)r * W.H + (h - 1)) * W.n + t] = pr;
    }
    W.fmask[(size_t)(h & 1) * W.n + t] = mask;
  }
  __syncthreads();
  for (int r = threadIdx.x; r < W.G; r += blockDim.x)
    if (changed[r]) {
      atomicAdd(W.cnt + r * (W.H + 1) + h, changed[r]);
      atomicAdd(W.tot + h, changed[r]);
    }
}

// Row r's walk into token t from level h, in DP order (t first): step w reached tok[w] from nbr[w]
// through the pool of global insertion index gi[w].  Each predecessor is taken at the latest level
// below the step's at which it changed (the level right below: include/cfmm_b200.h).  Returns the
// hop count.
__device__ __forceinline__ int tv_walk_from(const TvWork& W, int r, int64_t t, int h, int32_t* tok, int32_t* nbr,
                                            uint32_t* gi) {
  int n = 0;
  int64_t u = t;
  const uint64_t* pr = W.pred + (int64_t)r * W.H * W.n;
  while (h > 0 && n < kTvMaxHops) {
    const uint64_t key = pr[(int64_t)(h - 1) * W.n + u];
    tok[n] = (int32_t)u;
    nbr[n] = (int32_t)(key >> 32);
    gi[n++] = (uint32_t)key;
    u = (int64_t)(key >> 32);
    --h;
    while (h > 0 && pr[(int64_t)(h - 1) * W.n + u] == kTvNoPred) --h;
  }
  return n;
}

__device__ __forceinline__ bool tv_repeats(const uint32_t* gi, int n) {
  bool rep = false;
  for (int a = 1; a < n; ++a)
    for (int b = 0; b < a; ++b) rep |= gi[a] == gi[b];
  return rep;
}

// The entry (set << kPairSetShift | device position) of every pool at its global insertion index.
__global__ void tv_entry_kernel(const PathSets* __restrict__ P, TvSets S, int64_t* __restrict__ entry) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int k = 0;
  while (k < kPathSets && i >= S.start[k + 1]) ++k;
  if (k == kPathSets) return;
  const int64_t p = i - S.start[k];
  const int64_t g = P->s[k].gidx[p];
  if (g >= 0) entry[g & ~(1ll << 62)] = ((int64_t)k << kPairSetShift) | p;
}

// ---- net of a per-hop cost (cfmm_quote_token_values_net) -------------------------------------------
// The DP with max_hops = L is the first L levels of this one: token t's value, walk and hops at L are
// those of the last level ≤ L it changed at.  So after each level h a token that changed at h is a
// candidate: its level-h walk is checked for repeats, and a filled one's net (value ∓ hops·κ_t) is
// compared with the best kept, the later level winning a tie.
struct TvNet {
  const double* cost;  // [n] κ_t, per hop in units of token t
  double* val;         // [G][n] the selected level's value
  double* net;         // [G][n] its net
  uint8_t* lvl;        // [G][n] the selected level (kTvNever: no level filled yet); null: no selection
};

// value ∓ n·κ: one IEEE multiply, then one add (exact-out) or subtract (exact-in); no fma.
__device__ __forceinline__ double tv_net(double v, int n, double kappa, bool out) {
  const double c = __dmul_rn((double)n, kappa);
  return out ? __dadd_rn(v, c) : __dsub_rn(v, c);
}

// Per (row, token), after tv_finalize_kernel at level h.  Level 1 also starts the selection.
__global__ void tv_select_kernel(TvWork W, TvNet N, int h) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)W.G * W.n) return;
  if (h == 1) N.lvl[i] = kTvNever;
  if (W.tot[h] == 0 || W.lvl[i] != h) return;
  const int r = (int)(i / W.n);
  const int64_t t = i - (int64_t)r * W.n;
  int32_t tok[kTvMaxHops], nbr[kTvMaxHops];
  uint32_t gi[kTvMaxHops];
  const int n = tv_walk_from(W, r, t, h, tok, nbr, gi);
  if (tv_repeats(gi, n)) return;
  const bool out = tv_out(W, r);
  const double v = W.val[i], x = tv_net(v, n, N.cost[t], out);
  if (N.lvl[i] != kTvNever && !(out ? x <= N.net[i] : x >= N.net[i])) return;
  N.val[i] = v;
  N.net[i] = x;
  N.lvl[i] = (uint8_t)h;
}

// ---- the outputs ------------------------------------------------------------------------------------
// A (row, token)'s outputs come from the level selected by tv_select_kernel when there is one (N.lvl
// null: cfmm_quote_token_values, none), else from the last level the token changed at: the DP with
// max_hops = H.

// Per (row, token) of the group: value, hops and status at [r·n + t] of the group's outputs; net
// (NULL: not written) gets the selected net, or the value when none is selected.
__global__ void tv_rebuild_kernel(TvWork W, TvNet N, double* __restrict__ value, uint8_t* __restrict__ hops,
                                  uint8_t* __restrict__ status, double* __restrict__ net) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)W.G * W.n) return;
  const int r = (int)(i / W.n);
  const int64_t t = i - (int64_t)r * W.n;
  const bool sel = N.lvl && N.lvl[i] != kTvNever;
  const uint8_t L = sel ? N.lvl[i] : W.lvl[i];
  value[i] = sel ? N.val[i] : W.val[i];
  if (net) net[i] = sel ? N.net[i] : value[i];
  if (L == kTvNever || L == 0) {
    hops[i] = 0;
    status[i] = L == 0 ? 0 : 2;  // CFMM_ORDER_FILLED (the root), CFMM_ORDER_UNREACHABLE
    return;
  }
  int32_t tok[kTvMaxHops], nbr[kTvMaxHops];
  uint32_t gi[kTvMaxHops];
  const int n = tv_walk_from(W, r, t, L, tok, nbr, gi);
  hops[i] = (uint8_t)n;
  status[i] = tv_repeats(gi, n) ? 4 : 0;  // CFMM_PATH_REPEATS_POOL, CFMM_ORDER_FILLED
}

// Requested (row, token) pairs j with row in the group (row0 .. row0 + G): the walk in path order at
// H·j .. (set, device position, tendered side, delivered token 1-based), priced by path_run.
// Exact-in walks run root → t, exact-out walks t → root.  nhop[j] = 0 for the root, an unreached
// token and a walk that repeats a pool.
__global__ void tv_path_kernel(const PathSets* __restrict__ P, TvWork W, TvNet N, int64_t row0,
                               const int64_t* __restrict__ entry, int64_t n_req, const int64_t* __restrict__ req_row,
                               const int64_t* __restrict__ req_token, int32_t* __restrict__ nhop,
                               uint8_t* __restrict__ hop_set, int64_t* __restrict__ hop_pos,
                               uint8_t* __restrict__ hop_tok1, int64_t* __restrict__ hop_token,
                               double* __restrict__ tender, double* __restrict__ received,
                               uint8_t* __restrict__ status) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_req || req_row[j] < row0 || req_row[j] >= row0 + W.G) return;
  const int r = (int)(req_row[j] - row0);
  const int64_t t = req_token[j] - 1, i = (int64_t)r * W.n + t;
  const uint8_t L = N.lvl && N.lvl[i] != kTvNever ? N.lvl[i] : W.lvl[i];
  nhop[j] = 0;
  if (L == kTvNever || L == 0) {
    status[j] = L == 0 ? 0 : 2;
    return;
  }
  int32_t tok[kTvMaxHops], nbr[kTvMaxHops];
  uint32_t gi[kTvMaxHops];
  const int n = tv_walk_from(W, r, t, L, tok, nbr, gi);
  uint8_t* row_set = hop_set + (int64_t)W.H * j;
  int64_t* row_pos = hop_pos + (int64_t)W.H * j;
  uint8_t* row_tok1 = hop_tok1 + (int64_t)W.H * j;
  if (walk_hops(P, n, [&](int w) { return entry[gi[w]]; }, nbr, tok, tv_out(W, r), row_set, row_pos, row_tok1,
                hop_token + (int64_t)W.H * j)) {
    status[j] = 4;
    return;
  }
  walk_price(P, n, row_set, row_pos, row_tok1, W.kind + r, W.amount + r, tender + (int64_t)W.H * j,
             received + (int64_t)W.H * j, status + j);
  nhop[j] = n;
}

}  // namespace cfmm
