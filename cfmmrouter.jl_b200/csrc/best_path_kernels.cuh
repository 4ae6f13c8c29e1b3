// best_path_kernels.cuh -- the path search of cfmm_find_order_paths (sm_90a, include/cfmm_b200.h).
// Off the sweep path: no sweep kernel reads anything these kernels add.
//
// The intermediate tokens B of a call are dense slots 0 .. nB−1 in token order.  best_path_graph_kernel
// builds, once per call, each slot's neighbours in B from the token adjacency (arb_scan_kernels.cuh).
// best_path_kernel runs one order row per CTA: an exact dynamic programme over "at most h hops" on
// the tokens of B, two levels of amounts and every level's predecessors in shared memory.  Every
// candidate is one quote, path_hop_f / path_hop_exact_out: cfmm_quote_swaps /
// cfmm_quote_swaps_exact_out bit for bit.  The rebuilt walk is priced by path_run, the code of
// cfmm_quote_paths, so its amounts are that call's on the same CSR.  best_path_kernel<true>
// (cfmm_find_order_paths_net) runs the same DP with the final pass after every level and emits the
// max_hops = L result that is best net of a per-hop cost.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "hub_kernels.cuh"

namespace cfmm {

constexpr int kBestPathMaxTokens = 1024;  // CFMM_BEST_PATH_MAX_TOKENS
constexpr int kBestPathThreads = 256;
constexpr int kBestPathMaxHops = 8;       // CFMM_PATH_MAX_HOPS

// The B-subgraph of a call.  Slot s is token tok[s] (0-based, ascending); slot_of[t] is t's slot or
// −1.  Slot s's neighbours in B are nbr[nB·s + m], m < deg[s], ascending, with pair ids pair[nB·s + m].
struct BestPathGraph {
  const int32_t* tok;
  const int32_t* slot_of;
  const int32_t* deg;
  const int16_t* nbr;
  const int32_t* pair;
  int nB;
};

// The position of b in the adjacency list A.nbr[a0 .. a1) (ascending), bisected; a1 when b is absent.
__device__ __forceinline__ int64_t adj_find(AdjView A, int64_t a0, int64_t a1, int32_t b) {
  int64_t lo = a0, hi = a1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (A.nbr[mid] < b)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo < a1 && A.nbr[lo] == b ? lo : a1;
}

// The pair {a, b} from a's adjacency list, −1 when there is none.
__device__ __forceinline__ int32_t adj_pair(AdjView A, int32_t a, int32_t b) {
  const int64_t a0 = A.off[a], a1 = A.off[a + 1], e = adj_find(A, a0, a1, b);
  return e < a1 ? A.pair[e] : -1;
}

// The pair {t, tok[s]} into dst[s] for every slot s that has one, from t's adjacency list: walked when
// it is short, else bisected per slot.  (Graph: BestPathGraph, or subgraph_kernels.cuh's RowGraph.)
template <class Graph>
__device__ __forceinline__ void side_pairs(AdjView A, const Graph& G, int32_t t, int32_t* dst) {
  const int64_t a0 = A.off[t], a1 = A.off[t + 1];
  if (a1 - a0 <= (int64_t)G.nB) {
    for (int64_t e = a0 + threadIdx.x; e < a1; e += blockDim.x) {
      const int32_t u = G.slot_of[A.nbr[e]];
      if (u >= 0) dst[u] = A.pair[e];
    }
  } else {
    for (int s = threadIdx.x; s < G.nB; s += blockDim.x) {
      const int64_t e = adj_find(A, a0, a1, G.tok[s]);
      if (e < a1) dst[s] = A.pair[e];
    }
  }
}

// One warp per slot: its adjacency list filtered to B, compacted in list order with a ballot.
__global__ void best_path_graph_kernel(AdjView A, const int32_t* __restrict__ tok,
                                       const int32_t* __restrict__ slot_of, int nB, int32_t* __restrict__ deg,
                                       int16_t* __restrict__ nbr, int32_t* __restrict__ pair) {
  const int s = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (s >= nB) return;
  const int64_t e0 = A.off[tok[s]], e1 = A.off[tok[s] + 1];
  int n = 0;
  for (int64_t b = e0; b < e1; b += 32) {
    const int64_t e = b + lane;
    const int32_t u = e < e1 ? slot_of[A.nbr[e]] : -1;
    const unsigned in = __ballot_sync(kFull, u >= 0);
    if (u >= 0) {
      const int at = n + __popc(in & ((1u << lane) - 1u));
      nbr[(int64_t)nB * s + at] = (int16_t)u;
      pair[(int64_t)nB * s + at] = A.pair[e];
    }
    n += __popc(in);
  }
  if (lane == 0) deg[s] = n;
}

// A candidate's rank key: score (the amount, negated for exact-out), then fewer hops, then the
// smaller predecessor token, then the earlier position in the pair's pool list.  from is how the
// walk is rebuilt (an edge index, or a slot at the final hop), not part of the order.
struct BpKey {
  double s;
  int32_t hops, tok, pos, from;
};

__device__ __forceinline__ bool bp_before(const BpKey& a, const BpKey& b) {
  if (a.s != b.s) return a.s > b.s;
  if (a.hops != b.hops) return a.hops < b.hops;
  if (a.tok != b.tok) return a.tok < b.tok;
  return a.pos < b.pos;
}

__device__ __forceinline__ BpKey bp_none() { return BpKey{-kPathInf, 0, INT32_MAX, INT32_MAX, -1}; }

__device__ __forceinline__ BpKey bp_warp_best(BpKey k) {
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) {
    BpKey o;
    o.s = __shfl_xor_sync(kFull, k.s, m);
    o.hops = __shfl_xor_sync(kFull, k.hops, m);
    o.tok = __shfl_xor_sync(kFull, k.tok, m);
    o.pos = __shfl_xor_sync(kFull, k.pos, m);
    o.from = __shfl_xor_sync(kFull, k.from, m);
    if (bp_before(o, k)) k = o;
  }
  return k;
}

// The candidates of one hop over the active pools of pair k: from an amount a of the DP's
// predecessor token (exact-in: a tendered, the hop pays out; exact-out: a wanted, the hop's tender
// is the candidate).  tender is the token the hop tenders.  key gets the best, ranked as above.
__device__ __forceinline__ void bp_hop(const PathSets* P, PairIndexView ix, int32_t k, int64_t tender, double a,
                                       bool out, int32_t hops, int32_t tok, int32_t from, BpKey& key) {
  const int64_t e0 = ix.off[k], e1 = ix.off[k + 1];
  for (int64_t e = e0; e < e1; ++e) {
    const HubHop h = hub_hop(P, ix.pool[e], tender);
    if (!h.active) continue;
    double s;
    if (!out) {
      const double v = path_hop_f(P, h.k, h.p, a, h.tok1);
      if (!(v > 0.0)) continue;  // NaN or nothing out
      s = v;
    } else {
      const double x = path_hop_exact_out(P, h.k, h.p, a, h.tok1);
      if (!(x < kPathInf)) continue;  // NaN or unreachable
      s = -x;
    }
    const BpKey c{s, hops, tok, (int32_t)(e - e0), from};
    if (bp_before(c, key)) key = c;
  }
}

// The shared-memory layout of one row: two levels of amounts and hop counts, the start- and
// end-side pairs of every slot, and per level 1 .. H−1 each slot's predecessor (an edge index of
// the slot, kBpFromSource, or kBpCarry: the level before's value kept) and pool position.
constexpr int16_t kBpCarry = -1, kBpFromSource = -2;

__host__ __device__ inline size_t best_path_smem(int nB, int H) {
  const size_t n = (size_t)nB;
  return 2 * n * sizeof(double) + 2 * n * sizeof(int32_t) + (size_t)(H - 1) * n * (sizeof(int32_t) + sizeof(int16_t)) +
         2 * n + 32 * sizeof(BpKey) + 16;
}

// Level 1 of row's DP: one thread per slot, the pools of {S, b}, from the row's amount.  Returns
// whether this thread's slots changed.
__device__ __forceinline__ int bp_first_level(const PathSets* P, PairIndexView ix, const BestPathGraph& G,
                                              const int32_t* spair, int32_t j, int32_t i, int32_t S, bool out,
                                              double amt, double* val, uint8_t* hops, int16_t* pred, int32_t* ppos) {
  const int nB = G.nB;
  int changed = 0;
  for (int s = threadIdx.x; s < nB; s += blockDim.x) {
    const int32_t b = G.tok[s];
    BpKey key = bp_none();
    if (b != j && b != i && spair[s] >= 0) bp_hop(P, ix, spair[s], out ? b : S, amt, out, 1, S, kBpFromSource, key);
    const bool got = key.from != -1;
    if (got) {
      val[nB + s] = out ? -key.s : key.s;
      hops[nB + s] = 1;
    }
    pred[s] = got ? kBpFromSource : kBpCarry;
    ppos[s] = got ? key.pos : 0;
    changed |= got;
  }
  return changed;
}

// Level h ≥ 2: warps own destination slots, lanes scan the incoming pools.  A slot changed at level
// h−1 iff its hop count is h−1; only those can improve a slot at level h (an unchanged predecessor's
// candidates were all candidates of level h−1 already), so the others are skipped.  Returns whether
// this thread's slots changed.
__device__ __forceinline__ int bp_next_level(const PathSets* P, PairIndexView ix, const BestPathGraph& G, int32_t j,
                                             int32_t i, bool out, int h, double* val, uint8_t* hops, int16_t* pred,
                                             int32_t* ppos) {
  const int nB = G.nB, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  const double* vp = val + (size_t)((h - 1) & 1) * nB;
  double* vc = val + (size_t)(h & 1) * nB;
  const uint8_t* hp = hops + (size_t)((h - 1) & 1) * nB;
  uint8_t* hc = hops + (size_t)(h & 1) * nB;
  int changed = 0;
  for (int s = warp; s < nB; s += nwarp) {
    const int32_t b = G.tok[s];
    BpKey key = bp_none();
    if (b != j && b != i) {
      const int32_t d = G.deg[s];
      for (int m = lane; m < d; m += 32) {
        const int u = G.nbr[(int64_t)nB * s + m];
        if (hp[u] != h - 1) continue;
        bp_hop(P, ix, G.pair[(int64_t)nB * s + m], out ? b : G.tok[u], vp[u], out, h, G.tok[u], m, key);
      }
    }
    key = bp_warp_best(key);
    if (lane == 0) {
      const double prev = vp[s];
      const bool better = key.from != -1 && (out ? -key.s < prev : key.s > prev);
      vc[s] = better ? (out ? -key.s : key.s) : prev;
      hc[s] = better ? (uint8_t)h : hp[s];
      pred[(size_t)(h - 1) * nB + s] = better ? (int16_t)key.from : kBpCarry;
      ppos[(size_t)(h - 1) * nB + s] = better ? key.pos : 0;
      changed |= better;
    }
  }
  return changed;
}

// The final hop into T, one thread per slot reached at level top, and S itself (the direct pair,
// pseudo-slot nB): each warp's best into red[warp].  This is the final hop of the DP with
// max_hops = top + 1.
__device__ __forceinline__ void bp_final_pass(const PathSets* P, PairIndexView ix, const BestPathGraph& G,
                                              const int32_t* epair, const int32_t& direct, int32_t j, int32_t i,
                                              int32_t S, bool out, double amt, int top, const double* val,
                                              const uint8_t* hops, BpKey* red) {
  const int nB = G.nB, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* vt = val + (size_t)(top & 1) * nB;
  const uint8_t* ht = hops + (size_t)(top & 1) * nB;
  BpKey key = bp_none();
  for (int s = threadIdx.x; s <= nB; s += blockDim.x) {
    if (s == nB) {
      if (direct >= 0) bp_hop(P, ix, direct, j, amt, out, 1, S, nB, key);
    } else {
      const int32_t b = G.tok[s];
      if (b == j || b == i || epair[s] < 0 || !(out ? vt[s] < kPathInf : vt[s] > 0.0)) continue;
      bp_hop(P, ix, epair[s], out ? j : b, vt[s], out, ht[s] + 1, b, s, key);
    }
  }
  key = bp_warp_best(key);
  if (lane == 0) red[warp] = key;
}

__device__ __forceinline__ BpKey bp_cta_best(const BpKey* red, int nwarp) {
  BpKey best = red[0];
  for (int w = 1; w < nwarp; ++w)
    if (bp_before(red[w], best)) best = red[w];
  return best;
}

// A walk of n steps in DP order, step w through the pool entry(w) (set << kPairSetShift | device
// position) from token from[w] to token to[w], written in path order to one row's hop slots: set,
// device position, tendered side, delivered token 1-based.  An exact-in DP runs back from the sink
// (path hop g is step n−1−g, which tenders from and delivers to); an exact-out DP runs forward from
// the token delivered last (path hop g is step g, which tenders to and delivers from).  Returns
// whether the walk uses a pool twice.  (Also token_value_kernels.cuh's requested walks.)
template <class Entry>
__device__ __forceinline__ bool walk_hops(const PathSets* P, int n, Entry entry, const int32_t* from,
                                          const int32_t* to, bool out, uint8_t* row_set, int64_t* row_pos,
                                          uint8_t* row_tok1, int64_t* row_token) {
  bool repeats = false;
  for (int g = 0; g < n; ++g) {
    const int w = out ? g : n - 1 - g;
    const int32_t a = out ? to[w] : from[w], c = out ? from[w] : to[w];
    const HubHop hh = hub_hop(P, entry(w), a);
    row_set[g] = (uint8_t)hh.k;
    row_pos[g] = hh.p;
    row_tok1[g] = hh.tok1;
    row_token[g] = c + 1;
    for (int f = 0; f < g; ++f) repeats |= row_set[f] == row_set[g] && row_pos[f] == row_pos[g];
  }
  return repeats;
}

// The n hops of one row's slots priced by path_run (cfmm_quote_paths' code, as a one-path CSR):
// each hop's tender and received, and the walk's status into *st.
__device__ __forceinline__ void walk_price(const PathSets* P, int n, const uint8_t* row_set, const int64_t* row_pos,
                                           const uint8_t* row_tok1, const uint8_t* kind, const double* amount,
                                           double* tender, double* received, uint8_t* st) {
  const int64_t off[2] = {0, n};
  path_run<false>(P, 0, off, row_set, row_pos, row_tok1, kind, amount, nullptr, tender, received, st);
}

// The walk of the final-hop winner best after level top, rebuilt from the predecessors in DP order
// and written to the row's hop slots by walk_hops.  Returns the hop count; repeats: whether the walk
// uses a pool twice.
__device__ __forceinline__ int bp_walk(const PathSets* P, PairIndexView ix, const BestPathGraph& G,
                                       const int32_t* spair, const int32_t* epair, const int32_t& direct,
                                       const int16_t* pred, const int32_t* ppos, int32_t S, int32_t T, bool out,
                                       int top, const BpKey& best, uint8_t* row_set, int64_t* row_pos,
                                       uint8_t* row_tok1, int64_t* row_token, bool& repeats) {
  const int nB = G.nB;
  // rebuild the walk in DP order: (pair, position, DP-predecessor token, DP-successor token)
  int32_t wk[kBestPathMaxHops], wpos[kBestPathMaxHops], wfrom[kBestPathMaxHops], wto[kBestPathMaxHops];
  int n = 0;
  int s = best.from;
  wk[n] = s == nB ? direct : epair[s];
  wpos[n] = best.pos;
  wfrom[n] = s == nB ? S : G.tok[s];
  wto[n++] = T;
  for (int h = top; s != nB && h >= 1; --h) {
    const int16_t pr = pred[(size_t)(h - 1) * nB + s];
    if (pr == kBpCarry) continue;
    const int ps = ppos[(size_t)(h - 1) * nB + s];
    if (pr == kBpFromSource) {
      wk[n] = spair[s];
      wpos[n] = ps;
      wfrom[n] = S;
      wto[n++] = G.tok[s];
      break;
    }
    const int u = G.nbr[(int64_t)nB * s + pr];
    wk[n] = G.pair[(int64_t)nB * s + pr];
    wpos[n] = ps;
    wfrom[n] = G.tok[u];
    wto[n++] = G.tok[s];
    s = u;
  }
  repeats = walk_hops(P, n, [&](int w) { return ix.pool[ix.off[wk[w]] + wpos[w]]; }, wfrom, wto, out, row_set,
                      row_pos, row_tok1, row_token);
  return n;
}

// Row r's outputs for the final-hop winner best after level top: no path, a walk that repeats a
// pool, or the walk priced by walk_price.
__device__ __forceinline__ void bp_emit(const PathSets* P, PairIndexView ix, const BestPathGraph& G,
                                        const int32_t* spair, const int32_t* epair, const int32_t& direct,
                                        const int16_t* pred, const int32_t* ppos, int32_t S, int32_t T, bool out,
                                        int top, const BpKey& best, int64_t r, int H, const uint8_t* kind,
                                        const double* amount, int32_t* nhop, uint8_t* hop_set, int64_t* hop_pos,
                                        uint8_t* hop_tok1, int64_t* hop_token, double* tender, double* received,
                                        double* value, uint8_t* status) {
  int64_t* row_pos = hop_pos + (int64_t)H * r;
  uint8_t* row_set = hop_set + (int64_t)H * r;
  uint8_t* row_tok1 = hop_tok1 + (int64_t)H * r;
  if (best.from < 0) {
    nhop[r] = 0;
    value[r] = 0.0;
    status[r] = 2;  // CFMM_ORDER_UNREACHABLE
    return;
  }
  bool repeats;
  const int n = bp_walk(P, ix, G, spair, epair, direct, pred, ppos, S, T, out, top, best, row_set, row_pos, row_tok1,
                        hop_token + (int64_t)H * r, repeats);
  if (repeats) {
    nhop[r] = 0;
    value[r] = 0.0;
    status[r] = 4;  // CFMM_PATH_REPEATS_POOL
    return;
  }
  uint8_t st;
  walk_price(P, n, row_set, row_pos, row_tok1, kind + r, amount + r, tender + (int64_t)H * r, received + (int64_t)H * r,
             &st);
  nhop[r] = n;
  value[r] = out ? tender[(int64_t)H * r] : received[(int64_t)H * r + n - 1];
  status[r] = st;
}

// Row r (include/cfmm_b200.h).  The DP runs from the source S (exact-in: j forward; exact-out: i
// backward) to the sink T.  Outputs: nhop[r], and at H·r .. the hops' set, device position, tendered
// side, delivered token (1-based), tender and received; value[r], status[r].
// kNet = false (cfmm_find_order_paths): the final pass after the last level computed, whose winner is
// emitted.  hop_cost and net are not read.
// kNet = true (cfmm_find_order_paths_net): the final pass after every level, so the CTA's best final
// hop of the DP with max_hops = L is kept at lk[L − 1] for L = 1 .. top + 1 (a level that changed
// nothing ends the DP: the levels and final passes after it repeat it).  Thread 0 then rebuilds each
// L's walk, checks it for repeats, and emits the filled L whose value net of hop_cost[r] per hop is
// best (the larger L on a tie); none filled: the max_hops = H outputs.  net[r] (NULL: not written) is
// the emitted net, or the value.
template <bool kNet>
__global__ void __launch_bounds__(kBestPathThreads)
    best_path_kernel(const PathSets* __restrict__ P, PairIndexView ix, AdjView A, BestPathGraph G,
                     const int64_t* __restrict__ token_in, const int64_t* __restrict__ token_out,
                     const uint8_t* __restrict__ kind, const double* __restrict__ amount, int H,
                     int32_t* __restrict__ nhop, uint8_t* __restrict__ hop_set, int64_t* __restrict__ hop_pos,
                     uint8_t* __restrict__ hop_tok1, int64_t* __restrict__ hop_token, double* __restrict__ tender,
                     double* __restrict__ received, double* __restrict__ value, uint8_t* __restrict__ status,
                     const double* __restrict__ hop_cost, double* __restrict__ net) {
  extern __shared__ __align__(16) unsigned char bp_smem[];
  const int64_t r = blockIdx.x;
  const int nB = G.nB, tid = threadIdx.x, nwarp = blockDim.x >> 5;
  const int32_t j = (int32_t)(token_in[r] - 1), i = (int32_t)(token_out[r] - 1);
  const bool out = kind[r] != 0;
  const double amt = amount[r];
  const int32_t S = out ? i : j, T = out ? j : i;
  const double none = out ? kPathInf : 0.0;
  double* val = reinterpret_cast<double*>(bp_smem);                  // [2][nB]
  int32_t* spair = reinterpret_cast<int32_t*>(val + 2 * nB);        // [nB] pair {S, b}
  int32_t* epair = spair + nB;                                       // [nB] pair {b, T}
  int32_t* ppos = epair + nB;                                        // [H−1][nB]
  int16_t* pred = reinterpret_cast<int16_t*>(ppos + (size_t)(H - 1) * nB);  // [H−1][nB]
  uint8_t* hops = reinterpret_cast<uint8_t*>(pred + (size_t)(H - 1) * nB);  // [2][nB]
  BpKey* red = reinterpret_cast<BpKey*>(
      (reinterpret_cast<uintptr_t>(hops + 2 * nB) + 15) & ~(uintptr_t)15);  // [nwarp]
  __shared__ int32_t direct;  // pair {S, T}, −1 when no pool holds it
  __shared__ BpKey lk[kBestPathMaxHops];
  if (!(amt > 0.0)) {  // nothing to route: filled, no hops (uniform across the CTA)
    if (tid == 0) {
      nhop[r] = 0;
      value[r] = 0.0;
      status[r] = 0;  // CFMM_ORDER_FILLED
      if (kNet && net) net[r] = 0.0;
    }
    return;
  }
  for (int s = tid; s < nB; s += blockDim.x) {
    val[s] = val[nB + s] = none;
    hops[s] = hops[nB + s] = 0;
    spair[s] = epair[s] = -1;
  }
  if (tid == 0) direct = -1;
  __syncthreads();
  // the pairs {S, b} and {b, T}
  for (int side = 0; side < 2; ++side) side_pairs(A, G, side ? T : S, side ? epair : spair);
  if (tid == 0) {
    const int64_t a1 = A.off[S + 1], e = adj_find(A, A.off[S], a1, T);
    if (e < a1) direct = A.pair[e];
  }
  __syncthreads();
  // kNet: the final pass after level top, the best of the DP with max_hops = top + 1, into lk[top].
  // red is free again once thread 0 has read it: the next writes follow the next level's barrier.
  const auto keep = [&](int top) {
    bp_final_pass(P, ix, G, epair, direct, j, i, S, out, amt, top, val, hops, red);
    __syncthreads();
    if (tid == 0) lk[top] = bp_cta_best(red, nwarp);
  };
  if (kNet) keep(0);
  int top = 0;  // the last level computed; the levels above it only carry
  bool more = false;
  if (H > 1) {
    const int changed = bp_first_level(P, ix, G, spair, j, i, S, out, amt, val, hops, pred, ppos);
    top = 1;
    more = __syncthreads_or(changed);
    if (kNet) keep(1);
  }
  for (int h = 2; more && h < H; ++h) {
    const int changed = bp_next_level(P, ix, G, j, i, out, h, val, hops, pred, ppos);
    top = h;
    more = __syncthreads_or(changed);
    if (kNet) keep(h);
  }
  if (!kNet) {
    bp_final_pass(P, ix, G, epair, direct, j, i, S, out, amt, top, val, hops, red);
    __syncthreads();
    if (tid == 0)
      bp_emit(P, ix, G, spair, epair, direct, pred, ppos, S, T, out, top, bp_cta_best(red, nwarp), r, H, kind, amount,
              nhop, hop_set, hop_pos, hop_tok1, hop_token, tender, received, value, status);
    return;
  }
  if (tid != 0) return;
  // each L's walk, rebuilt into the row's hop slots for the repeat check, and a filled L's net: one
  // IEEE multiply, then one add or subtract (no fma)
  const double kappa = hop_cost[r];
  int sel = 0;
  double best_net = 0.0;
  for (int L = 1; L <= top + 1; ++L) {
    const BpKey& c = lk[L - 1];
    if (c.from < 0) continue;
    bool repeats;
    const int n = bp_walk(P, ix, G, spair, epair, direct, pred, ppos, S, T, out, L - 1, c, hop_set + (int64_t)H * r,
                          hop_pos + (int64_t)H * r, hop_tok1 + (int64_t)H * r, hop_token + (int64_t)H * r, repeats);
    if (repeats) continue;
    const double cost = __dmul_rn((double)n, kappa);
    const double x = out ? __dadd_rn(-c.s, cost) : __dsub_rn(c.s, cost);
    if (sel == 0 || (out ? x <= best_net : x >= best_net)) {
      sel = L;
      best_net = x;
    }
  }
  const int L = sel ? sel : top + 1;  // none filled: the max_hops = H outputs as they are
  bp_emit(P, ix, G, spair, epair, direct, pred, ppos, S, T, out, L - 1, lk[L - 1], r, H, kind, amount, nhop, hop_set,
          hop_pos, hop_tok1, hop_token, tender, received, value, status);
  if (net) net[r] = sel ? best_net : value[r];
}

}  // namespace cfmm
