// pool_layout.hpp -- host-side device layout of one pool type (pure C++, no CUDA:
// unit-tested on CPU through cfmm_debug_product_layout).
//
//  * orientation: ProductTwoCoin is exactly symmetric under exchanging its two
//    tokens, so when hub tokens are detected every pool is stored with its
//    higher-degree token first (hubs on the register-accumulated run side);
//  * order: stable counting sort by the (oriented) first token a; for the TMA
//    kernel additionally grouped by bucket(b) = b / nb, each bucket padded to
//    whole tiles (padding = position with order -1), one bucket id per tile.
#pragma once
#include <cstdint>
#include <memory>
#include <utility>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace cfmm {

// Host vectors of the layout: default-initialised on resize (no serial zero-fill -- and no serial
// page-fault pass -- over arrays every element of which a parallel loop is about to write).
template <class T>
struct DefaultInitAlloc : std::allocator<T> {
  template <class U>
  struct rebind {
    using other = DefaultInitAlloc<U>;
  };
  using std::allocator<T>::allocator;
  template <class U>
  void construct(U* p) noexcept {
    ::new (static_cast<void*>(p)) U;
  }
  template <class U, class... Args>
  void construct(U* p, Args&&... args) {
    ::new (static_cast<void*>(p)) U(std::forward<Args>(args)...);
  }
};
template <class T>
using HVec = std::vector<T, DefaultInitAlloc<T>>;

inline int layout_threads(int64_t m) {
#ifdef _OPENMP
  return m < (1 << 16) ? 1 : omp_get_max_threads();
#else
  (void)m;
  return 1;
#endif
}

// Stable counting sort of `m` items by key(item) in [0, K): out[pos] = item, items taken from `src`
// (the current order; null = identity).  Every thread counts and then scatters its own contiguous
// block with per-(thread, key) offsets -- stable, no atomics; the offsets come from a key-blocked
// parallel scan (thread-major counters, so each block is read row by row).  `totals` (optional):
// the K key counts.
template <class KeyFn>
inline void counting_sort_stable(const int64_t* src, int64_t m, int64_t K, KeyFn key, int64_t* out,
                                 std::vector<int64_t>* totals = nullptr) {
  int T = layout_threads(m);
  // the counters must stay small next to the items: each thread sweeps K of them twice
  while (T > 1 && (int64_t)T * K > 4 * m) T /= 2;
  HVec<int64_t> cnt((size_t)T * (size_t)K);
  std::vector<int64_t> base((size_t)K + 1, 0);
#pragma omp parallel num_threads(T)
  {
#ifdef _OPENMP
    const int t = omp_get_thread_num();
#else
    const int t = 0;
#endif
    const int64_t lo = m * t / T, hi = m * (t + 1) / T;
    int64_t* c = cnt.data() + (size_t)t * (size_t)K;
    for (int64_t k = 0; k < K; ++k) c[k] = 0;
    for (int64_t p = lo; p < hi; ++p) c[key(src ? src[p] : p)]++;
#pragma omp barrier
    const int64_t k0 = K * t / T, k1 = K * (t + 1) / T;  // this thread's block of keys
    for (int64_t k = k0; k < k1; ++k) base[(size_t)k + 1] = 0;
    for (int tt = 0; tt < T; ++tt) {
      const int64_t* row = cnt.data() + (size_t)tt * (size_t)K;
      for (int64_t k = k0; k < k1; ++k) base[(size_t)k + 1] += row[k];
    }
#pragma omp barrier
#pragma omp single
    {
      for (int64_t k = 0; k < K; ++k) base[(size_t)k + 1] += base[(size_t)k];  // exclusive starts
    }
    // (implicit barrier) offsets in (key, thread) order, key block by key block
    {
      std::vector<int64_t> run(base.begin() + k0, base.begin() + k1);
      for (int tt = 0; tt < T; ++tt) {
        int64_t* row = cnt.data() + (size_t)tt * (size_t)K;
        for (int64_t k = k0; k < k1; ++k) {
          const int64_t v = row[k];
          row[k] = run[(size_t)(k - k0)];
          run[(size_t)(k - k0)] += v;
        }
      }
    }
#pragma omp barrier
    for (int64_t p = lo; p < hi; ++p) {
      const int64_t item = src ? src[p] : p;
      out[c[key(item)]++] = item;
    }
  }
  if (totals) {
    totals->resize((size_t)K);
    for (int64_t k = 0; k < K; ++k) (*totals)[(size_t)k] = base[(size_t)k + 1] - base[(size_t)k];
  }
}

// Serial form over a small block (one b-bucket): counters are 32-bit and caller-provided.
template <class KeyFn>
inline void counting_sort_block(const int64_t* src, int64_t m, int64_t K, KeyFn key, int64_t* out,
                                std::vector<int32_t>& cnt) {
  cnt.assign((size_t)K + 1, 0);
  for (int64_t p = 0; p < m; ++p) cnt[(size_t)key(src[p]) + 1]++;
  for (int64_t k = 0; k < K; ++k) cnt[(size_t)k + 1] += cnt[(size_t)k];
  for (int64_t p = 0; p < m; ++p) out[cnt[(size_t)key(src[p])]++] = src[p];
}

struct TileShape {
  int64_t tile = 0;   // padding unit in pools (one warp-chunk of the TMA kernel); 0 = no bucketing
  int64_t nbmax = 0;  // capacity of the shared ν / Ψ slices, in tokens
  int64_t nb_align = 1;  // bucket width is a multiple of this
};

struct PoolLayout {
  HVec<int64_t> order;           // device position -> insertion index within the type, -1 = padding
  HVec<int> oa, ob;              // device orientation per insertion index (0-based tokens)
  HVec<uint8_t> swapped;         // per insertion index: stored with its two tokens exchanged
  std::vector<int> tile_bucket;  // bucket of every chunk (bucketed layouts only)
  int64_t m_padded = 0;
  int64_t nb = 0;                // bucket width in tokens
  bool bucketed = false;
  bool skewed = false;           // hub tokens detected
  bool used_skew_shape = false;
};

// Token degrees (pools per token), by per-thread histograms merged key block by key block: no
// atomics, so a hub token costs what any other token does.
inline std::vector<int64_t> token_degrees(const int64_t* Ai, int64_t m, int64_t n_tokens) {
  int T = layout_threads(m);
  while (T > 1 && (int64_t)T * n_tokens > 4 * m) T /= 2;
  HVec<int32_t> part((size_t)T * (size_t)n_tokens);
  std::vector<int64_t> deg((size_t)n_tokens, 0);
#pragma omp parallel num_threads(T)
  {
#ifdef _OPENMP
    const int t = omp_get_thread_num();
#else
    const int t = 0;
#endif
    int32_t* c = part.data() + (size_t)t * (size_t)n_tokens;
    for (int64_t k = 0; k < n_tokens; ++k) c[k] = 0;
    for (int64_t i = m * t / T; i < m * (t + 1) / T; ++i) {
      c[Ai[2 * i] - 1]++;
      c[Ai[2 * i + 1] - 1]++;
    }
#pragma omp barrier
    for (int tt = 0; tt < T; ++tt) {
      const int32_t* row = part.data() + (size_t)tt * (size_t)n_tokens;
      for (int64_t k = n_tokens * t / T; k < n_tokens * (t + 1) / T; ++k) deg[(size_t)k] += row[k];
    }
  }
  return deg;
}

// Ai: [2m] 1-based token ids (validated by the caller).  orient: -1 auto (orient
// only when hubs are detected), 0 never, 1 always; only honoured when `symmetric`
// (ProductTwoCoin).  `normal` / `skew`: tile shapes for uniform / hub-detected graphs.
// `mark` (optional): called after each phase with its name (finalize timing).
inline PoolLayout build_pool_layout(const int64_t* Ai, int64_t m, int64_t n_tokens, int orient,
                                    bool symmetric, TileShape normal, TileShape skew,
                                    void (*mark)(const char*) = nullptr) {
  PoolLayout lay;
  lay.oa.resize((size_t)m);
  lay.ob.resize((size_t)m);
  lay.swapped.resize((size_t)m);
  lay.m_padded = m;
  std::vector<int64_t> deg;
  if (symmetric && orient != 0) {
    deg = token_degrees(Ai, m, n_tokens);
    // hub detection: some token sits in far more pools than the average token.
    // On uniform graphs orientation only perturbs the layout (it was slightly slower),
    // so in auto mode it is applied to skewed graphs only.
    int64_t max_deg = 0;
    for (int64_t d : deg) max_deg = d > max_deg ? d : max_deg;
    const double mean_deg = 2.0 * (double)m / (double)n_tokens;
    lay.skewed = (double)max_deg > 4.0 * mean_deg + 64.0;
    if (orient < 0 && !lay.skewed) deg.clear();
  }
#pragma omp parallel for schedule(static) if (m > (1 << 16))
  for (int64_t i = 0; i < m; ++i) {
    const int a = (int)(Ai[2 * i] - 1), b = (int)(Ai[2 * i + 1] - 1);
    const bool sw = !deg.empty() && deg[(size_t)b] > deg[(size_t)a];
    lay.swapped[(size_t)i] = sw;
    lay.oa[(size_t)i] = sw ? b : a;
    lay.ob[(size_t)i] = sw ? a : b;
  }
  if (mark) mark("layout: degrees, orientation");
  lay.used_skew_shape = lay.skewed && skew.tile > 0;
  const TileShape shape = lay.used_skew_shape ? skew : normal;
  const auto by_a = [&](int64_t i) { return (int64_t)lay.oa[(size_t)i]; };
  const auto sort_by_a_only = [&]() {
    lay.order.resize((size_t)m);
    counting_sort_stable(nullptr, m, n_tokens, by_a, lay.order.data());
    if (mark) mark("layout: sort by first token");
  };
  if (shape.tile <= 0 || m == 0) {
    sort_by_a_only();
    return lay;
  }
  // b-bucketed order (bucket(b), a, insertion index), each bucket padded to whole tiles: group
  // by bucket first (few keys), then sort every bucket by a on its own
  const int64_t tile = shape.tile;
  const int64_t B = (n_tokens + shape.nbmax - 1) / shape.nbmax;
  int64_t nb = (n_tokens + B - 1) / B;
  if (shape.nb_align > 1) {  // round up; stays within the slice capacity when nbmax is a multiple too
    const int64_t up = (nb + shape.nb_align - 1) / shape.nb_align * shape.nb_align;
    if (up <= shape.nbmax) nb = up;
  }
  HVec<int64_t> grouped((size_t)m);
  std::vector<int64_t> cnt;
  counting_sort_stable(nullptr, m, B, [&](int64_t i) { return (int64_t)(lay.ob[(size_t)i] / nb); },
                       grouped.data(), &cnt);
  if (mark) mark("layout: group by bucket");
  std::vector<int64_t> start((size_t)B + 1, 0), first((size_t)B + 1, 0);  // padded / unpadded starts
  for (int64_t k = 0; k < B; ++k) {
    start[(size_t)k + 1] = start[(size_t)k] + (cnt[(size_t)k] + tile - 1) / tile * tile;
    first[(size_t)k + 1] = first[(size_t)k] + cnt[(size_t)k];
  }
  const int64_t padded = start[(size_t)B];
  if (padded > 2 * m + 8 * tile) {  // too sparse per bucket: a-sorted layout only
    sort_by_a_only();
    return lay;
  }
  lay.order.resize((size_t)padded);
  const int T = layout_threads(m);
  if (B >= 4 || T == 1) {
#pragma omp parallel num_threads(T)
    {
      std::vector<int32_t> c;
#pragma omp for schedule(dynamic, 1)
      for (int64_t k = 0; k < B; ++k) {
        int64_t* out = lay.order.data() + start[(size_t)k];
        counting_sort_block(grouped.data() + first[(size_t)k], cnt[(size_t)k], n_tokens, by_a, out, c);
        for (int64_t q = cnt[(size_t)k]; q < start[(size_t)k + 1] - start[(size_t)k]; ++q) out[q] = -1;
      }
    }
  } else {
    for (int64_t k = 0; k < B; ++k) {
      int64_t* out = lay.order.data() + start[(size_t)k];
      counting_sort_stable(grouped.data() + first[(size_t)k], cnt[(size_t)k], n_tokens, by_a, out);
      for (int64_t q = cnt[(size_t)k]; q < start[(size_t)k + 1] - start[(size_t)k]; ++q) out[q] = -1;
    }
  }
  if (mark) mark("layout: sort buckets by first token");
  lay.m_padded = padded;
  lay.nb = nb;
  lay.bucketed = true;
  lay.tile_bucket.resize((size_t)(padded / tile));
  for (int64_t k = 0; k < B; ++k)
    for (int64_t t = start[(size_t)k] / tile; t < start[(size_t)k + 1] / tile; ++t)
      lay.tile_bucket[(size_t)t] = (int)k;
  return lay;
}

}  // namespace cfmm
