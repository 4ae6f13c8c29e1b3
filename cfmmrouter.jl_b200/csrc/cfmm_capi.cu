// cfmm_capi.cu -- libcfmm_b200.so: C ABI (include/cfmm_b200.h) over the sm_90a
// sweep kernels.  Host side of the drop-in boundary: pool ingest, token sort,
// SoA upload, sweep orchestration, trade read-back, multi-GPU exchange set-up.
//
// There is deliberately no CPU fallback in this file: every compute entry
// point needs a CUDA device and fails with CFMM_ERR_CUDA otherwise.
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <new>
#include <numeric>
#include <optional>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/cfmm_b200.h"
#include "peer_exchange.cuh"
#include "pool_layout.hpp"
#include "sweep_kernels.cuh"
#include "product_tma.cuh"
#include "solver.cuh"
#include "solver_control.cuh"
#include "subgraph_kernels.cuh"
#include "basket_kernels.cuh"
#include "price_arb_kernels.cuh"
#include "swap_kernels.cuh"
#include "path_kernels.cuh"
#include "split_kernels.cuh"
#include "route_kernels.cuh"
#include "arb_scan_kernels.cuh"
#include "hub_kernels.cuh"
#include "best_path_kernels.cuh"
#include "token_value_kernels.cuh"
#include "univ3_state.cuh"

#include <cub/cub.cuh>

namespace {

thread_local std::string g_create_error;

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;  // owns its allocation: freed on every exit path
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) {
    o.p = nullptr;
    o.n = 0;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    std::swap(p, o.p);
    std::swap(n, o.n);
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t alloc(size_t count) {
    release();
    if (count == 0) return cudaSuccess;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
  // alloc + copy_in of count host elements; a null h or count == 0 leaves the buffer empty (an
  // optional argument not given)
  cudaError_t upload(const T* h, size_t count) {
    cudaError_t e = alloc(h ? count : 0);
    if (e != cudaSuccess || !h || count == 0) return e;
    return copy_in(p, h, count * sizeof(T));
  }
  cudaError_t upload(const std::vector<T>& h) { return upload(h.data(), h.size()); }
  // H2D from pageable memory, COMPLETE on return.  cudaMemcpy alone is not: for pageable sources
  // it returns once the data sits in the driver's staging buffer, the DMA may still be in flight --
  // and the contexts' streams are non-blocking, so a kernel launched on them right afterwards does
  // not wait for the legacy stream the copy ran on (seen as a rare illegal address in
  // update_reserves_kernel reading a position array that had not landed yet).
  static cudaError_t copy_in(void* dst, const void* src, size_t bytes) {
    cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
    return e == cudaSuccess ? cudaStreamSynchronize(cudaStreamLegacy) : e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
};

// One pool type's shard: host staging until finalize, device SoA afterwards.  Each type has a
// main set (laid out at cfmm_finalize / cfmm_compact) and a tail set (the pools appended since,
// cfmm_append_*: a-sorted layout, first-generation kernel).  A set is movable (std::swap), so a
// new layout is built beside the live one and swapped in.
struct PoolSet {
  int64_t m = 0;
  // host staging (insertion order)
  std::vector<double> R, gamma, w;        // 2m, m, 2m
  std::vector<int64_t> Ai;                // 2m, 1-based, validated
  std::vector<int64_t> gidx;              // m, global insertion index
  std::vector<double> cp;                 // univ3: m
  std::vector<int64_t> tick_off;          // univ3: m+1
  std::vector<double> lower, liq;         // univ3: CSR
  // after finalize
  cfmm::HVec<int64_t> order;              // sorted position -> insertion index within type
  std::vector<int64_t> pos_of;            // lazily: insertion index -> sorted position
  DevBuf<double2> d_R, d_w, d_outD, d_outL;
  DevBuf<double> d_gam, d_tickdata;
  DevBuf<double2> d_first[4];             // univ3: the current tick of every pool, four streams (arb_math.cuh)
  DevBuf<int2> d_Ai, d_tick;
  DevBuf<int64_t> d_gidx;                 // sorted position -> global insertion index
  DevBuf<double> d_lower, d_liq;          // univ3: raw tick data, CSR in device order (univ3_state.cuh)
  std::vector<double> first_lower;        // univ3: T₁ = lower_ticks[1] per pool (insertion order)
  std::vector<int64_t> n_ticks;           // univ3: tick count per pool (insertion order)
  int64_t total_ticks = 0;
  int64_t m_padded = 0;        // product: arrays padded to whole 96-pool chunks, per b-bucket
  bool in_fast_range = false;  // every R, γ in [2^-100, 2^100] and γ <= 1
  bool tma_ok = false;         // b-bucketed layout built (product only)
  int nb = 0;                  // bucket width in tokens
  int64_t n_chunks = 0;        // product: 96-pool chunks of the padded device order
  cfmm::BucketTable buckets;   // product: first chunk of every b-bucket (travels as a kernel parameter)
  // derived data of the TMA gradient kernel (product_tma.cuh): the chunk-blocked packed
  // stream (built lazily for the mode a sweep asks for) and the per-token 2^-s_b table of
  // the fixed-point Ψ[b] slice
  DevBuf<unsigned char> d_packed;
  int packed_mode = -1;        // -1 = stale; else (econ ? 1 : 0) | (fixed ? 2 : 0) | (compact ? 4 : 0)
  // compact stream: γ dictionary (<= 256 distinct fees) and the per-pool codes (device order);
  // compact_ok also needs every chunk's first tokens to span less than 2^13
  DevBuf<unsigned short> d_gcode;
  DevBuf<double> d_gtab;       // [256] 1/γ by code, then [256] γ by code
  bool compact_ok = false;
  // the 192-pool compact records pair consecutive chunks of one bucket: their count, the first
  // record of every bucket, and per chunk its record << 2 | (second of its record) << 1 | (alone in
  // its record: the last chunk of a bucket with an odd chunk count)
  int64_t n_recs = 0;
  cfmm::BucketTable rec_buckets;
  DevBuf<int> d_chunk_rec;
  // ... which take the 18-byte pool record when every record's lanes, lane offsets and fees fit its
  // fields (else the set runs the 96-pool records), with the records' 64-byte headers
  bool rec18_ok = false;
  DevBuf<unsigned> d_rec_hdr;
  int range_pools = 0;         // pools per unit of the range table (96-pool chunks or 192-pool records)
  int l2_keep = 0;             // keep rule the last TMA launch ran with (> 0: d_packed holds evict_last lines)
  DevBuf<double> d_inv_scale, d_tok_sum;
  bool fixed_ok = false;       // every token fits the fixed-point rules (range, totals)
  // speed-weighted CTA ranges of the TMA kernel (product_tma.cuh): the table passed to the next
  // launch, the smoothed per-CTA speed it was derived from, and the mapped pinned words the CTAs
  // report their loop durations to (tagged with the table version they ran under)
  cfmm::RangeTable ranges;
  std::vector<double> speed;
  DevBuf<unsigned> d_dur;      // per-CTA loop durations of the latest launch (device)
  unsigned* h_dur = nullptr;   // pinned landing zone of the occasional D2H copy of d_dur
  cudaEvent_t ev_dur = nullptr;
  bool dur_pending = false;    // a copy is in flight (ev_dur)
  bool balancing = false;      // the last TMA launch ran with speed feedback on
  int since_copy = 0;
  unsigned range_version = 1;
  int range_updates = 0;
  int64_t tma_launches = 0;
  cfmm::HVec<uint8_t> swapped;  // product: pool stored with its two tokens exchanged (insertion index)
  bool skewed = false;          // product: hub tokens detected at finalize
  // retired pools (cfmm_set_active): the host flags (insertion order; empty = none retired), the
  // device-order mask the off-path kernels read (1 = active; allocated on the first retire) and,
  // for the two-coin types, the parked reserves of the retired pools (R itself holds (0, 0))
  std::vector<uint8_t> retired;
  DevBuf<uint8_t> d_active;
  DevBuf<double2> d_park;
  void release() {
    d_R.release(); d_w.release(); d_outD.release(); d_outL.release();
    d_gam.release(); d_tickdata.release();
    for (auto& f : d_first) f.release();
    d_Ai.release(); d_tick.release(); d_gidx.release();
    d_lower.release(); d_liq.release();
    d_packed.release(); d_inv_scale.release(); d_tok_sum.release(); d_gcode.release(); d_gtab.release();
    d_chunk_rec.release(); d_rec_hdr.release();
    d_active.release(); d_park.release();
    if (h_dur) cudaFreeHost(h_dur);
    h_dur = nullptr;
    if (ev_dur) cudaEventDestroy(ev_dur);
    ev_dur = nullptr;
    d_dur.release();
  }
};

}  // namespace

struct cfmm_ctx {
  int device = 0;
  int64_t n_tokens = 0;
  int64_t n_pools = 0;
  bool finalized = false;
  bool has_trades = false;
  PoolSet sets[3];
  PoolSet tails[3];  // pools appended after finalize (cfmm_append_*), folded into sets by cfmm_compact
  cudaStream_t stream = nullptr;
  cudaStream_t last_stream = nullptr;  // stream of the last sweep (cfmm_sweep_device* may use the caller's)
  cudaEvent_t ev_order = nullptr;      // orders work across a change of stream
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  DevBuf<double> d_nu;  // n
  DevBuf<double> d_nu_mat;  // n, UniV3 sets only: ν of the last materialising sweep (cfmm_apply_trades)
  double* h_stage = nullptr;   // pinned, n+1
  // finalize uploads: device-order arrays are gathered block by block into two pinned bounce
  // buffers and copied from there (DMA at link rate, overlapped with the next block's gather)
  void* h_bounce[2] = {nullptr, nullptr};
  cudaEvent_t ev_bounce[2] = {nullptr, nullptr};
  int sm_count = 132;  // (H100 SXM; cfmm_create reads the device's own count)
  int64_t l2_bytes = 50 << 20;  // (H100; cfmm_create reads the device's own size)
  // options
  int exact = 0;
  int debug_skip = 0;  // measurement only (tools/explore.py)
  int tma_variant = 0; // 0: b-bucketed ProductTwoCoin layout + TMA kernel; -1: a-sorted layout, first-generation kernel only (fixed at finalize)
  int use_tma = 1;     // 0: run the first-generation kernel even when the layout exists
  int orient_by_degree = -1; // ProductTwoCoin: store each pool with its higher-degree token first: -1 auto (skewed graphs only), 0 never, 1 always (fixed at finalize)
  int psi_fixed_point = 1;   // Ψ[b] partials of the TMA kernel: 1 = 64-bit fixed point on native shared atomics when the pool set allows it, 0 = fp64 CAS adds
  int sweep_events = 0;      // 1 = record ev0/ev1 around every sweep (cfmm_last_sweep_ms); disables the sweep graphs
  bool events_recorded = false;
  int geomean_log2 = 1;   // gradient-only GeometricMean sweeps: power through exp2/log2 (1, default) or pow (0)
  int gradient_math = 1;  // gradient-only ProductTwoCoin sweeps: 1 = economized (few-ulp), 0 = reference order (bit-identical per pool)
  unsigned long long epoch = 0;  // sweeps enqueued so far
  DevBuf<double> d_accum[2];     // ping-pong [Ψ; acc] accumulators, zeroed one sweep ahead in-kernel
  double* zero_pending = nullptr; // accumulator the first kernel of the current sweep must zero
  DevBuf<unsigned long long> d_grid_done;  // fused exchange: CTAs arrived, summed over all sweeps
  unsigned long long grid_done_target = 0;
  int fused_exchange = 1;         // product-only sets: run the peer exchange in the sweep kernel's tail
  int grid_waves = -1;            // first-generation kernel: waves of CTAs (-1 = 1; 0 = one CTA per 512 pools; see launch_sweep)
  int exchange_protocol = 0;      // 0 = by world size, 1 = LL one-shot, 2 = LL two-shot, 3 = direct 8-byte push (peer_exchange.cuh)
  int coop_launch = 0;            // fused exchange: launch the sweep kernel cooperatively
  int exchange_bypass = 0;        // 1 = sweeps return this rank's partial [Ψ; acc] (no exchange); every rank must agree
  cfmm::FusedExchange fx_pending; // set by enqueue_sweep when the next TMA launch must carry the exchange
  int blocks_per_sm = 0;  // 0 = occupancy-derived
  DevBuf<unsigned long long> d_trace;  // option "trace": per-CTA phase timestamps of the last TMA sweep
  int trace_grid = 0;
  // cfmm_sweep as ONE graph launch {H2D ν, sweep kernels, D2H [Ψ; acc]} per (accumulator
  // parity, counter-set parity): captured the second time the same pinned host buffers are
  // passed with unchanged options; any option / reserve / comm change invalidates (version)
  struct SweepGraph {
    cudaGraphExec_t exec = nullptr;
    const double* v = nullptr;
    double* psi = nullptr;
    unsigned long long version = 0;
    const double* seen_v = nullptr;  // key of the last eager call (capture on the next match)
    double* seen_psi = nullptr;
    unsigned long long seen_version = ~0ull;
    int64_t launches = 0;            // kernel launches one replay stands for
  } graphs[2][4];
  unsigned long long state_version = 1;
  int use_graphs = 1;
  bool capturing = false;  // cfmm_sweep is recording a graph: no event queries / side copies
  bool calibrating = false;  // cfmm_finalize is running its calibration sweeps (range table feedback every launch)
  const void* pinned_ok[2] = {nullptr, nullptr};  // host pointers already verified as pinned
  int balance = 1;              // 1 = TMA kernel: CTA ranges sized by measured CTA speed (feedback), 0 = even split
  int geomean_tma = 1;          // gradient-only GeometricMean sweeps on the TMA kernel (0: first-generation kernel)
  int compact_stream = 1;       // ProductTwoCoin, economized math: 20-byte pool records (γ dictionary, chunk-relative a) when the set allows it
  int compact_record = 0;       // pools per compact record: 96 or 192; 0 = 192 on sets with at least 4 records per resident warp
  int l2_keep = -1;             // TMA sweeps of streams larger than the L2: keep the first h records of every CTA's range in the L2 (-1 = h by L2 size, 0 = no hints)
  // resident CTAs per SM of every kernel instantiation this context has launched.
  // Per context, not per process: cudaFuncSetAttribute (the > 48 KB dynamic shared
  // memory opt-in) acts on the current device only, and contexts of one process
  // may sit on different devices and be driven from different host threads.
  std::unordered_map<const void*, int> occupancy;
  // the pair index of cfmm_pair_pools and the split orders (split_kernels.cuh): built on first use
  // after cfmm_finalize, cfmm_append_* or cfmm_compact (which move pools); retiring or restoring a
  // pool keeps it, activity is read when a row is priced
  struct PairIndex {
    bool built = false;
    int64_t n_pairs = 0;
    DevBuf<int64_t> keys, off, pool;  // distinct keys ascending; CSR [n_pairs + 1]; entries by key
    // the token adjacency of cfmm_scan_arbitrage (arb_scan_kernels.cuh): built on first use after
    // the index, kept with it
    bool adj_built = false;
    DevBuf<int64_t> adj_off;             // [n_tokens + 1]
    DevBuf<int32_t> adj_nbr, adj_pair;   // [2·n_pairs]
    std::vector<int64_t> adj_off_host;
  } pairs;
  // the workspace of cfmm_quote_token_values (token_value_kernels.cuh): grown on demand, holds
  // nothing between calls
  DevBuf<unsigned char> tv_ws;
  int64_t launches = 0;
  std::string err;
  cfmm::PeerExchange comm;
  // optional per-kernel timing (option "profile"): event pairs per launch
  struct Prof {
    std::vector<cudaEvent_t> ev;  // 2 per recorded launch
    std::vector<int> type;        // pool type (3 = peer exchange, 4 = swap kernels)
    size_t used = 0;              // launches recorded
  } prof;
};

namespace {

int fail(cfmm_ctx* ctx, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (ctx)
    ctx->err = buf;
  else
    g_create_error = buf;
  return code;
}

#define CU_TRY(ctx, expr)                                                      \
  do {                                                                         \
    cudaError_t _e = (expr);                                                   \
    if (_e != cudaSuccess)                                                     \
      return fail((ctx), CFMM_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,        \
                  cudaGetErrorString(_e), __FILE__, __LINE__);                 \
  } while (0)

int check_common(cfmm_ctx* ctx, int64_t m, const double* R, const double* gamma,
                 const int64_t* Ai, bool append = false) {
  if (!ctx) return CFMM_ERR_INVALID;
  if (append && !ctx->finalized)
    return fail(ctx, CFMM_ERR_STATE, "pools are appended after cfmm_finalize (cfmm_add_* before it)");
  if (!append && ctx->finalized)
    return fail(ctx, CFMM_ERR_STATE, "pools cannot be added after cfmm_finalize");
  if (m < 0) return fail(ctx, CFMM_ERR_INVALID, "negative pool count");
  if (m > 0 && (!gamma || !Ai || !R))
    return fail(ctx, CFMM_ERR_INVALID, "null array argument");
  // first offending pool, if any (parallel scan; the error names the lowest index like a serial one)
  int64_t bad = m;
  const int64_t nt = ctx->n_tokens;
#pragma omp parallel for schedule(static) reduction(min : bad) if (m > (1 << 16))
  for (int64_t i = 0; i < m; ++i) {
    const int64_t a = Ai[2 * i], b = Ai[2 * i + 1];
    if (a < 1 || a > nt || b < 1 || b > nt || a == b) bad = i < bad ? i : bad;
  }
  for (int64_t i = bad; i < m && i == bad; ++i) {
    const int64_t a = Ai[2 * i], b = Ai[2 * i + 1];
    if (a < 1 || a > ctx->n_tokens || b < 1 || b > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID,
                  "pool %lld: token index (%lld, %lld) outside 1..%lld",
                  (long long)i, (long long)a, (long long)b,
                  (long long)ctx->n_tokens);
    if (a == b)
      return fail(ctx, CFMM_ERR_INVALID,
                  "pool %lld: Ai[1] == Ai[2] == %lld (a two-coin pool needs two "
                  "distinct tokens)",
                  (long long)i, (long long)a);
  }
  return CFMM_OK;
}

void append_common(cfmm_ctx* ctx, PoolSet& s, int64_t m, const double* R,
                   const double* gamma, const int64_t* Ai) {
  if (R) s.R.insert(s.R.end(), R, R + 2 * m);
  s.gamma.insert(s.gamma.end(), gamma, gamma + m);
  s.Ai.insert(s.Ai.end(), Ai, Ai + 2 * m);
  {
    const size_t old = s.gidx.size();
    s.gidx.resize(old + (size_t)m);
    int64_t* gi = s.gidx.data() + old;
    const int64_t base = ctx->n_pools;
#pragma omp parallel for schedule(static) if (m > (1 << 16))
    for (int64_t i = 0; i < m; ++i) gi[i] = base + i;
  }
  s.m += m;
  ctx->n_pools += m;
}

inline bool fast_range_ok(double v) { return v >= cfmm::kFastLo && v <= cfmm::kFastHi; }

// layout of one pool type (pool_layout.hpp): ProductTwoCoin gets the b-bucketed,
// chunk-padded layout of the TMA kernel; the other types are a-sorted only.
// Tail sets (bucketed = false) always get the a-sorted layout of tma_variant -1.
cfmm::PoolLayout layout_for(const cfmm_ctx* ctx, int type, const int64_t* Ai, int64_t m, bool bucketed,
                            void (*mark)(const char*) = nullptr) {
  const bool product = type == CFMM_POOL_PRODUCT;
  cfmm::TileShape shape;
  if ((product || type == CFMM_POOL_GEOMEAN) && bucketed && ctx->tma_variant >= 0) {
    shape.tile = cfmm::kTmaChunk;
    shape.nbmax = cfmm::kTmaNbMax;
  }
  return cfmm::build_pool_layout(Ai, m, ctx->n_tokens, ctx->orient_by_degree, product, shape, shape, mark);
}

int refresh_scale(cfmm_ctx* ctx, PoolSet& s);

// finalize timing (environment CFMM_TIMING): phase marks on stderr
struct PhaseClock {
  bool on = getenv("CFMM_TIMING") != nullptr;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  void mark(const char* what) {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    fprintf(stderr, "[cfmm]   %-36s %.3f s\n", what, std::chrono::duration<double>(t1 - t0).count());
    t0 = t1;
  }
};
PhaseClock* g_layout_clock = nullptr;  // (finalize is serialised per process while timing is on)
void layout_mark(const char* what) {
  if (g_layout_clock) g_layout_clock->mark(what);
}

constexpr size_t kBounceBytes = (size_t)16 << 20;

// dst[p] = fill(p) for p in [0, count): gathered in parallel into the pinned bounce buffers,
// block by block, each block copied asynchronously on the context stream while the next one is
// gathered.  Returns with copies possibly still in flight (upload_set synchronises once).
template <class T, class Fill>
cudaError_t upload_streamed(cfmm_ctx* ctx, DevBuf<T>& dst, int64_t count, Fill fill) {
  cudaError_t e = dst.alloc((size_t)count);
  if (e != cudaSuccess || count == 0) return e;
  for (int k = 0; k < 2; ++k) {
    if (!ctx->h_bounce[k] && (e = cudaMallocHost(&ctx->h_bounce[k], kBounceBytes)) != cudaSuccess) return e;
    if (!ctx->ev_bounce[k] &&
        (e = cudaEventCreateWithFlags(&ctx->ev_bounce[k], cudaEventDisableTiming)) != cudaSuccess)
      return e;
  }
  const int64_t per = (int64_t)(kBounceBytes / sizeof(T));
  int k = 0;
  for (int64_t lo = 0; lo < count; lo += per, k ^= 1) {
    const int64_t hi = std::min(count, lo + per);
    if ((e = cudaEventSynchronize(ctx->ev_bounce[k])) != cudaSuccess) return e;
    T* out = (T*)ctx->h_bounce[k];
#pragma omp parallel for schedule(static) if (hi - lo > (1 << 14))
    for (int64_t p = lo; p < hi; ++p) out[p - lo] = fill(p);
    if ((e = cudaMemcpyAsync(dst.p + lo, out, (size_t)(hi - lo) * sizeof(T), cudaMemcpyHostToDevice,
                             ctx->stream)) != cudaSuccess)
      return e;
    if ((e = cudaEventRecord(ctx->ev_bounce[k], ctx->stream)) != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cfmm::Univ3State univ3_state(PoolSet& s) {
  cfmm::Univ3State u;
  u.f0 = s.d_first[0].p;
  u.f1 = s.d_first[1].p;
  u.f2 = s.d_first[2].p;
  u.f3 = s.d_first[3].p;
  u.tick = s.d_tick.p;
  u.tickdata = s.d_tickdata.p;
  u.lower = s.d_lower.p;
  u.liq = s.d_liq.p;
  u.active = s.d_active.p;
  u.m = s.m;
  u.total_ticks = s.total_ticks;
  return u;
}

// Rebuild the derived UniV3 state (univ3_state.cuh) of the pools d_pos[0..count) (d_pos ==
// nullptr: all pools), whose ticks d_cum lists (n_ticks in all), after storing the optional new
// prices / liquidities (device arrays in listing order).  Enqueued on the context stream.
cudaError_t univ3_rebuild(cfmm_ctx* ctx, PoolSet& s, const int64_t* d_pos, const int64_t* d_cum, int64_t count,
                          int64_t n_ticks, const double* d_price, const double* d_liq, bool new_tick) {
  const cfmm::Univ3State u = univ3_state(s);
  const int threads = 256;
  if (count > 0 && (new_tick || d_price)) {
    cfmm::univ3_current_tick_kernel<<<(unsigned)((count + threads - 1) / threads), threads, 0, ctx->stream>>>(
        u, d_pos, d_price, count);
    ctx->launches++;
  }
  if (n_ticks > 0) {
    cfmm::univ3_ticks_kernel<<<(unsigned)((n_ticks + threads - 1) / threads), threads, 0, ctx->stream>>>(
        u, d_pos, d_cum, count, n_ticks, d_liq);
    ctx->launches++;
  }
  return cudaGetLastError();
}

// Lay out the staged pools of s (a main set, or a tail: tail = true) and upload them.
int upload_set(cfmm_ctx* ctx, int type, PoolSet& s, bool tail) {
  if (s.m == 0) return CFMM_OK;
  const int64_t m = s.m;
  PhaseClock clock;
  g_layout_clock = clock.on ? &clock : nullptr;
  cfmm::PoolLayout lay = layout_for(ctx, type, s.Ai.data(), m, !tail, clock.on ? layout_mark : nullptr);
  g_layout_clock = nullptr;
  const cfmm::HVec<int>&oa = lay.oa, &ob = lay.ob;
  s.swapped.swap(lay.swapped);
  s.skewed = lay.skewed;
  s.order.swap(lay.order);
  s.m_padded = lay.m_padded;
  s.tma_ok = lay.bucketed;
  s.nb = (int)lay.nb;
  if (s.tma_ok) {
    // bucket boundaries in chunks, for the kernel-parameter table
    const int B = lay.tile_bucket.empty() ? 0 : lay.tile_bucket.back() + 1;
    if (B > cfmm::kTmaMaxBuckets) {
      s.tma_ok = false;  // more b-buckets than the parameter table holds: first-generation kernel
    } else {
      s.n_chunks = (int64_t)lay.tile_bucket.size();
      s.buckets.n_buckets = B;
      int b = 0;
      s.buckets.first_chunk[0] = 0;
      for (int64_t c = 0; c < s.n_chunks; ++c)
        while (b < lay.tile_bucket[(size_t)c]) s.buckets.first_chunk[++b] = (int)c;
      while (b < B) s.buckets.first_chunk[++b] = (int)s.n_chunks;
    }
  }
  const int64_t mp = s.m_padded;
  const int64_t* order = s.order.data();
  // padding pools trail their bucket (fewer than one chunk of them): keyed like the last real
  // pool before them (monotone a), zero reserves, unit fee
  const auto real_before = [order](int64_t p) -> int64_t {
    while (p >= 0 && order[p] < 0) --p;
    return p < 0 ? -1 : order[p];
  };
  CU_TRY(ctx, upload_streamed(ctx, s.d_gam, mp, [&](int64_t p) {
    const int64_t i = order[p];
    return i < 0 ? 1.0 : s.gamma[(size_t)i];
  }));
  CU_TRY(ctx, upload_streamed(ctx, s.d_Ai, mp, [&](int64_t p) {
    const int64_t i = real_before(p);
    return i < 0 ? make_int2(0, 1) : make_int2(oa[(size_t)i], ob[(size_t)i]);
  }));
  // bit 62 of the global index marks a pool stored with its tokens exchanged
  CU_TRY(ctx, upload_streamed(ctx, s.d_gidx, mp, [&](int64_t p) {
    const int64_t i = order[p];
    return i < 0 ? (int64_t)-1 : (s.gidx[(size_t)i] | (s.swapped[(size_t)i] ? (1ll << 62) : 0));
  }));
  clock.mark("gather + upload gamma, Ai, gidx");
  s.compact_ok = false;
  s.rec18_ok = false;
  if (type == CFMM_POOL_PRODUCT && s.tma_ok) {
    // 192-pool records: consecutive chunks of a bucket in pairs
    std::vector<int> chunk_rec((size_t)s.n_chunks);
    s.n_recs = 0;
    for (int b = 0; b < s.buckets.n_buckets; ++b) {
      const int c0 = s.buckets.first_chunk[b], c1 = s.buckets.first_chunk[b + 1];
      s.rec_buckets.first_chunk[b] = (int)s.n_recs;
      for (int c = c0; c < c1; ++c) {
        const int k = c - c0;
        chunk_rec[(size_t)c] = (int)((s.n_recs + k / 2) << 2) | ((k & 1) << 1) | ((k & 1) == 0 && c + 1 == c1 ? 1 : 0);
      }
      s.n_recs += (c1 - c0 + 1) / 2;
    }
    s.rec_buckets.n_buckets = s.buckets.n_buckets;
    s.rec_buckets.first_chunk[s.buckets.n_buckets] = (int)s.n_recs;
    // the compact stream stores a as an offset from its record's first a: the span of every
    // 192-pool record must fit the field (the 96-pool records are its halves).  The layout is fixed
    // here and reserve updates do not move a.
    int64_t max_span = 0;
#pragma omp parallel for schedule(static) reduction(max : max_span) if (s.n_chunks > (1 << 12))
    for (int64_t c = 0; c < s.n_chunks; ++c) {
      const int v = chunk_rec[(size_t)c];
      if (v & 2) continue;  // second chunk of a record
      const int64_t end = (v & 1) ? c + 1 : c + 2;
      const int64_t first = real_before(c * cfmm::kTmaChunk), last = real_before(end * cfmm::kTmaChunk - 1);
      const int64_t span = (first < 0 || last < 0) ? 0 : (int64_t)oa[(size_t)last] - (int64_t)oa[(size_t)first];
      max_span = std::max(max_span, span);
    }
    // γ dictionary of the compact stream: fees are categorical in practice.  Pass 1 (serial,
    // cheap): the distinct values, through a 1024-slot open-addressing table on the bit pattern;
    // pass 2 (the upload's gather): the codes
    std::vector<double> vals;
    constexpr int kSlots = 1024;
    std::vector<long long> key(kSlots, -1);
    std::vector<int> val(kSlots, 0);
    auto slot_of = [&](double g, bool insert) -> int {
      long long bits;
      memcpy(&bits, &g, sizeof(bits));
      if (bits == -1) return -1;  // (a NaN pattern: no dictionary)
      unsigned h = (unsigned)((unsigned long long)bits * 0x9E3779B97F4A7C15ull >> 54);
      for (;;) {
        if (key[h] == bits) return val[h];
        if (key[h] == -1) {
          if (!insert || vals.size() == (size_t)cfmm::kTmaGammaCodes) return -1;
          key[h] = bits;
          val[h] = (int)vals.size();
          vals.push_back(g);
          return val[h];
        }
        h = (h + 1) & (kSlots - 1);
      }
    };
    // (the padding pools' fee, inserted first: code 0, which pack_chunks_compact_kernel relies on)
    bool ok = max_span <= cfmm::kMetaMaxSpan && slot_of(1.0, true) >= 0;
    double last = 1.0;
    for (int64_t i = 0; i < m && ok; ++i) {
      const double g = s.gamma[(size_t)i];
      if (g != last) {
        ok = (g == g) && slot_of(g, true) >= 0;
        last = g;
      }
    }
    if (ok) {
      std::vector<double> tab(2 * cfmm::kTmaGammaCodes, 1.0);
      for (size_t k = 0; k < vals.size(); ++k) {
        volatile double inv = 1.0 / vals[k];  // IEEE division, as inv of the 32-byte stream (pack_chunks_kernel)
        tab[k] = inv;
        tab[cfmm::kTmaGammaCodes + k] = vals[k];
      }
      CU_TRY(ctx, upload_streamed(ctx, s.d_gcode, mp, [&](int64_t p) {
        const int64_t i = order[p];
        return (unsigned short)slot_of(i < 0 ? 1.0 : s.gamma[(size_t)i], false);
      }));
      CU_TRY(ctx, s.d_gtab.upload(tab));
      CU_TRY(ctx, s.d_chunk_rec.upload(chunk_rec));
      s.compact_ok = true;
      // the 192-pool record's 64-byte headers (product_tma.cuh, kTmaRec18PoolBytes): a_base, the
      // record's γ codes (at most four among its real pools), the a of every lane's first pool
      // relative to a_base (<= 255); and every lane's first tokens must span at most 7
      constexpr int kHdrWords = cfmm::kTmaRec18HeaderBytes / 4;
      std::vector<unsigned> hdr((size_t)s.n_recs * kHdrWords, 0u);
      int rec18_bad = 0;
#pragma omp parallel for schedule(static) reduction(| : rec18_bad) if (s.n_chunks > (1 << 12))
      for (int64_t c = 0; c < s.n_chunks; ++c) {
        const int v = chunk_rec[(size_t)c];
        if (v & 2) continue;  // second chunk of a record
        unsigned* h = hdr.data() + (size_t)(v >> 2) * kHdrWords;
        // logical pool q of the record: device position c·96 + q; the second half of a record
        // without a second chunk repeats the first half's last a (pack_chunks_compact_kernel)
        auto a_at = [&](int q) {
          const int64_t i = real_before(c * cfmm::kTmaChunk + ((v & 1) ? std::min(q, cfmm::kTmaChunk - 1) : q));
          return i < 0 ? (int64_t)0 : (int64_t)oa[(size_t)i];
        };
        const int64_t a_base = a_at(0);
        h[0] = (unsigned)a_base;
        int n_fees = 0;
        unsigned fees[cfmm::kRec18Fees] = {};
        bool ok18 = true;
        for (int l = 0; l < 32 && ok18; ++l) {
          const int64_t a_lane = a_at(l * cfmm::kTmaL6);
          ok18 = a_lane - a_base <= cfmm::kRec18MaxLaneOff &&
                 a_at(l * cfmm::kTmaL6 + cfmm::kTmaL6 - 1) - a_lane < (1 << cfmm::kRec18ABits);
          h[2 + l / 4] |= (unsigned)(a_lane - a_base) << (8 * (l % 4));
          for (int j = 0; j < cfmm::kTmaL6 && ok18; ++j) {
            const int q = l * cfmm::kTmaL6 + j;
            if ((v & 1) && q >= cfmm::kTmaChunk) break;
            const int64_t i = order[c * cfmm::kTmaChunk + q];
            if (i < 0) continue;  // padding: fee slot 0, whatever its code
            const unsigned code = (unsigned)slot_of(s.gamma[(size_t)i], false);
            int k = 0;
            while (k < n_fees && fees[k] != code) ++k;
            if (k == n_fees) {
              if (n_fees == cfmm::kRec18Fees) ok18 = false;
              else fees[n_fees++] = code;
            }
          }
        }
        for (int k = 0; k < cfmm::kRec18Fees; ++k) h[1] |= fees[k < n_fees ? k : 0] << (8 * k);
        rec18_bad |= ok18 ? 0 : 1;
      }
      s.rec18_ok = rec18_bad == 0;
      if (s.rec18_ok) CU_TRY(ctx, s.d_rec_hdr.upload(hdr));
    }
    clock.mark("fee dictionary + codes");
  }
  if (type != CFMM_POOL_UNIV3) {
    int bad_range = 0;
#pragma omp parallel for schedule(static) reduction(| : bad_range) if (m > (1 << 16))
    for (int64_t i = 0; i < m; ++i) {
      const bool ok = fast_range_ok(s.R[2 * i]) && fast_range_ok(s.R[2 * i + 1]) &&
                      fast_range_ok(s.gamma[(size_t)i]) && s.gamma[(size_t)i] <= 1.0;
      bad_range |= ok ? 0 : 1;
    }
    s.in_fast_range = bad_range == 0;
    CU_TRY(ctx, upload_streamed(ctx, s.d_R, mp, [&](int64_t p) {
      const int64_t i = order[p];
      if (i < 0) return make_double2(0.0, 0.0);
      return s.swapped[(size_t)i] ? make_double2(s.R[2 * i + 1], s.R[2 * i])
                                  : make_double2(s.R[2 * i], s.R[2 * i + 1]);
    }));
    clock.mark("range check, gather + upload R");
    if (s.tma_ok) {
      int rc = refresh_scale(ctx, s);
      if (rc != CFMM_OK) return rc;
      clock.mark("scale table (device)");
    }
  }
  if (type == CFMM_POOL_GEOMEAN) {
    CU_TRY(ctx, upload_streamed(ctx, s.d_w, mp, [&](int64_t p) {
      const int64_t i = order[p];  // (padding pools: any valid weights)
      return i < 0 ? make_double2(0.5, 0.5) : make_double2(s.w[2 * i], s.w[2 * i + 1]);
    }));
  }
  if (type == CFMM_POOL_UNIV3) {
    // the raw tick data goes to the device in device pool order; the tick records and the
    // current-tick streams are computed there (univ3_state.cuh)
    std::vector<int64_t> dev_off((size_t)m + 1, 0);
    for (int64_t p = 0; p < m; ++p) {
      const int64_t i = order[p];
      dev_off[(size_t)p + 1] = dev_off[(size_t)p] + (s.tick_off[(size_t)i + 1] - s.tick_off[(size_t)i]);
    }
    s.total_ticks = dev_off[(size_t)m];
    s.first_lower.resize((size_t)m);
    s.n_ticks.resize((size_t)m);
    for (int64_t i = 0; i < m; ++i) {
      s.first_lower[(size_t)i] = s.lower[(size_t)s.tick_off[(size_t)i]];
      s.n_ticks[(size_t)i] = s.tick_off[(size_t)i + 1] - s.tick_off[(size_t)i];
    }
    std::vector<double> lower((size_t)s.total_ticks), liq((size_t)s.total_ticks);
#pragma omp parallel for schedule(static) if (m > (1 << 14))
    for (int64_t p = 0; p < m; ++p) {
      const int64_t i = order[p], b = s.tick_off[(size_t)i], nt = s.n_ticks[(size_t)i];
      std::copy(s.lower.begin() + b, s.lower.begin() + b + nt, lower.begin() + dev_off[(size_t)p]);
      std::copy(s.liq.begin() + b, s.liq.begin() + b + nt, liq.begin() + dev_off[(size_t)p]);
    }
    CU_TRY(ctx, s.d_lower.upload(lower));
    CU_TRY(ctx, s.d_liq.upload(liq));
    CU_TRY(ctx, upload_streamed(ctx, s.d_tick, m, [&](int64_t p) { return make_int2((int)dev_off[(size_t)p], 0); }));
    CU_TRY(ctx, upload_streamed(ctx, s.d_first[1], m, [&](int64_t p) {
      return make_double2(0.0, s.cp[(size_t)order[p]]);
    }));
    for (int f : {0, 2, 3}) {
      CU_TRY(ctx, s.d_first[f].alloc((size_t)m));
      CU_TRY(ctx, cudaMemsetAsync(s.d_first[f].p, 0, (size_t)m * sizeof(double2), ctx->stream));
    }
    CU_TRY(ctx, s.d_tickdata.alloc((size_t)s.total_ticks * cfmm::kTickStride));
    CU_TRY(ctx, univ3_rebuild(ctx, s, nullptr, nullptr, m, s.total_ticks, nullptr, nullptr, true));
    if (ctx->d_nu_mat.n != (size_t)ctx->n_tokens) CU_TRY(ctx, ctx->d_nu_mat.alloc((size_t)ctx->n_tokens));
    clock.mark("univ3 tick data: upload + device rebuild");
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // the bounce copies read the staging below
  clock.mark("other arrays, drain");
  // host staging is no longer needed (order is kept for update_reserves)
  std::vector<double>().swap(s.R);
  std::vector<double>().swap(s.gamma);
  std::vector<double>().swap(s.w);
  std::vector<int64_t>().swap(s.Ai);
  std::vector<int64_t>().swap(s.gidx);
  std::vector<double>().swap(s.cp);
  std::vector<int64_t>().swap(s.tick_off);
  std::vector<double>().swap(s.lower);
  std::vector<double>().swap(s.liq);
  clock.mark("free host staging");
  return CFMM_OK;
}

// Sweeps may be enqueued on a caller-supplied stream (cfmm_sweep_device*), everything else runs
// on the context's own stream; the ping-pong accumulators, the trade buffers and the reserves
// make consecutive operations dependent.  Whenever the stream changes, the new one waits for
// the work enqueued on the previous one.
int use_stream(cfmm_ctx* ctx, cudaStream_t st) {
  if (ctx->last_stream && ctx->last_stream != st) {
    cudaError_t e = cudaEventRecord(ctx->ev_order, ctx->last_stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, ctx->ev_order, 0);
    if (e != cudaSuccess)
      return fail(ctx, CFMM_ERR_CUDA, "stream ordering failed: %s", cudaGetErrorString(e));
  }
  ctx->last_stream = st;
  return CFMM_OK;
}

// the first kernel of a sweep zeroes the other ping-pong accumulator
inline double* take_zero_pending(cfmm_ctx* ctx) {
  double* p = ctx->zero_pending;
  ctx->zero_pending = nullptr;
  return p;
}

// profiling: bracket one launch with events on its stream
struct ProfScope {
  cfmm_ctx* ctx;
  cudaStream_t st;
  bool on;
  ProfScope(cfmm_ctx* c, int type, cudaStream_t s) : ctx(c), st(s) {
    on = c->prof.used < c->prof.type.size();
    if (on) {
      c->prof.type[c->prof.used] = type;
      cudaEventRecord(c->prof.ev[2 * c->prof.used], st);
    }
  }
  ~ProfScope() {
    if (on) {
      cudaEventRecord(ctx->prof.ev[2 * ctx->prof.used + 1], st);
      ctx->prof.used++;
    }
  }
};

constexpr int kProfSwaps = 4;  // cfmm_profile_read: the slot of the swap, path, order and arbitrage kernels
constexpr int kNoProf = -1;    // launch: not timed

// One launch site on ctx->stream: enqueue() enqueues the site's n kernels, timed as one profile
// entry of slot prof (kNoProf: not timed).  enqueue returns void, or an int status when it also
// makes library calls that can fail (cub).
template <class F>
int launch(cfmm_ctx* ctx, int prof, int64_t n, F&& enqueue) {
  int rc = CFMM_OK;
  {
    std::optional<ProfScope> scope;
    if (prof != kNoProf) scope.emplace(ctx, prof, ctx->stream);
    if constexpr (std::is_void_v<decltype(enqueue())>)
      enqueue();
    else
      rc = enqueue();
  }
  if (rc != CFMM_OK) return rc;
  ctx->launches += n;
  CU_TRY(ctx, cudaGetLastError());
  return CFMM_OK;
}

// Async D2H copy of n elements on ctx->stream, skipped when dst is null (an output not asked for)
// or n == 0.
template <class T>
cudaError_t read_back(cfmm_ctx* ctx, T* dst, const T* src, size_t n) {
  if (!dst || n == 0) return cudaSuccess;
  return cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream);
}

template <class P>
int launch_sweep(cfmm_ctx* ctx, int ptype, const P& pools, PoolSet& s,
                 const double* d_v, double* d_psi, bool mat, cudaStream_t st) {
  constexpr int U = 2;
  const int64_t per_block = (int64_t)cfmm::kSweepThreads * U;
  const int64_t m_all = s.m_padded;  // includes the zero-trade padding pools, if any
  int64_t blocks = (m_all + per_block - 1) / per_block;
  // persistent-style grid: one wave of resident CTAs (SM count x occupancy)
  int& occ = ctx->occupancy[mat ? reinterpret_cast<const void*>(&cfmm::sweep_kernel<P, true, U>)
                                 : reinterpret_cast<const void*>(&cfmm::sweep_kernel<P, false, U>)];
  if (occ == 0) {
    if (mat)
      CU_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                      &occ, cfmm::sweep_kernel<P, true, U>, cfmm::kSweepThreads, 0));
    else
      CU_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                      &occ, cfmm::sweep_kernel<P, false, U>, cfmm::kSweepThreads, 0));
    if (occ < 1) occ = 1;
  }
  const int per_sm = ctx->blocks_per_sm > 0 && ctx->blocks_per_sm < occ ? ctx->blocks_per_sm : occ;
  // grid_waves: 1 (default) = one wave of resident CTAs striding over the pools; 0 = one CTA per
  // 512 pools, handed out by the hardware block scheduler (an alternative for UniV3, whose tick
  // walks make the work per pool uneven -- kept as a knob)
  const int waves = ctx->grid_waves >= 0 ? ctx->grid_waves : 1;
  const int64_t cap = (int64_t)ctx->sm_count * per_sm * (waves > 0 ? waves : 1);
  if (waves > 0 && blocks > cap) blocks = cap;
  if (mat && s.d_outD.n != (size_t)m_all) {
    CU_TRY(ctx, s.d_outD.alloc((size_t)m_all));
    CU_TRY(ctx, s.d_outL.alloc((size_t)m_all));
  }
  ProfScope prof(ctx, ptype, st);
  if (mat) {
    cfmm::sweep_kernel<P, true, U><<<(unsigned)blocks, cfmm::kSweepThreads, 0, st>>>(
        pools, d_v, d_psi, (int)ctx->n_tokens, s.d_outD.p, s.d_outL.p, m_all,
        ctx->exact | (ctx->debug_skip << 1), take_zero_pending(ctx));
  } else {
    cfmm::sweep_kernel<P, false, U><<<(unsigned)blocks, cfmm::kSweepThreads, 0, st>>>(
        pools, d_v, d_psi, (int)ctx->n_tokens, nullptr, nullptr, m_all,
        ctx->exact | (ctx->debug_skip << 1) | (ctx->gradient_math ? 16 : 0), take_zero_pending(ctx));
  }
  ctx->launches++;
  CU_TRY(ctx, cudaGetLastError());
  return CFMM_OK;
}

// (Re)compute the per-token scale table of the fixed-point slice and whether the pool set
// qualifies for it (three small kernels, off the hot path: finalize and every reserve
// mutation).  Marks the packed stream stale.
int refresh_scale(cfmm_ctx* ctx, PoolSet& s) {
  s.fixed_ok = false;
  s.packed_mode = -1;
  if (!s.tma_ok || s.m_padded == 0) return CFMM_OK;
  const int64_t mp = s.m_padded;
  const int n = (int)ctx->n_tokens;
  cudaStream_t st = ctx->stream;
  const int threads = 256;
  const unsigned pblocks = (unsigned)((mp + threads - 1) / threads);
  if (s.d_inv_scale.n != (size_t)n) CU_TRY(ctx, s.d_inv_scale.alloc((size_t)n));
  if (s.d_tok_sum.n != (size_t)n + 2) CU_TRY(ctx, s.d_tok_sum.alloc((size_t)n + 2));  // + 2 flag words
  CU_TRY(ctx, cudaMemsetAsync(s.d_tok_sum.p, 0, ((size_t)n + 2) * sizeof(double), st));
  int* d_flags = reinterpret_cast<int*>(s.d_tok_sum.p + n);
  cfmm::token_reserve_sum_kernel<<<pblocks, threads, 0, st>>>(s.d_R.p, s.d_Ai.p, mp, s.d_tok_sum.p);
  cfmm::token_scale_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, st>>>(
      s.d_tok_sum.p, n, s.d_inv_scale.p, d_flags);
  cfmm::scale_check_kernel<<<pblocks, threads, 0, st>>>(s.d_R.p, s.d_Ai.p, mp, s.d_tok_sum.p,
                                                      s.d_inv_scale.p, d_flags);
  ctx->launches += 3;
  int h_flags[2] = {0, 0};
  CU_TRY(ctx, cudaMemcpyAsync(h_flags, d_flags, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  CU_TRY(ctx, cudaGetLastError());
  s.fixed_ok = h_flags[0] == 0 && h_flags[1] == 0;
  return CFMM_OK;
}

// Keep rule of a TMA sweep over the 192-pool records, `stream_bytes` in all (see product_sweep_tma): 0 = no
// L2 hints, else the first h records of every CTA's range are kept in the L2 across sweeps.  A
// stream that fits in the L2 stays there without hints.  Else h = the records every warp of a CTA
// fetches before the CTA's shared counter takes over (two per warp), at most 40 % of the L2 over the
// grid.  On an H100 (50 MB L2, 264 CTAs) with the headline set's records, h = 8 / 16 / 24 / 32 / 48
// measured 78.3 / 77.3 / 77.6 / 77.0 / 79.7 against 81.2 µs without hints (DESIGN §4.1 r3 g).
int l2_keep_of(const cfmm_ctx* ctx, int64_t stream_bytes) {
  if (ctx->l2_keep == 0 || ctx->l2_bytes <= 0 || stream_bytes <= ctx->l2_bytes) return 0;
  if (ctx->l2_keep > 0) return ctx->l2_keep;
  constexpr int L6 = cfmm::kTmaL6;
  const int64_t ctas = (int64_t)ctx->sm_count * cfmm::tma_ctas_per_sm<0, L6>();
  const int64_t fit = ctx->l2_bytes * 40 / 100 / (ctas * cfmm::tma_chunk_bytes_c<0, true, L6>());
  return (int)std::min<int64_t>(2 * cfmm::tma_warps<0, L6>(), fit);
}

// the kept records of the stream back to evict_normal, once no sweep reads them under the same rule
int l2_release(cfmm_ctx* ctx, PoolSet& s, cudaStream_t st) {
  if (s.l2_keep == 0 || !s.d_packed.p) return CFMM_OK;
  s.l2_keep = 0;
  cfmm::l2_evict_normal_kernel<<<(unsigned)ctx->sm_count * 4, 256, 0, st>>>(s.d_packed.p, s.d_packed.n);
  ctx->launches++;
  CU_TRY(ctx, cudaGetLastError());
  return CFMM_OK;
}

// the packed stream of the mode this sweep runs in (rebuilt when the mode or the reserves changed)
template <int POOL, int L = cfmm::kTmaL>
int ensure_packed(cfmm_ctx* ctx, PoolSet& s, bool econ, bool fixed, bool compact, cudaStream_t st) {
  const int mode = (econ ? 1 : 0) | (fixed ? 2 : 0) | (compact ? 4 : 0) | (L != cfmm::kTmaL ? 8 : 0);
  if (s.packed_mode == mode) return CFMM_OK;
  {
    const int rc = l2_release(ctx, s, st);  // (the buffer is rewritten or freed)
    if (rc != CFMM_OK) return rc;
  }
  const size_t wide = (size_t)s.n_chunks * cfmm::tma_chunk_bytes<POOL>();
  const size_t bytes = !compact ? wide
                       : L == cfmm::kTmaL ? (size_t)s.n_chunks * cfmm::tma_chunk_bytes_c<POOL, true>()
                                          : (size_t)s.n_recs * cfmm::tma_chunk_bytes_c<POOL, true, L>();
  if (s.d_packed.n < bytes) CU_TRY(ctx, s.d_packed.alloc(std::max(bytes, wide)));
  const int threads = 256;
  if (compact) {
    cfmm::pack_chunks_compact_kernel<L><<<(unsigned)((s.m_padded + threads - 1) / threads), threads, 0, st>>>(
        s.d_R.p, s.d_Ai.p, s.d_gcode.p, s.m_padded, s.nb, fixed ? s.d_inv_scale.p : nullptr, s.d_chunk_rec.p,
        s.d_packed.p, s.d_rec_hdr.p);
    ctx->launches++;
    CU_TRY(ctx, cudaGetLastError());
    s.packed_mode = mode;
    return CFMM_OK;
  }
  // ProductTwoCoin's economized form streams 1/γ; GeometricMean always γ
  cfmm::pack_chunks_kernel<<<(unsigned)((s.m_padded + threads - 1) / threads), threads, 0, st>>>(
      s.d_R.p, s.d_gam.p, s.d_Ai.p, POOL == 1 ? s.d_w.p : nullptr, s.m_padded,
      fixed ? s.d_inv_scale.p : nullptr, (POOL == 0 && econ) ? 1 : 0, cfmm::tma_chunk_bytes<POOL>(), s.d_packed.p);
  ctx->launches++;
  CU_TRY(ctx, cudaGetLastError());
  s.packed_mode = mode;
  return CFMM_OK;
}

template <int POOL, bool ECON, bool SKEW, bool FIXED, bool COMPACT = false, int L = cfmm::kTmaL>
int launch_tma_cfg(cfmm_ctx* ctx, PoolSet& s, const double* d_v, double* d_psi, cudaStream_t st) {
  auto kern = cfmm::product_sweep_tma<POOL, ECON, SKEW, FIXED, COMPACT, L>;
  constexpr int kThreads = cfmm::tma_threads<POOL, L>(), kSmem = cfmm::tma_smem_bytes_c<POOL, COMPACT, L>();
  int& occ = ctx->occupancy[reinterpret_cast<const void*>(kern)];
  if (occ == 0) {
    CU_TRY(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    CU_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kThreads, kSmem));
    if (occ < 1) return fail(ctx, CFMM_ERR_CUDA, "product_sweep_tma does not fit on an SM");
  }
  int rc = ensure_packed<POOL, L>(ctx, s, ECON, FIXED, COMPACT, st);
  if (rc != CFMM_OK) return rc;
  // the unit of the bucket and range tables: 96-pool chunks, or the 192-pool records
  const int64_t n_units = L == cfmm::kTmaL ? s.n_chunks : s.n_recs;
  const cfmm::BucketTable& tab = L == cfmm::kTmaL ? s.buckets : s.rec_buckets;
  if (s.range_pools != 32 * L) {  // a table in the other unit: start over
    s.range_pools = 32 * L;
    s.ranges.n = -1;
  }
  // (grid and range table)
  const int per_sm = ctx->blocks_per_sm > 0 && ctx->blocks_per_sm < occ ? ctx->blocks_per_sm : occ;
  int grid = ctx->sm_count * per_sm;
  if (grid > n_units) grid = (int)n_units;
  // ---- speed-weighted ranges (see product_tma.cuh) ---------------------------------------
  unsigned* d_dur = nullptr;
  const bool tabled = grid <= cfmm::kTmaMaxRanges;
  const bool balancing = ctx->balance && tabled && n_units >= (int64_t)grid * 32;
  auto set_buckets = [&]() {  // b-bucket of every range's first chunk
    int b = 0;
    for (int g = 0; g <= grid; ++g) {
      const int c = g < grid ? s.ranges.first[g] : (int)n_units - 1;
      while (b + 1 < tab.n_buckets && tab.first_chunk[b + 1] <= c) ++b;
      s.ranges.bucket[g] = (short)b;
    }
  };
  if (!tabled) {
    s.ranges.n = 0;
  } else if (s.ranges.n != grid || !balancing) {
    if (s.ranges.n != grid || s.range_updates != 0) {  // (first launch with this grid, or balancing switched off)
      s.ranges.n = grid;
      for (int g = 0; g <= grid; ++g) s.ranges.first[g] = (int)(n_units * g / grid);
      set_buckets();
      s.speed.assign((size_t)grid, 1.0);
      s.range_version = (s.range_version % 250) + 1;
      s.range_updates = 0;
      s.dur_pending = false;
    }
  }
  if (balancing) {
    if (!s.h_dur) {
      CU_TRY(ctx, cudaMallocHost((void**)&s.h_dur, (cfmm::kTmaMaxRanges + 1) * sizeof(unsigned)));
      memset(s.h_dur, 0, (cfmm::kTmaMaxRanges + 1) * sizeof(unsigned));
      CU_TRY(ctx, s.d_dur.alloc(cfmm::kTmaMaxRanges + 1));
      CU_TRY(ctx, cudaMemset(s.d_dur.p, 0, (cfmm::kTmaMaxRanges + 1) * sizeof(unsigned)));
      CU_TRY(ctx, cudaStreamSynchronize(cudaStreamLegacy));  // (memsets run on the legacy stream; ours do not wait for it)
      CU_TRY(ctx, cudaEventCreateWithFlags(&s.ev_dur, cudaEventDisableTiming));
    }
    d_dur = s.d_dur.p;
    // a copy of the durations has landed: were they all measured under the CURRENT table?
    if (s.dur_pending && !ctx->capturing && cudaEventQuery(s.ev_dur) == cudaSuccess) {
      s.dur_pending = false;
      bool complete = true;
      const unsigned* hd = s.h_dur;
      for (int g = 0; g < grid && complete; ++g) complete = (hd[g] >> 24) == s.range_version && (hd[g] & 0xffffffu) != 0;
      if (complete) {
        double total = 0.0;
        for (int g = 0; g < grid; ++g) {
          const double len = (double)(s.ranges.first[g + 1] - s.ranges.first[g]);
          const double dur = (double)(hd[g] & 0xffffffu);
          const double rel = len / dur;  // chunks per tick
          const double keep = ctx->calibrating ? 0.5 : 0.8;
          s.speed[(size_t)g] = s.range_updates == 0 ? rel : keep * s.speed[(size_t)g] + (1.0 - keep) * rel;
          total += s.speed[(size_t)g];
        }
        // only the persistent part of the speed differences is worth following (SM position on the
        // die); launch-to-launch noise is as large: heavy smoothing, and lengths within +-15 % of even
        {
          const double mean = total / grid;
          total = 0.0;
          for (int g = 0; g < grid; ++g) {
            double& sp = s.speed[(size_t)g];
            sp = std::min(1.15 * mean, std::max(0.85 * mean, sp));
            total += sp;
          }
        }
        // new boundaries: lengths proportional to speed, exact total
        double acc_len = 0.0;
        int prev = 0;
        for (int g = 0; g < grid; ++g) {
          acc_len += (double)n_units * s.speed[(size_t)g] / total;
          int end = g + 1 == grid ? (int)n_units : (int)(acc_len + 0.5);
          const int min_end = prev + 1, max_end = (int)n_units - (grid - 1 - g);
          end = end < min_end ? min_end : (end > max_end ? max_end : end);
          s.ranges.first[g + 1] = end;
          prev = end;
        }
        set_buckets();
        s.range_version = (s.range_version % 250) + 1;
        s.range_updates++;
      }
    }
  }
  s.ranges.version = s.range_version;
  s.balancing = balancing;
  s.tma_launches++;
  cfmm::FusedExchange fx = ctx->fx_pending;
  if (fx.mode != 0) {
    fx.target = ctx->grid_done_target + (unsigned long long)grid;
    fx.grid_done = ctx->d_grid_done.p;
    ctx->fx_pending.mode = 0;  // consumed
  }
  const int a_keep = COMPACT && L == cfmm::kTmaL6 ? l2_keep_of(ctx, n_units * cfmm::tma_chunk_bytes_c<POOL, COMPACT, L>()) : 0;
  if (a_keep != s.l2_keep && (rc = l2_release(ctx, s, st)) != CFMM_OK) return rc;
  s.l2_keep = a_keep;
  ProfScope prof(ctx, POOL == 0 ? CFMM_POOL_PRODUCT : CFMM_POOL_GEOMEAN, st);
  const unsigned char* a_packed = s.d_packed.p;
  const double* a_gam = COMPACT ? s.d_gtab.p : s.d_gam.p;  // compact stream: the γ dictionary instead of per-pool γ
  int a_nb = s.nb, a_n = (int)ctx->n_tokens, a_range = s.in_fast_range ? 1 : 0, a_flags = ctx->exact;
  const double* a_scale = FIXED ? s.d_inv_scale.p : nullptr;
  double* a_zero = take_zero_pending(ctx);
  unsigned long long* a_trace = ctx->d_trace.n ? ctx->d_trace.p : nullptr;
  if (fx.mode != 0 && ctx->coop_launch) {
    // the fused exchange meets at a grid-wide barrier: a COOPERATIVE launch makes the driver
    // guarantee that every CTA is resident (or fail the launch) instead of inferring it
    void* args[] = {&a_packed, &a_gam, const_cast<cfmm::BucketTable*>(&tab), &a_nb, &d_v, &a_scale, &d_psi, &a_n, &a_zero,
                    &a_range, &a_flags, const_cast<int*>(&a_keep), &fx, &s.ranges, &d_dur, &a_trace};
    CU_TRY(ctx, cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(kThreads),
                                            args, kSmem, st));
  } else {
    kern<<<grid, kThreads, kSmem, st>>>(a_packed, a_gam, tab, a_nb, d_v, a_scale, d_psi, a_n, a_zero,
                                        a_range, a_flags, a_keep, fx, s.ranges, d_dur, a_trace);
  }
  if (ctx->d_trace.n) ctx->trace_grid = grid;
  ctx->launches++;
  CU_TRY(ctx, cudaGetLastError());
  // the grid-barrier target moves only once the launch is known to be accepted
  if (fx.mode != 0) ctx->grid_done_target = fx.target;
  // fetch the durations now and then: often while the table is still settling, rarely afterwards
  if (balancing && !ctx->capturing && !s.dur_pending &&
      ++s.since_copy >= (ctx->calibrating ? 1 : (s.range_updates < 8 ? 4 : 256))) {
    s.since_copy = 0;
    CU_TRY(ctx, cudaMemcpyAsync(s.h_dur, s.d_dur.p, (size_t)grid * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    CU_TRY(ctx, cudaEventRecord(s.ev_dur, st));
    s.dur_pending = true;
  }
  return CFMM_OK;
}

// Pools per compact record a gradient-only ProductTwoCoin sweep of the main set s streams under the
// current options: 192 (18-byte pool records), 96 (20-byte pool records), 0 (the 32-byte stream).
int compact_record_of(const cfmm_ctx* ctx, const PoolSet& s) {
  if (!(ctx->gradient_math != 0 && ctx->compact_stream && s.compact_ok && !ctx->exact)) return 0;
  // 192-pool records halve the per-record work (wait, counter, re-arm) and combine Ψ[a] over
  // the warp, but leave warps idle on small sets: taken when every resident warp gets several
  constexpr int L6 = cfmm::kTmaL6;
  const int64_t warps = (int64_t)ctx->sm_count * cfmm::tma_ctas_per_sm<0, L6>() * cfmm::tma_warps<0, L6>();
  const bool rec192 = s.rec18_ok && (ctx->compact_record == 192 || (ctx->compact_record == 0 && s.n_recs >= 4 * warps));
  return rec192 ? 192 : 96;
}

template <int POOL>
int launch_tma(cfmm_ctx* ctx, PoolSet& s, const double* d_v, double* d_psi, cudaStream_t st) {
  const bool econ = ctx->gradient_math != 0;
  const bool fixed = ctx->psi_fixed_point && s.fixed_ok;
  if constexpr (POOL == 0) {
    const int rec = compact_record_of(ctx, s);
    if (rec != 0) {
      constexpr int L6 = cfmm::kTmaL6;
      if (rec == 192) {
        if (!s.skewed && fixed) return launch_tma_cfg<0, true, false, true, true, L6>(ctx, s, d_v, d_psi, st);
        if (!s.skewed && !fixed) return launch_tma_cfg<0, true, false, false, true, L6>(ctx, s, d_v, d_psi, st);
        if (s.skewed && fixed) return launch_tma_cfg<0, true, true, true, true, L6>(ctx, s, d_v, d_psi, st);
        return launch_tma_cfg<0, true, true, false, true, L6>(ctx, s, d_v, d_psi, st);
      }
      if (!s.skewed && fixed) return launch_tma_cfg<0, true, false, true, true>(ctx, s, d_v, d_psi, st);
      if (!s.skewed && !fixed) return launch_tma_cfg<0, true, false, false, true>(ctx, s, d_v, d_psi, st);
      if (s.skewed && fixed) return launch_tma_cfg<0, true, true, true, true>(ctx, s, d_v, d_psi, st);
      return launch_tma_cfg<0, true, true, false, true>(ctx, s, d_v, d_psi, st);
    }
  }
#define CFMM_TMA_CASE(E, K, F) \
  if (econ == E && s.skewed == K && fixed == F) return launch_tma_cfg<POOL, E, K, F>(ctx, s, d_v, d_psi, st);
  CFMM_TMA_CASE(true, false, true)
  CFMM_TMA_CASE(true, false, false)
  CFMM_TMA_CASE(false, false, true)
  CFMM_TMA_CASE(false, false, false)
  if constexpr (POOL == 0) {  // hub orientation exists for the symmetric pool type only
    CFMM_TMA_CASE(true, true, true)
    CFMM_TMA_CASE(true, true, false)
    CFMM_TMA_CASE(false, true, true)
    CFMM_TMA_CASE(false, true, false)
  }
#undef CFMM_TMA_CASE
  return fail(ctx, CFMM_ERR_INVALID, "unreachable");
}

// One sweep.  The kernels accumulate into the internal ping-pong accumulator
// of this sweep (already zero: the previous sweep's first kernel cleared it) and
// clear the other one for the next sweep.  The result goes to d_dst if given
// (peer exchange writes it there directly; single GPU: one D2D copy), else it
// stays in the accumulator; *view receives the device pointer that holds it.
int enqueue_sweep(cfmm_ctx* ctx, const double* d_v, double* d_dst, bool mat,
                  cudaStream_t st, const double** view) {
  {
    int rc0 = use_stream(ctx, st);
    if (rc0 != CFMM_OK) return rc0;
  }
  if (ctx->sweep_events) CU_TRY(ctx, cudaEventRecord(ctx->ev0, st));
  ctx->events_recorded = ctx->sweep_events != 0;
  ctx->epoch++;
  double* d_psi = ctx->d_accum[ctx->epoch & 1].p;
  ctx->zero_pending = ctx->d_accum[(ctx->epoch + 1) & 1].p;
  const size_t acc_bytes = (size_t)(ctx->n_tokens + 1) * sizeof(double);
  // Fused compute+collective: when the TMA ProductTwoCoin kernel is the only
  // kernel of this sweep, it runs the peer exchange in its own tail.
  bool fused = false;
  {
    const PoolSet& ps = ctx->sets[CFMM_POOL_PRODUCT];
    const bool no_tails = ctx->tails[0].m == 0 && ctx->tails[1].m == 0 && ctx->tails[2].m == 0;
    if (ctx->comm.attached() && !ctx->exchange_bypass && ctx->fused_exchange && !mat && ps.m > 0 && ps.tma_ok && ctx->use_tma &&
        ctx->debug_skip == 0 && ctx->sets[CFMM_POOL_GEOMEAN].m == 0 && ctx->sets[CFMM_POOL_UNIV3].m == 0 && no_tails) {
      fused = true;
      ctx->fx_pending.view = ctx->comm.view();
      ctx->fx_pending.dst = d_dst ? d_dst : d_psi;
      ctx->fx_pending.epoch = ctx->comm.begin_fused(&ctx->fx_pending.mode);
    }
  }
  int rc;
  {
    PoolSet& s = ctx->sets[CFMM_POOL_PRODUCT];
    constexpr int PT = CFMM_POOL_PRODUCT;
    if (s.m > 0) {
      if (!mat && s.tma_ok && ctx->use_tma && ctx->debug_skip == 0) {
        if ((rc = launch_tma<0>(ctx, s, d_v, d_psi, st)) != CFMM_OK) return rc;
      } else {
        cfmm::ProductPools p{s.d_R.p, s.d_gam.p, s.d_Ai.p};
        if ((rc = launch_sweep(ctx, PT, p, s, d_v, d_psi, mat, st)) != CFMM_OK) return rc;
      }
    }
    PoolSet& t = ctx->tails[PT];  // appended pools: first-generation kernel, same accumulator
    if (t.m > 0) {
      cfmm::ProductPools p{t.d_R.p, t.d_gam.p, t.d_Ai.p};
      if ((rc = launch_sweep(ctx, PT, p, t, d_v, d_psi, mat, st)) != CFMM_OK) return rc;
    }
  }
  {
    PoolSet& s = ctx->sets[CFMM_POOL_GEOMEAN];
    constexpr int PT = CFMM_POOL_GEOMEAN;
    if (s.m > 0) {
      cfmm::GeomeanPools p{s.d_R.p, s.d_gam.p, s.d_Ai.p, s.d_w.p};
      if (!mat && s.tma_ok && ctx->use_tma && ctx->geomean_tma && ctx->geomean_log2 && ctx->debug_skip == 0) {
        if ((rc = launch_tma<1>(ctx, s, d_v, d_psi, st)) != CFMM_OK) return rc;
      } else if (ctx->geomean_log2 && !mat) {
        cfmm::GeomeanPoolsLog2 q;
        static_cast<cfmm::GeomeanPools&>(q) = p;
        if ((rc = launch_sweep(ctx, PT, q, s, d_v, d_psi, mat, st)) != CFMM_OK) return rc;
      } else if ((rc = launch_sweep(ctx, PT, p, s, d_v, d_psi, mat, st)) != CFMM_OK) {
        return rc;
      }
    }
    PoolSet& t = ctx->tails[PT];
    if (t.m > 0) {
      cfmm::GeomeanPools p{t.d_R.p, t.d_gam.p, t.d_Ai.p, t.d_w.p};
      if (ctx->geomean_log2 && !mat) {
        cfmm::GeomeanPoolsLog2 q;
        static_cast<cfmm::GeomeanPools&>(q) = p;
        if ((rc = launch_sweep(ctx, PT, q, t, d_v, d_psi, mat, st)) != CFMM_OK) return rc;
      } else if ((rc = launch_sweep(ctx, PT, p, t, d_v, d_psi, mat, st)) != CFMM_OK) {
        return rc;
      }
    }
  }
  {
    constexpr int PT = CFMM_POOL_UNIV3;
    for (PoolSet* ps : {&ctx->sets[PT], &ctx->tails[PT]}) {
      PoolSet& s = *ps;
      if (s.m == 0) continue;
      cfmm::Univ3Pools p{s.d_first[0].p, s.d_first[1].p, s.d_first[2].p, s.d_first[3].p, s.d_gam.p, s.d_Ai.p, s.d_tick.p,
                         s.d_tickdata.p, s.m_padded, (int)s.total_ticks};
      if ((rc = launch_sweep(ctx, PT, p, s, d_v, d_psi, mat, st)) != CFMM_OK) return rc;
    }
    // cfmm_apply_trades moves UniV3 prices by the ν of the last materialising sweep: keep it,
    // since the caller's d_v (and the context's own ν buffer) may be overwritten before then
    if (mat && (ctx->sets[PT].m > 0 || ctx->tails[PT].m > 0))
      CU_TRY(ctx, cudaMemcpyAsync(ctx->d_nu_mat.p, d_v, (size_t)ctx->n_tokens * sizeof(double),
                                  cudaMemcpyDeviceToDevice, st));
  }
  if (ctx->zero_pending) {  // no kernel ran (empty pool set): clear the other accumulator here
    CU_TRY(ctx, cudaMemsetAsync(take_zero_pending(ctx), 0, acc_bytes, st));
  }
  const double* result = d_psi;
  if (fused) {
    result = d_dst ? d_dst : d_psi;
  } else if (ctx->comm.attached() && !ctx->exchange_bypass) {
    ProfScope prof(ctx, 3, st);
    double* dst = d_dst ? d_dst : d_psi;
    if (!ctx->comm.all_reduce(d_psi, dst, ctx->n_tokens + 1, st))
      return fail(ctx, CFMM_ERR_COMM, "peer exchange failed: %s",
                  ctx->comm.error().c_str());
    ctx->launches += ctx->comm.launches_per_reduce();
    result = dst;
  } else if (d_dst) {
    CU_TRY(ctx, cudaMemcpyAsync(d_dst, d_psi, acc_bytes, cudaMemcpyDeviceToDevice, st));
    result = d_dst;
  }
  if (view) *view = result;
  if (ctx->sweep_events) CU_TRY(ctx, cudaEventRecord(ctx->ev1, st));
  if (mat) ctx->has_trades = true;
  return CFMM_OK;
}

int ready(cfmm_ctx* ctx) {
  if (!ctx) return CFMM_ERR_INVALID;
  if (!ctx->finalized)
    return fail(ctx, CFMM_ERR_STATE, "cfmm_finalize has not been called");
  return CFMM_OK;
}

// Calibration (cfmm_finalize, cfmm_compact): a dozen gradient sweeps at ν = 1 settle the
// speed-weighted CTA ranges of the TMA kernels (and pay the one-time costs of the first launch:
// function attributes, stream packing) here rather than in the caller's first sweeps.  ~1 ms.
int calibrate(cfmm_ctx* ctx) {
  bool any = false;
  for (int t : {CFMM_POOL_PRODUCT, CFMM_POOL_GEOMEAN}) any = any || (ctx->sets[t].m > 0 && ctx->sets[t].tma_ok);
  if (!any || !ctx->balance) return CFMM_OK;
  std::vector<double> ones((size_t)ctx->n_tokens, 1.0);
  CU_TRY(ctx, DevBuf<double>::copy_in(ctx->d_nu.p, ones.data(), ones.size() * sizeof(double)));
  ctx->calibrating = true;
  int rc = CFMM_OK;
  for (int it = 0; it < 12 && rc == CFMM_OK; ++it) {
    const double* view = nullptr;
    rc = enqueue_sweep(ctx, ctx->d_nu.p, nullptr, false, ctx->stream, &view);
    if (rc == CFMM_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess)
      rc = fail(ctx, CFMM_ERR_CUDA, "calibration sweep failed: %s", cudaGetErrorString(cudaGetLastError()));
  }
  ctx->calibrating = false;
  return rc;
}

}  // namespace

// ---------------------------------------------------------------------------

extern "C" {

const char* cfmm_version(void) { return "0.1.0"; }

const char* cfmm_last_error(const cfmm_ctx* ctx) {
  return ctx ? ctx->err.c_str() : g_create_error.c_str();
}

int cfmm_create(cfmm_ctx** out, int device, int64_t n_tokens) {
  if (!out) return fail(nullptr, CFMM_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (n_tokens < 1 || n_tokens > (int64_t)0x7ffffff0)
    return fail(nullptr, CFMM_ERR_INVALID, "n_tokens must be in 1..2^31-16");
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0)
    return fail(nullptr, CFMM_ERR_CUDA,
                "no CUDA device available (%s); libcfmm_b200 has no CPU path",
                e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device < 0 || device >= n_dev)
    return fail(nullptr, CFMM_ERR_INVALID, "device %d out of range 0..%d", device,
                n_dev - 1);
  cfmm_ctx* ctx = new (std::nothrow) cfmm_ctx();
  if (!ctx) return fail(nullptr, CFMM_ERR_NOMEM, "out of host memory");
  ctx->device = device;
  ctx->n_tokens = n_tokens;
#define CREATE_TRY(expr)                                                    \
  do {                                                                      \
    cudaError_t _e = (expr);                                                \
    if (_e != cudaSuccess) {                                                \
      fail(nullptr, CFMM_ERR_CUDA, "%s failed: %s", #expr,                  \
           cudaGetErrorString(_e));                                         \
      cfmm_destroy(ctx);                                                    \
      return CFMM_ERR_CUDA;                                                 \
    }                                                                       \
  } while (0)
  CREATE_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CREATE_TRY(cudaGetDeviceProperties(&prop, device));
  ctx->sm_count = prop.multiProcessorCount;
  ctx->l2_bytes = prop.l2CacheSize;
  CREATE_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CREATE_TRY(cudaEventCreateWithFlags(&ctx->ev_order, cudaEventDisableTiming));
  CREATE_TRY(cudaEventCreate(&ctx->ev0));
  CREATE_TRY(cudaEventCreate(&ctx->ev1));
  CREATE_TRY(ctx->d_nu.alloc((size_t)n_tokens));
  CREATE_TRY(ctx->d_grid_done.alloc(1));
  CREATE_TRY(cudaMemset(ctx->d_grid_done.p, 0, sizeof(unsigned long long)));
  memset(&ctx->fx_pending, 0, sizeof(ctx->fx_pending));
  for (auto& a : ctx->d_accum) {
    CREATE_TRY(a.alloc((size_t)n_tokens + 1));
    CREATE_TRY(cudaMemset(a.p, 0, ((size_t)n_tokens + 1) * sizeof(double)));
  }
  CREATE_TRY(cudaStreamSynchronize(cudaStreamLegacy));  // the memsets above ran on the legacy stream; ctx->stream does not wait for it
  CREATE_TRY(cudaMallocHost((void**)&ctx->h_stage, (size_t)(n_tokens + 1) * sizeof(double)));
#undef CREATE_TRY
  *out = ctx;
  return CFMM_OK;
}

namespace {
void drop_graphs(cfmm_ctx* ctx);
}

void cfmm_destroy(cfmm_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  for (auto& s : ctx->sets)
    if (ctx->stream) l2_release(ctx, s, ctx->stream);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  ctx->comm.detach();
  drop_graphs(ctx);
  for (auto e : ctx->prof.ev)
    if (e) cudaEventDestroy(e);
  for (auto& s : ctx->sets) s.release();
  for (auto& s : ctx->tails) s.release();
  ctx->d_nu.release();
  ctx->d_nu_mat.release();
  ctx->d_grid_done.release();
  ctx->d_trace.release();
  ctx->d_accum[0].release();
  ctx->d_accum[1].release();
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  for (void* b : ctx->h_bounce)
    if (b) cudaFreeHost(b);
  for (cudaEvent_t e : ctx->ev_bounce)
    if (e) cudaEventDestroy(e);
  if (ctx->ev_order) cudaEventDestroy(ctx->ev_order);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

int cfmm_add_product(cfmm_ctx* ctx, int64_t m, const double* R,
                     const double* gamma, const int64_t* Ai) {
  int rc = check_common(ctx, m, R, gamma, Ai);
  if (rc != CFMM_OK) return rc;
  append_common(ctx, ctx->sets[CFMM_POOL_PRODUCT], m, R, gamma, Ai);
  return CFMM_OK;
}

int cfmm_add_geomean(cfmm_ctx* ctx, int64_t m, const double* R,
                     const double* gamma, const int64_t* Ai, const double* w) {
  int rc = check_common(ctx, m, R, gamma, Ai);
  if (rc != CFMM_OK) return rc;
  if (m > 0 && !w) return fail(ctx, CFMM_ERR_INVALID, "null weight array");
  PoolSet& s = ctx->sets[CFMM_POOL_GEOMEAN];
  append_common(ctx, s, m, R, gamma, Ai);
  s.w.insert(s.w.end(), w, w + 2 * m);
  return CFMM_OK;
}

namespace {

// cfmm_add_univ3's checks of the CSR arrays (the pools are checked by check_common); ticks_before:
// the ticks already staged in the set the pools go to
int check_univ3(cfmm_ctx* ctx, int64_t m, const double* current_price, const int64_t* tick_off,
                const double* lower_ticks, const double* liquidity, int64_t ticks_before) {
  if (!current_price || !tick_off || !lower_ticks || !liquidity)
    return fail(ctx, CFMM_ERR_INVALID, "null array argument");
  if (tick_off[0] != 0)
    return fail(ctx, CFMM_ERR_INVALID, "tick_off[0] must be 0");
  for (int64_t i = 0; i < m; ++i) {
    const int64_t b = tick_off[i], e = tick_off[i + 1];
    if (e <= b)
      return fail(ctx, CFMM_ERR_INVALID, "univ3 pool %lld has no ticks", (long long)i);
    for (int64_t t = b + 1; t < e; ++t)
      if (!(lower_ticks[t] < lower_ticks[t - 1]))
        return fail(ctx, CFMM_ERR_INVALID,
                    "univ3 pool %lld: lower_ticks must be strictly decreasing",
                    (long long)i);
    if (!(lower_ticks[b] >= current_price[i]))
      return fail(ctx, CFMM_ERR_INVALID,
                  "univ3 pool %lld: current_price above the first lower tick "
                  "(current_tick == 0; BoundsError in the reference)",
                  (long long)i);
  }
  if (ticks_before + tick_off[m] > (int64_t)0x7fffffff)
    return fail(ctx, CFMM_ERR_INVALID, "more than 2^31-1 ticks in one context");
  return CFMM_OK;
}

void stage_univ3(cfmm_ctx* ctx, PoolSet& s, int64_t m, const double* current_price, const double* gamma,
                 const int64_t* Ai, const int64_t* tick_off, const double* lower_ticks, const double* liquidity) {
  const int64_t n_ticks = tick_off[m];
  const int64_t base = (int64_t)s.lower.size();
  if (s.tick_off.empty()) s.tick_off.push_back(0);
  for (int64_t i = 1; i <= m; ++i) s.tick_off.push_back(base + tick_off[i]);
  s.cp.insert(s.cp.end(), current_price, current_price + m);
  s.lower.insert(s.lower.end(), lower_ticks, lower_ticks + n_ticks);
  s.liq.insert(s.liq.end(), liquidity, liquidity + n_ticks);
  append_common(ctx, s, m, nullptr, gamma, Ai);
}

}  // namespace

int cfmm_add_univ3(cfmm_ctx* ctx, int64_t m, const double* current_price,
                   const double* gamma, const int64_t* Ai,
                   const int64_t* tick_off, const double* lower_ticks,
                   const double* liquidity) {
  static const double dummy = 0.0;
  int rc = check_common(ctx, m, m > 0 ? &dummy : nullptr, gamma, Ai);
  if (rc != CFMM_OK) return rc;
  if (m == 0) return CFMM_OK;
  PoolSet& s = ctx->sets[CFMM_POOL_UNIV3];
  if ((rc = check_univ3(ctx, m, current_price, tick_off, lower_ticks, liquidity, (int64_t)s.lower.size())) != CFMM_OK)
    return rc;
  stage_univ3(ctx, s, m, current_price, gamma, Ai, tick_off, lower_ticks, liquidity);
  return CFMM_OK;
}

// ---- flat pool files (SURVEY §8f rank 1: an ingest format that is not an array of heap
// objects).  Little-endian, 64-byte header {magic "CFMMPOOL", u32 version = 1, u32 pool
// type, i64 m, i64 n_tokens, zero pad}, then the SoA arrays exactly as cfmm_add_* take
// them: R [2m] f64, gamma [m] f64, Ai [2m] i64 (1-based), and w [2m] f64 for
// GeometricMeanTwoCoin.  The file is mmap-ed; cfmm_add_pool_file feeds it to cfmm_add_*.
namespace {
struct PoolFileHeader {
  char magic[8];
  uint32_t version, type;
  int64_t m, n_tokens;
  char pad[32];
};
static_assert(sizeof(PoolFileHeader) == 64, "pool file header");

size_t pool_file_bytes(int type, int64_t m) {
  return sizeof(PoolFileHeader) + (size_t)m * (16 + 8 + 16 + (type == CFMM_POOL_GEOMEAN ? 16 : 0));
}
}  // namespace

int cfmm_pool_file_write(const char* path, int type, int64_t n_tokens, int64_t m, const double* R,
                         const double* gamma, const int64_t* Ai, const double* w) {
  if (!path || m < 0 || n_tokens < 1 || (type != CFMM_POOL_PRODUCT && type != CFMM_POOL_GEOMEAN) ||
      (m > 0 && (!R || !gamma || !Ai || (type == CFMM_POOL_GEOMEAN && !w))))
    return CFMM_ERR_INVALID;
  FILE* f = fopen(path, "wb");
  if (!f) return CFMM_ERR_INVALID;
  PoolFileHeader h;
  memset(&h, 0, sizeof(h));
  memcpy(h.magic, "CFMMPOOL", 8);
  h.version = 1;
  h.type = (uint32_t)type;
  h.m = m;
  h.n_tokens = n_tokens;
  bool ok = fwrite(&h, sizeof(h), 1, f) == 1;
  ok = ok && fwrite(R, 16, (size_t)m, f) == (size_t)m && fwrite(gamma, 8, (size_t)m, f) == (size_t)m &&
       fwrite(Ai, 16, (size_t)m, f) == (size_t)m;
  if (type == CFMM_POOL_GEOMEAN) ok = ok && fwrite(w, 16, (size_t)m, f) == (size_t)m;
  ok = (fclose(f) == 0) && ok;
  return ok ? CFMM_OK : CFMM_ERR_INVALID;
}

int cfmm_pool_file_info(const char* path, int* type, int64_t* n_tokens, int64_t* m) {
  if (!path || !type || !n_tokens || !m) return CFMM_ERR_INVALID;
  FILE* f = fopen(path, "rb");
  if (!f) return CFMM_ERR_INVALID;
  PoolFileHeader h;
  const bool ok = fread(&h, sizeof(h), 1, f) == 1;
  fseek(f, 0, SEEK_END);
  const long size = ftell(f);
  fclose(f);
  if (!ok || memcmp(h.magic, "CFMMPOOL", 8) != 0 || h.version != 1 || h.m < 0 ||
      (h.type != CFMM_POOL_PRODUCT && h.type != CFMM_POOL_GEOMEAN) ||
      (size_t)size != pool_file_bytes((int)h.type, h.m))
    return CFMM_ERR_INVALID;
  *type = (int)h.type;
  *n_tokens = h.n_tokens;
  *m = h.m;
  return CFMM_OK;
}

int cfmm_add_pool_file(cfmm_ctx* ctx, const char* path) {
  if (!ctx) return CFMM_ERR_INVALID;
  int type = 0;
  int64_t n_tokens = 0, m = 0;
  if (cfmm_pool_file_info(path, &type, &n_tokens, &m) != CFMM_OK)
    return fail(ctx, CFMM_ERR_INVALID, "'%s' is not a readable CFMM pool file", path ? path : "(null)");
  if (n_tokens != ctx->n_tokens)
    return fail(ctx, CFMM_ERR_INVALID, "pool file is for %lld tokens, the context for %lld",
                (long long)n_tokens, (long long)ctx->n_tokens);
  if (m == 0) return CFMM_OK;
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return fail(ctx, CFMM_ERR_INVALID, "cannot open '%s'", path);
  const size_t bytes = pool_file_bytes(type, m);
  void* map = mmap(nullptr, bytes, PROT_READ, MAP_PRIVATE | MAP_POPULATE, fd, 0);
  close(fd);
  if (map == MAP_FAILED) return fail(ctx, CFMM_ERR_NOMEM, "mmap of '%s' failed", path);
  const char* base = (const char*)map + sizeof(PoolFileHeader);
  const double* R = (const double*)base;
  const double* gamma = R + 2 * m;
  const int64_t* Ai = (const int64_t*)(gamma + m);
  const double* w = (const double*)(Ai + 2 * m);
  const int rc = type == CFMM_POOL_PRODUCT ? cfmm_add_product(ctx, m, R, gamma, Ai)
                                           : cfmm_add_geomean(ctx, m, R, gamma, Ai, w);
  munmap(map, bytes);
  return rc;
}

int cfmm_finalize(cfmm_ctx* ctx) {
  if (!ctx) return CFMM_ERR_INVALID;
  if (ctx->finalized) return fail(ctx, CFMM_ERR_STATE, "already finalized");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  const bool timing = getenv("CFMM_TIMING") != nullptr;
  auto t0 = std::chrono::steady_clock::now();
  for (int t = 0; t < 3; ++t) {
    int rc = upload_set(ctx, t, ctx->sets[t], false);
    if (rc != CFMM_OK) return rc;
    if (timing) {
      const auto t1 = std::chrono::steady_clock::now();
      fprintf(stderr, "[cfmm] finalize: pool type %d (%lld pools) %.3f s\n", t, (long long)ctx->sets[t].m,
              std::chrono::duration<double>(t1 - t0).count());
      t0 = t1;
    }
  }
  ctx->finalized = true;
  const int rc = calibrate(ctx);
  if (rc == CFMM_OK && timing)
    fprintf(stderr, "[cfmm] finalize: calibration %.3f s\n",
            std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
  return rc;
}

int64_t cfmm_num_pools(const cfmm_ctx* ctx) { return ctx ? ctx->n_pools : -1; }
int64_t cfmm_num_tokens(const cfmm_ctx* ctx) { return ctx ? ctx->n_tokens : -1; }
int64_t cfmm_launch_count(const cfmm_ctx* ctx) { return ctx ? ctx->launches : -1; }

int cfmm_sweep_device(cfmm_ctx* ctx, const double* d_v, double* d_psi_acc,
                      int materialize, void* stream) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!d_v || !d_psi_acc) return fail(ctx, CFMM_ERR_INVALID, "null device pointer");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  return enqueue_sweep(ctx, d_v, d_psi_acc, materialize != 0, st, nullptr);
}

int cfmm_sweep_device_view(cfmm_ctx* ctx, const double* d_v, int materialize, void* stream,
                           const double** d_psi_acc_out) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!d_v || !d_psi_acc_out) return fail(ctx, CFMM_ERR_INVALID, "null pointer");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
  return enqueue_sweep(ctx, d_v, nullptr, materialize != 0, st, d_psi_acc_out);
}

namespace {

bool host_pinned(cfmm_ctx* ctx, const void* p) {
  if (p == ctx->pinned_ok[0] || p == ctx->pinned_ok[1]) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  if (a.type != cudaMemoryTypeHost) return false;
  ctx->pinned_ok[1] = ctx->pinned_ok[0];
  ctx->pinned_ok[0] = p;
  return true;
}

void drop_graphs(cfmm_ctx* ctx) {
  for (auto& row : ctx->graphs)
    for (auto& g : row) {
      if (g.exec) cudaGraphExecDestroy(g.exec);
      g = cfmm_ctx::SweepGraph();
    }
}

}  // namespace

int cfmm_sweep(cfmm_ctx* ctx, const double* v, double* psi_out, double* acc_out,
               int materialize) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!v || !psi_out || !acc_out)
    return fail(ctx, CFMM_ERR_INVALID, "null host pointer");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  const size_t nb = (size_t)ctx->n_tokens * sizeof(double);
  cudaStream_t st = ctx->stream;
  const bool contiguous = acc_out == psi_out + ctx->n_tokens;

  // ---- graph path: the whole call is one cudaGraphLaunch ---------------------------------
  // (a graph freezes the kernel parameters, the range table among them: capture only once the
  // speed feedback of the TMA kernels has settled)
  bool settled = true;
  for (int t : {CFMM_POOL_PRODUCT, CFMM_POOL_GEOMEAN}) {
    const PoolSet& ps = ctx->sets[t];
    if (ps.m > 0 && ps.tma_ok && ctx->use_tma && ctx->balance && (ps.tma_launches == 0 || (ps.balancing && ps.range_updates < 6)))
      settled = false;
  }
  const bool graphable = ctx->use_graphs && !materialize && contiguous && !ctx->sweep_events &&
                         !ctx->comm.attached() && ctx->prof.type.empty() && !ctx->d_trace.n &&
                         ctx->debug_skip == 0 && settled;
  cfmm_ctx::SweepGraph* g = nullptr;
  if (graphable) {
    g = &ctx->graphs[(ctx->epoch + 1) & 1][0];
    if (g->exec && g->v == v && g->psi == psi_out && g->version == ctx->state_version) {
      ctx->epoch++;
      ctx->launches += g->launches;
      ctx->events_recorded = false;
      CU_TRY(ctx, cudaGraphLaunch(g->exec, st));
      CU_TRY(ctx, cudaStreamSynchronize(st));
      return CFMM_OK;
    }
    const bool second = g->seen_v == v && g->seen_psi == psi_out && g->seen_version == ctx->state_version;
    if (second && host_pinned(ctx, v) && host_pinned(ctx, psi_out)) {
      // same buffers, same options as the last call on this parity: capture
      if (g->exec) cudaGraphExecDestroy(g->exec);
      g->exec = nullptr;
      const int64_t l0 = ctx->launches;
      cudaGraph_t graph = nullptr;
      CU_TRY(ctx, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      ctx->capturing = true;
      cudaError_t e = cudaMemcpyAsync(ctx->d_nu.p, v, nb, cudaMemcpyHostToDevice, st);
      const double* res = nullptr;
      if (e == cudaSuccess) rc = enqueue_sweep(ctx, ctx->d_nu.p, nullptr, false, st, &res);
      if (e == cudaSuccess && rc == CFMM_OK)
        e = cudaMemcpyAsync(psi_out, res, nb + sizeof(double), cudaMemcpyDeviceToHost, st);
      cudaError_t e2 = cudaStreamEndCapture(st, &graph);
      ctx->capturing = false;
      if (e == cudaSuccess && rc == CFMM_OK && e2 == cudaSuccess && graph &&
          cudaGraphInstantiate(&g->exec, graph, 0) == cudaSuccess) {
        g->v = v;
        g->psi = psi_out;
        g->version = ctx->state_version;
        g->launches = ctx->launches - l0;
        cudaGraphDestroy(graph);
        CU_TRY(ctx, cudaGraphLaunch(g->exec, st));
        CU_TRY(ctx, cudaStreamSynchronize(st));
        return CFMM_OK;
      }
      // capture failed: the sweep state has advanced without any work being done -- undo and
      // take the eager path for good
      if (graph) cudaGraphDestroy(graph);
      cudaGetLastError();
      g->exec = nullptr;
      ctx->use_graphs = 0;
      ctx->epoch--;
      ctx->launches = l0;
      if (rc != CFMM_OK) return rc;
    }
    g->seen_v = v;
    g->seen_psi = psi_out;
    g->seen_version = ctx->state_version;
  }

  CU_TRY(ctx, cudaMemcpyAsync(ctx->d_nu.p, v, nb, cudaMemcpyHostToDevice, st));
  const double* res = nullptr;
  rc = enqueue_sweep(ctx, ctx->d_nu.p, nullptr, materialize != 0, st, &res);
  if (rc != CFMM_OK) return rc;
  // A peer that died leaves the exchange polling until its timeout (seconds): only a sweep that
  // took that long looks at the error word.
  const auto t_wait = std::chrono::steady_clock::now();
  auto comm_ok = [&]() -> int {
    if (!ctx->comm.attached()) return CFMM_OK;
    if (std::chrono::steady_clock::now() - t_wait < std::chrono::seconds(1)) return CFMM_OK;
    if (ctx->comm.timed_out())
      return fail(ctx, CFMM_ERR_COMM, "peer exchange timed out: a rank of the group did not deliver its packets");
    return CFMM_OK;
  };
  if (contiguous) {
    // caller keeps [psi ; acc] contiguous: one D2H copy
    CU_TRY(ctx, cudaMemcpyAsync(psi_out, res, nb + sizeof(double), cudaMemcpyDeviceToHost, st));
    CU_TRY(ctx, cudaStreamSynchronize(st));
    return comm_ok();
  }
  CU_TRY(ctx, cudaMemcpyAsync(psi_out, res, nb, cudaMemcpyDeviceToHost, st));
  CU_TRY(ctx, cudaMemcpyAsync(ctx->h_stage, res + ctx->n_tokens,
                              sizeof(double), cudaMemcpyDeviceToHost, st));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  *acc_out = ctx->h_stage[0];
  return comm_ok();
}

// ---- cfmm_solve: the outer iteration of route! on the device (solver.cuh) ----------------
int cfmm_solve(cfmm_ctx* ctx, const double* lin, const double* lower, const double* upper,
               const double* v0, const cfmm_solve_opts* opts_in, double* v_out, cfmm_solve_info* info) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!lower || !v_out) return fail(ctx, CFMM_ERR_INVALID, "cfmm_solve: lower and v_out are required");
  cfmm_solve_opts o;
  o.max_iter = 15000;
  o.max_fun = 15000;
  o.pgtol = 1e-5;
  o.factr = 1e1;
  if (opts_in) o = *opts_in;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int64_t n = ctx->n_tokens;
  constexpr int M = cfmm::kSolverM, K = cfmm::kSolverK, NG = cfmm::kSolverGram;
  for (int64_t i = 0; i < n; ++i)
    if (!(lower[i] == lower[i]) || (upper && !(upper[i] >= lower[i])))
      return fail(ctx, CFMM_ERR_INVALID, "cfmm_solve: bad bounds at token %lld", (long long)(i + 1));
  // device state
  DevBuf<double> vec, hist, red, box;
  DevBuf<unsigned> ticket;
  DevBuf<unsigned long long> pgbits;
  CU_TRY(ctx, vec.alloc((size_t)6 * n));
  CU_TRY(ctx, hist.alloc((size_t)2 * M * n));
  CU_TRY(ctx, red.alloc((size_t)cfmm::kSolverMaxBlocks * NG + NG + 8));
  CU_TRY(ctx, box.alloc((size_t)3 * n));
  CU_TRY(ctx, ticket.alloc(1));
  CU_TRY(ctx, pgbits.alloc(1));
  CU_TRY(ctx, cudaMemsetAsync(hist.p, 0, (size_t)2 * M * n * sizeof(double), st));
  CU_TRY(ctx, cudaMemsetAsync(ticket.p, 0, sizeof(unsigned), st));
  CU_TRY(ctx, cudaMemsetAsync(vec.p, 0, (size_t)6 * n * sizeof(double), st));
  cfmm::SolverVecs q;
  q.n = n;
  q.x = vec.p;
  q.g = vec.p + n;
  q.xt = vec.p + 2 * n;
  q.gt = vec.p + 3 * n;
  q.d = vec.p + 4 * n;
  q.pg = vec.p + 5 * n;
  q.S = hist.p;
  q.Y = hist.p + (size_t)M * n;
  q.partials = red.p;
  q.scal = red.p + (size_t)cfmm::kSolverMaxBlocks * NG;
  q.ticket = ticket.p;
  CU_TRY(ctx, cudaMemcpyAsync(box.p, lower, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
  q.lower = box.p;
  q.upper = nullptr;
  q.lin = nullptr;
  if (upper) {
    bool finite = false;
    for (int64_t i = 0; i < n && !finite; ++i) finite = upper[i] < 1.0e300;
    if (finite) {
      CU_TRY(ctx, cudaMemcpyAsync(box.p + n, upper, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
      q.upper = box.p + n;
    }
  }
  if (lin) {
    CU_TRY(ctx, cudaMemcpyAsync(box.p + 2 * n, lin, (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
    q.lin = box.p + 2 * n;
  }
  {
    std::vector<double> start((size_t)n, 1.0 / (double)n);  // route!'s default start, router.jl:62
    if (v0) start.assign(v0, v0 + n);
    CU_TRY(ctx, cudaMemcpyAsync(q.d, start.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
    CU_TRY(ctx, cudaStreamSynchronize(st));  // `start` leaves scope
  }
  int blocks = (int)((n + cfmm::kSolverThreads - 1) / cfmm::kSolverThreads);
  if (blocks > cfmm::kSolverMaxBlocks) blocks = cfmm::kSolverMaxBlocks;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  cudaEventCreate(&t0);
  cudaEventCreate(&t1);
  cudaEventRecord(t0, st);

  double h[NG + 8];
  int fevals = 0;
  auto evaluate = [&](double* f_out) -> int {  // sweep at xt, gt = lin + Ψ, f = linᵀxt + acc
    const double* view = nullptr;
    int r = enqueue_sweep(ctx, q.xt, nullptr, false, st, &view);
    if (r != CFMM_OK) return r;
    cfmm::solver_grad_kernel<<<blocks, cfmm::kSolverThreads, 0, st>>>(q, view);
    ctx->launches++;
    cudaMemcpyAsync(h + NG, q.scal + NG, 5 * sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(h + NG + 5, view + n, sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, CFMM_ERR_CUDA, "cfmm_solve: %s", cudaGetErrorString(e));
    ++fevals;
    *f_out = h[NG + 1] + h[NG + 5];
    return CFMM_OK;
  };
  double W[K][K];
  double pgnorm = 0.0;
  auto commit = [&](int slot, int store) -> int {  // accept xt; W, |pg|_inf back
    cudaMemsetAsync(pgbits.p, 0, sizeof(unsigned long long), st);
    cfmm::solver_commit_kernel<<<blocks, cfmm::kSolverThreads, 0, st>>>(q, slot, store, pgbits.p);
    ctx->launches++;
    unsigned long long bits = 0;
    cudaMemcpyAsync(h, q.scal, NG * sizeof(double), cudaMemcpyDeviceToHost, st);
    cudaMemcpyAsync(&bits, pgbits.p, sizeof(bits), cudaMemcpyDeviceToHost, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, CFMM_ERR_CUDA, "cfmm_solve: %s", cudaGetErrorString(e));
    int k = 0;
    for (int r = 0; r < K; ++r)
      for (int c = r; c < K; ++c) W[r][c] = W[c][r] = h[k++];
    memcpy(&pgnorm, &bits, sizeof(double));
    return CFMM_OK;
  };

  // x = P(v0); first evaluation
  cfmm::solver_init_kernel<<<blocks, cfmm::kSolverThreads, 0, st>>>(q, q.d);
  ctx->launches++;
  double f = 0.0;
  if ((rc = evaluate(&f)) != CFMM_OK) return rc;
  if ((rc = commit(0, 0)) != CFMM_OK) return rc;

  cfmm::LbfgsHistory hist_ages;  // history slots, oldest first
  hist_ages.cnt = hist_ages.head = 0;
  int iter = 0, status = 2, small_steps = 0;
  while (true) {
    if (!(f == f)) { status = 5; break; }            // NaN objective
    if (pgnorm <= o.pgtol) { status = 0; break; }
    if (iter >= o.max_iter) { status = 2; break; }
    if (fevals >= o.max_fun) { status = 3; break; }
    // ---- two-loop recursion in coefficient space over B = [S Y pg] (solver_control.cuh) -------
    cfmm::SolverCoef cf;
    const double t_init = cfmm::lbfgs_direction(W, hist_ages, cf.c);
    cfmm::solver_direction_kernel<<<blocks, cfmm::kSolverThreads, 0, st>>>(q, cf);
    ctx->launches++;
    // ---- Armijo backtracking along the projected path ------------------------------------
    double t = t_init, f_new = f;
    bool accepted = false, stalled = false;
    for (int ls = 0; ls < 30 && fevals < o.max_fun; ++ls) {
      cfmm::solver_trial_kernel<<<blocks, cfmm::kSolverThreads, 0, st>>>(q, t);
      ctx->launches++;
      if ((rc = evaluate(&f_new)) != CFMM_OK) return rc;
      const int d = cfmm::lbfgs_trial(f, f_new, h[NG + 0], h[NG + 2], hist_ages.cnt, t);
      if (d == cfmm::kLsStall) { stalled = true; break; }
      if (d == cfmm::kLsAccept) { accepted = true; break; }
      if (d == cfmm::kLsRestart) break;
    }
    if (!accepted) {
      if (hist_ages.cnt > 0 && !stalled) {  // drop the history and retry with steepest descent
        hist_ages.cnt = 0;
        continue;
      }
      status = stalled ? 1 : 4;
      break;
    }
    // ---- accept: store (s, y), new Gram matrix / projected gradient --------------------------
    const int slot = hist_ages.head;
    if ((rc = commit(slot, 1)) != CFMM_OK) return rc;
    cfmm::lbfgs_store(W, slot, hist_ages);
    ++iter;
    const double f_old = f;
    f = f_new;
    if (cfmm::lbfgs_factr(f_old, f, o.factr, small_steps)) {
      status = 1;
      break;
    }
  }
  // final ν, and the trades at it (router.jl:106-107)
  CU_TRY(ctx, cudaMemcpyAsync(v_out, q.x, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
  const double* view = nullptr;
  if ((rc = enqueue_sweep(ctx, q.x, nullptr, true, st, &view)) != CFMM_OK) return rc;
  cudaEventRecord(t1, st);
  CU_TRY(ctx, cudaStreamSynchronize(st));
  if (info) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, t0, t1);
    info->iterations = iter;
    info->fun_evals = fevals;
    info->status = status;
    info->f = f;
    info->pg_norm = pgnorm;
    info->solve_ms = ms;
  }
  cudaEventDestroy(t0);
  cudaEventDestroy(t1);
  return CFMM_OK;
}

int cfmm_last_sweep_ms(cfmm_ctx* ctx, float* ms_out) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!ms_out) return fail(ctx, CFMM_ERR_INVALID, "ms_out is NULL");
  if (!ctx->events_recorded)
    return fail(ctx, CFMM_ERR_STATE, "the last sweep recorded no events: set option \"sweep_events\" to 1 first");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  CU_TRY(ctx, cudaEventSynchronize(ctx->ev1));
  CU_TRY(ctx, cudaEventElapsedTime(ms_out, ctx->ev0, ctx->ev1));
  return CFMM_OK;
}

namespace {

int64_t type_pools(const cfmm_ctx* ctx, int type) { return ctx->sets[type].m + ctx->tails[type].m; }

// Part of a type-local pool range [first, first + count) that falls in one set: pools
// [0, sets[t].m) of a type are its main set's, the rest its tail's.  `offset`: where the part
// starts within the caller's range.
struct Span {
  PoolSet* s;
  int64_t first, count, offset;
};
std::vector<Span> split_range(cfmm_ctx* ctx, int type, int64_t first, int64_t count) {
  std::vector<Span> out;
  PoolSet& a = ctx->sets[type];
  const int64_t hi = first + count;
  if (count <= 0) return out;
  if (first < a.m) out.push_back({&a, first, std::min(hi, a.m) - first, 0});
  if (hi > a.m) {
    const int64_t lo = std::max(first, a.m);
    out.push_back({&ctx->tails[type], lo - a.m, hi - lo, lo - first});
  }
  return out;
}

void ensure_pos_of(PoolSet& s) {
  if (!s.pos_of.empty() || s.m == 0) return;
  s.pos_of.resize((size_t)s.m);
  for (int64_t p = 0; p < s.m_padded; ++p)
    if (s.order[(size_t)p] >= 0) s.pos_of[(size_t)s.order[(size_t)p]] = p;
}

// A change of the pool set (append, retire / restore, compact): captured sweep graphs are stale,
// and the materialised trades no longer describe the set.
void membership_changed(cfmm_ctx* ctx) {
  ctx->state_version++;
  ctx->has_trades = false;
}

}  // namespace

int cfmm_get_trades(cfmm_ctx* ctx, double* Delta, double* Lambda) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!Delta || !Lambda) return fail(ctx, CFMM_ERR_INVALID, "null host pointer");
  if (!ctx->has_trades)
    return fail(ctx, CFMM_ERR_STATE,
                "no materialising sweep has run since the last change of the pool set (call cfmm_sweep with materialize=1)");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if (ctx->n_pools == 0) return CFMM_OK;
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  DevBuf<double2> allD, allL;
  CU_TRY(ctx, allD.alloc((size_t)ctx->n_pools));
  cudaError_t e = allL.alloc((size_t)ctx->n_pools);
  if (e != cudaSuccess) {
    allD.release();
    return fail(ctx, CFMM_ERR_CUDA, "cudaMalloc failed: %s", cudaGetErrorString(e));
  }
  for (PoolSet* group : {ctx->sets, ctx->tails})
    for (int t = 0; t < 3; ++t) {
      PoolSet& s = group[t];
      if (s.m == 0) continue;
      const int threads = 256;
      const int64_t blocks = (s.m_padded + threads - 1) / threads;
      cfmm::scatter_trades_kernel<<<(unsigned)blocks, threads, 0, ctx->stream>>>(
          s.d_outD.p, s.d_outL.p, s.d_gidx.p, allD.p, allL.p, s.m_padded);
      ctx->launches++;
    }
  const size_t bytes = (size_t)ctx->n_pools * sizeof(double2);
  cudaError_t e1 = cudaMemcpyAsync(Delta, allD.p, bytes, cudaMemcpyDeviceToHost, ctx->stream);
  cudaError_t e2 = cudaMemcpyAsync(Lambda, allL.p, bytes, cudaMemcpyDeviceToHost, ctx->stream);
  cudaError_t e3 = cudaStreamSynchronize(ctx->stream);
  allD.release();
  allL.release();
  if (e1 != cudaSuccess || e2 != cudaSuccess || e3 != cudaSuccess)
    return fail(ctx, CFMM_ERR_CUDA, "trade read-back failed: %s",
                cudaGetErrorString(e1 != cudaSuccess ? e1 : e2 != cudaSuccess ? e2 : e3));
  return CFMM_OK;
}

namespace {

// new reserves of the pools [first, first + count) of one set (insertion order within the set)
int update_reserves_set(cfmm_ctx* ctx, PoolSet& s, int64_t first, int64_t count, const double* R) {
  ensure_pos_of(s);
  std::vector<double2> newR((size_t)count);
  for (int64_t j = 0; j < count; ++j) {
    newR[(size_t)j] = s.swapped[(size_t)(first + j)] ? make_double2(R[2 * j + 1], R[2 * j])
                                                     : make_double2(R[2 * j], R[2 * j + 1]);
    if (!fast_range_ok(R[2 * j]) || !fast_range_ok(R[2 * j + 1])) s.in_fast_range = false;
  }
  DevBuf<double2> d_new;
  DevBuf<int64_t> d_pos;
  CU_TRY(ctx, d_new.upload(newR));
  cudaError_t e = d_pos.upload(s.pos_of.data() + first, (size_t)count);
  if (e == cudaSuccess) {
    const int threads = 256;
    cfmm::update_reserves_kernel<<<(unsigned)((count + threads - 1) / threads), threads, 0,
                                   ctx->stream>>>(s.d_R.p, d_pos.p, d_new.p, count, s.d_active.p, s.d_park.p);
    ctx->launches++;
    e = cudaStreamSynchronize(ctx->stream);
  }
  d_new.release();
  d_pos.release();
  if (e != cudaSuccess)
    return fail(ctx, CFMM_ERR_CUDA, "update_reserves failed: %s", cudaGetErrorString(e));
  if (s.tma_ok) return refresh_scale(ctx, s);
  return CFMM_OK;
}

}  // namespace

int cfmm_update_reserves(cfmm_ctx* ctx, int type, int64_t first, int64_t count,
                         const double* R) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (type != CFMM_POOL_PRODUCT && type != CFMM_POOL_GEOMEAN)
    return fail(ctx, CFMM_ERR_INVALID, "update_reserves: type must be PRODUCT or GEOMEAN");
  const int64_t m = type_pools(ctx, type);
  ctx->state_version++;
  if (first < 0 || count < 0 || first + count > m)
    return fail(ctx, CFMM_ERR_INVALID, "update_reserves: range [%lld, %lld) outside 0..%lld",
                (long long)first, (long long)(first + count), (long long)m);
  if (count == 0) return CFMM_OK;
  if (!R) return fail(ctx, CFMM_ERR_INVALID, "null reserve array");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  for (const Span& sp : split_range(ctx, type, first, count))
    if ((rc = update_reserves_set(ctx, *sp.s, sp.first, sp.count, R + 2 * sp.offset)) != CFMM_OK) return rc;
  return CFMM_OK;
}

namespace {

// Store new prices / liquidities (host arrays in listing order, either may be NULL) of the UniV3
// pools at device positions pos and rebuild their derived state on the device; synchronous.
int univ3_update_listed(cfmm_ctx* ctx, PoolSet& s, const std::vector<int64_t>& pos, const double* price,
                        const double* liq, bool new_tick) {
  const int64_t count = (int64_t)pos.size();
  std::vector<int64_t> cum((size_t)count + 1, 0);
  for (int64_t j = 0; j < count; ++j)
    cum[(size_t)j + 1] = cum[(size_t)j] + s.n_ticks[(size_t)s.order[(size_t)pos[(size_t)j]]];
  const int64_t n_ticks = cum[(size_t)count];
  DevBuf<int64_t> d_pos, d_cum;
  DevBuf<double> d_price, d_liq;
  CU_TRY(ctx, d_pos.upload(pos));
  CU_TRY(ctx, d_cum.upload(cum));
  CU_TRY(ctx, d_price.upload(price, (size_t)count));
  CU_TRY(ctx, d_liq.upload(liq, (size_t)n_ticks));
  CU_TRY(ctx, univ3_rebuild(ctx, s, d_pos.p, d_cum.p, count, n_ticks, d_price.p, d_liq.p, new_tick));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

}  // namespace

int cfmm_update_univ3(cfmm_ctx* ctx, int64_t first, int64_t count, const double* current_price,
                      const double* liquidity) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  const int64_t m = type_pools(ctx, CFMM_POOL_UNIV3);
  if (first < 0 || count < 0 || first + count > m)
    return fail(ctx, CFMM_ERR_INVALID, "update_univ3: range [%lld, %lld) outside 0..%lld",
                (long long)first, (long long)(first + count), (long long)m);
  if (count == 0 || (!current_price && !liquidity)) return CFMM_OK;
  const std::vector<Span> spans = split_range(ctx, CFMM_POOL_UNIV3, first, count);
  // validated like cfmm_add_univ3, all before any change: a rejected call changes no pool
  if (current_price)
    for (const Span& sp : spans)
      for (int64_t j = 0; j < sp.count; ++j)
        if (!(sp.s->first_lower[(size_t)(sp.first + j)] >= current_price[sp.offset + j]))
          return fail(ctx, CFMM_ERR_INVALID,
                      "univ3 pool %lld: current_price above the first lower tick "
                      "(current_tick == 0; BoundsError in the reference)",
                      (long long)(first + sp.offset + j));
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  ctx->state_version++;
  int64_t tick_base = 0;  // liquidities of the parts before this one
  for (const Span& sp : spans) {
    PoolSet& s = *sp.s;
    ensure_pos_of(s);
    std::vector<int64_t> pos(s.pos_of.begin() + sp.first, s.pos_of.begin() + sp.first + sp.count);
    rc = univ3_update_listed(ctx, s, pos, current_price ? current_price + sp.offset : nullptr,
                             liquidity ? liquidity + tick_base : nullptr, current_price != nullptr);
    if (rc != CFMM_OK) return rc;
    for (int64_t j = 0; j < sp.count; ++j) tick_base += s.n_ticks[(size_t)(sp.first + j)];
  }
  return CFMM_OK;
}

int cfmm_apply_trades(cfmm_ctx* ctx) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (!ctx->has_trades)
    return fail(ctx, CFMM_ERR_STATE,
                "no materialising sweep has run since the last change of the pool set (call cfmm_sweep with materialize=1)");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  ctx->state_version++;
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  DevBuf<int> flag;
  std::vector<int> zero(1, 0);
  for (int t : {CFMM_POOL_PRODUCT, CFMM_POOL_GEOMEAN})
    for (PoolSet* ps : {&ctx->sets[t], &ctx->tails[t]}) {
      PoolSet& s = *ps;
      if (s.m == 0) continue;
      if (s.d_outD.n != (size_t)s.m_padded)
        return fail(ctx, CFMM_ERR_STATE, "trades of this pool type were never materialised");
      CU_TRY(ctx, flag.upload(zero));
      const int threads = 256;
      cfmm::apply_trades_kernel<<<(unsigned)((s.m_padded + threads - 1) / threads), threads, 0, ctx->stream>>>(
          s.d_R.p, s.d_gam.p, s.d_outD.p, s.d_outL.p, s.d_gidx.p, s.m_padded, s.d_active.p, flag.p);
      ctx->launches++;
      int h = 0;
      cudaError_t e = cudaMemcpyAsync(&h, flag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
      flag.release();
      if (e != cudaSuccess) return fail(ctx, CFMM_ERR_CUDA, "apply_trades failed: %s", cudaGetErrorString(e));
      if (h) s.in_fast_range = false;  // later sweeps take the generic (guarded) form
      if (s.tma_ok) {
        int rc2 = refresh_scale(ctx, s);
        if (rc2 != CFMM_OK) return rc2;
      }
    }
  for (PoolSet* ps : {&ctx->sets[CFMM_POOL_UNIV3], &ctx->tails[CFMM_POOL_UNIV3]}) {
    PoolSet& u = *ps;
    if (u.m == 0) continue;
    // new prices from the kept ν (univ3_move_kernel), then the state of the pools that moved
    DevBuf<int64_t> moved;
    DevBuf<unsigned long long> n_moved;
    CU_TRY(ctx, moved.alloc((size_t)u.m));
    CU_TRY(ctx, n_moved.alloc(1));
    CU_TRY(ctx, cudaMemsetAsync(n_moved.p, 0, sizeof(unsigned long long), ctx->stream));
    const int threads = 256;
    cfmm::univ3_move_kernel<<<(unsigned)((u.m + threads - 1) / threads), threads, 0, ctx->stream>>>(
        univ3_state(u), u.d_gam.p, u.d_Ai.p, ctx->d_nu_mat.p, moved.p, n_moved.p);
    ctx->launches++;
    unsigned long long h = 0;
    CU_TRY(ctx, cudaMemcpyAsync(&h, n_moved.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (h > 0) {
      std::vector<int64_t> pos((size_t)h);
      CU_TRY(ctx, cudaMemcpy(pos.data(), moved.p, (size_t)h * sizeof(int64_t), cudaMemcpyDeviceToHost));
      std::sort(pos.begin(), pos.end());  // (the list order is the atomics'; sorted, the rebuild reads in device order)
      if ((rc = univ3_update_listed(ctx, u, pos, nullptr, nullptr, true)) != CFMM_OK) return rc;
    }
  }
  return CFMM_OK;
}

// ---- pool membership after finalize: append, retire / restore, read back, compact ----------
namespace {

// Retire (active[j] == 0) or restore the pools [first, first + count) of one set.  Only pools
// whose flag changes are touched; *changed counts them.
int set_active_set(cfmm_ctx* ctx, int type, PoolSet& s, int64_t first, int64_t count, const uint8_t* active,
                   int64_t* changed) {
  ensure_pos_of(s);
  if (s.retired.empty()) s.retired.assign((size_t)s.m, 0);
  std::vector<int64_t> pos[2];
  for (int64_t j = 0; j < count; ++j) {
    const int want = active[j] ? 1 : 0;
    if (want != (s.retired[(size_t)(first + j)] ? 0 : 1)) pos[want].push_back(s.pos_of[(size_t)(first + j)]);
  }
  *changed = (int64_t)(pos[0].size() + pos[1].size());
  if (*changed == 0) return CFMM_OK;
  const bool two_coin = type != CFMM_POOL_UNIV3;
  if (!s.d_active.n) {
    CU_TRY(ctx, s.d_active.alloc((size_t)s.m_padded));
    CU_TRY(ctx, cudaMemsetAsync(s.d_active.p, 1, (size_t)s.m_padded, ctx->stream));
    if (two_coin) CU_TRY(ctx, s.d_park.alloc((size_t)s.m_padded));
  }
  const int threads = 256;
  for (int flag : {0, 1}) {
    const int64_t n = (int64_t)pos[flag].size();
    if (n == 0) continue;
    DevBuf<int64_t> d_pos;
    CU_TRY(ctx, d_pos.upload(pos[flag]));
    cfmm::set_active_kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, ctx->stream>>>(
        two_coin ? s.d_R.p : nullptr, s.d_park.p, s.d_active.p, d_pos.p, n, flag);
    ctx->launches++;
    CU_TRY(ctx, cudaGetLastError());
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  for (int64_t j = 0; j < count; ++j) s.retired[(size_t)(first + j)] = active[j] ? 0 : 1;
  if (!two_coin) {  // tick records of the changed pools: zero liquidity while retired (univ3_state.cuh)
    std::vector<int64_t> all(pos[0]);
    all.insert(all.end(), pos[1].begin(), pos[1].end());
    std::sort(all.begin(), all.end());
    return univ3_update_listed(ctx, s, all, nullptr, nullptr, false);
  }
  return s.tma_ok ? refresh_scale(ctx, s) : CFMM_OK;
}

// After a new layout of s is uploaded (every pool active on the device), retire again the pools
// s.retired lists.
int reapply_retired(cfmm_ctx* ctx, int type, PoolSet& s) {
  if (s.retired.empty()) return CFMM_OK;
  std::vector<uint8_t> active((size_t)s.m);
  for (int64_t i = 0; i < s.m; ++i) active[(size_t)i] = s.retired[(size_t)i] ? 0 : 1;
  s.retired.clear();
  int64_t changed = 0;
  return set_active_set(ctx, type, s, 0, s.m, active.data(), &changed);
}

// Append the current state of every pool of src, in src's insertion order, to the host staging of
// dst (and its retired flags): what cfmm_add_* would have staged for a pool set built afresh from
// the device state.  Retired two-coin pools give their parked reserves.
int read_back(cfmm_ctx* ctx, int type, PoolSet& src, PoolSet& dst) {
  const int64_t m = src.m, mp = src.m_padded;
  if (m == 0) return CFMM_OK;
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  auto d2h = [](void* dst_p, const void* src_p, size_t bytes) {
    return cudaMemcpy(dst_p, src_p, bytes, cudaMemcpyDeviceToHost);
  };
  std::vector<double> gam((size_t)mp);
  std::vector<int2> ai((size_t)mp);
  std::vector<int64_t> gidx((size_t)mp);
  CU_TRY(ctx, d2h(gam.data(), src.d_gam.p, (size_t)mp * sizeof(double)));
  CU_TRY(ctx, d2h(ai.data(), src.d_Ai.p, (size_t)mp * sizeof(int2)));
  CU_TRY(ctx, d2h(gidx.data(), src.d_gidx.p, (size_t)mp * sizeof(int64_t)));
  std::vector<double2> R, park, w, f1;
  std::vector<int2> tick;
  std::vector<double> lower, liq;
  if (type != CFMM_POOL_UNIV3) {
    R.resize((size_t)mp);
    CU_TRY(ctx, d2h(R.data(), src.d_R.p, (size_t)mp * sizeof(double2)));
    if (src.d_park.n) {
      park.resize((size_t)mp);
      CU_TRY(ctx, d2h(park.data(), src.d_park.p, (size_t)mp * sizeof(double2)));
    }
  }
  if (type == CFMM_POOL_GEOMEAN) {
    w.resize((size_t)mp);
    CU_TRY(ctx, d2h(w.data(), src.d_w.p, (size_t)mp * sizeof(double2)));
  }
  if (type == CFMM_POOL_UNIV3) {
    f1.resize((size_t)m);
    tick.resize((size_t)m);
    lower.resize((size_t)src.total_ticks);
    liq.resize((size_t)src.total_ticks);
    CU_TRY(ctx, d2h(f1.data(), src.d_first[1].p, (size_t)m * sizeof(double2)));
    CU_TRY(ctx, d2h(tick.data(), src.d_tick.p, (size_t)m * sizeof(int2)));
    CU_TRY(ctx, d2h(lower.data(), src.d_lower.p, lower.size() * sizeof(double)));
    CU_TRY(ctx, d2h(liq.data(), src.d_liq.p, liq.size() * sizeof(double)));
  }
  const size_t b = (size_t)dst.m, n = b + (size_t)m;
  dst.gamma.resize(n);
  dst.Ai.resize(2 * n);
  dst.gidx.resize(n);
  if (type != CFMM_POOL_UNIV3) dst.R.resize(2 * n);
  if (type == CFMM_POOL_GEOMEAN) dst.w.resize(2 * n);
  if (type == CFMM_POOL_UNIV3) dst.cp.resize(n);
  if (!src.retired.empty() || !dst.retired.empty()) {
    dst.retired.resize(n, 0);
    if (!src.retired.empty()) std::copy(src.retired.begin(), src.retired.end(), dst.retired.begin() + b);
  }
  for (int64_t p = 0; p < mp; ++p) {
    const int64_t i = src.order[(size_t)p];
    if (i < 0) continue;  // padding
    const size_t k = b + (size_t)i;
    const bool sw = (gidx[(size_t)p] >> 62) & 1;
    const int64_t ta = ai[(size_t)p].x + 1, tb = ai[(size_t)p].y + 1;
    dst.gamma[k] = gam[(size_t)p];
    dst.Ai[2 * k] = sw ? tb : ta;
    dst.Ai[2 * k + 1] = sw ? ta : tb;
    dst.gidx[k] = gidx[(size_t)p] & ~(1ll << 62);
    if (type != CFMM_POOL_UNIV3) {
      const bool parked = !park.empty() && !src.retired.empty() && src.retired[(size_t)i];
      const double2 r = parked ? park[(size_t)p] : R[(size_t)p];
      dst.R[2 * k] = sw ? r.y : r.x;
      dst.R[2 * k + 1] = sw ? r.x : r.y;
    }
    if (type == CFMM_POOL_GEOMEAN) {
      dst.w[2 * k] = w[(size_t)p].x;
      dst.w[2 * k + 1] = w[(size_t)p].y;
    }
    if (type == CFMM_POOL_UNIV3) dst.cp[k] = f1[(size_t)p].y;
  }
  if (type == CFMM_POOL_UNIV3) {  // tick CSR in insertion order
    ensure_pos_of(src);
    if (dst.tick_off.empty()) dst.tick_off.push_back(0);
    for (int64_t i = 0; i < m; ++i) {
      const int64_t off = tick[(size_t)src.pos_of[(size_t)i]].x, nt = src.n_ticks[(size_t)i];
      dst.lower.insert(dst.lower.end(), lower.begin() + off, lower.begin() + off + nt);
      dst.liq.insert(dst.liq.end(), liq.begin() + off, liq.begin() + off + nt);
      dst.tick_off.push_back((int64_t)dst.lower.size());
    }
  }
  dst.m += m;
  return CFMM_OK;
}

// Lay out the staged pools of `next` where `live` was, retire again what was retired, and swap
// the new set in (the old one is released).
int install_set(cfmm_ctx* ctx, int type, PoolSet& live, PoolSet& next, bool tail) {
  ctx->pairs.built = false;  // device positions change
  int rc = upload_set(ctx, type, next, tail);
  if (rc == CFMM_OK) rc = reapply_retired(ctx, type, next);
  if (rc != CFMM_OK) {
    next.release();
    return rc;
  }
  std::swap(live, next);
  next.release();
  return CFMM_OK;
}

// cfmm_append_*: a new tail of one type = the current tail (its device state) + the new pools,
// staged by `stage` after the arguments were checked.  O(tail), never touches the main set.
int append_to_tail(cfmm_ctx* ctx, int type, const std::function<void(PoolSet&)>& stage) {
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  int rc = use_stream(ctx, ctx->stream);
  if (rc != CFMM_OK) return rc;
  PoolSet& tail = ctx->tails[type];
  auto next = std::make_unique<PoolSet>();
  if ((rc = read_back(ctx, type, tail, *next)) != CFMM_OK) return rc;
  stage(*next);
  if (!next->retired.empty()) next->retired.resize((size_t)next->m, 0);
  if ((rc = install_set(ctx, type, tail, *next, true)) != CFMM_OK) return rc;
  membership_changed(ctx);
  return CFMM_OK;
}

int check_type(cfmm_ctx* ctx, int type) {
  if (type != CFMM_POOL_PRODUCT && type != CFMM_POOL_GEOMEAN && type != CFMM_POOL_UNIV3)
    return fail(ctx, CFMM_ERR_INVALID, "unknown pool type %d", type);
  return CFMM_OK;
}

int check_range(cfmm_ctx* ctx, int type, int64_t first, int64_t count, const char* what) {
  const int64_t m = type_pools(ctx, type);
  if (first < 0 || count < 0 || first + count > m)
    return fail(ctx, CFMM_ERR_INVALID, "%s: range [%lld, %lld) outside 0..%lld", what, (long long)first,
                (long long)(first + count), (long long)m);
  return CFMM_OK;
}

}  // namespace

int cfmm_append_product(cfmm_ctx* ctx, int64_t m, const double* R, const double* gamma, const int64_t* Ai) {
  int rc = check_common(ctx, m, R, gamma, Ai, true);
  if (rc != CFMM_OK || m == 0) return rc;
  return append_to_tail(ctx, CFMM_POOL_PRODUCT, [&](PoolSet& s) { append_common(ctx, s, m, R, gamma, Ai); });
}

int cfmm_append_geomean(cfmm_ctx* ctx, int64_t m, const double* R, const double* gamma, const int64_t* Ai,
                        const double* w) {
  int rc = check_common(ctx, m, R, gamma, Ai, true);
  if (rc != CFMM_OK) return rc;
  if (m > 0 && !w) return fail(ctx, CFMM_ERR_INVALID, "null weight array");
  if (m == 0) return CFMM_OK;
  return append_to_tail(ctx, CFMM_POOL_GEOMEAN, [&](PoolSet& s) {
    append_common(ctx, s, m, R, gamma, Ai);
    s.w.insert(s.w.end(), w, w + 2 * m);
  });
}

int cfmm_append_univ3(cfmm_ctx* ctx, int64_t m, const double* current_price, const double* gamma,
                      const int64_t* Ai, const int64_t* tick_off, const double* lower_ticks,
                      const double* liquidity) {
  static const double dummy = 0.0;
  int rc = check_common(ctx, m, m > 0 ? &dummy : nullptr, gamma, Ai, true);
  if (rc != CFMM_OK || m == 0) return rc;
  PoolSet& tail = ctx->tails[CFMM_POOL_UNIV3];
  if ((rc = check_univ3(ctx, m, current_price, tick_off, lower_ticks, liquidity, tail.total_ticks)) != CFMM_OK)
    return rc;
  return append_to_tail(ctx, CFMM_POOL_UNIV3, [&](PoolSet& s) {
    stage_univ3(ctx, s, m, current_price, gamma, Ai, tick_off, lower_ticks, liquidity);
  });
}

int cfmm_set_active(cfmm_ctx* ctx, int type, int64_t first, int64_t count, const uint8_t* active) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if ((rc = check_range(ctx, type, first, count, "set_active")) != CFMM_OK) return rc;
  if (count == 0) return CFMM_OK;
  if (!active) return fail(ctx, CFMM_ERR_INVALID, "null active array");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  int64_t changed = 0;
  for (const Span& sp : split_range(ctx, type, first, count)) {
    int64_t c = 0;
    rc = set_active_set(ctx, type, *sp.s, sp.first, sp.count, active + sp.offset, &c);
    changed += c;
    if (rc != CFMM_OK) break;
  }
  if (changed > 0) membership_changed(ctx);
  return rc;
}

int cfmm_get_pool_state(cfmm_ctx* ctx, int type, int64_t first, int64_t count, double* state, uint8_t* active) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if ((rc = check_range(ctx, type, first, count, "get_pool_state")) != CFMM_OK) return rc;
  if (count == 0) return CFMM_OK;
  if (!state) return fail(ctx, CFMM_ERR_INVALID, "null state array");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  const int width = type == CFMM_POOL_UNIV3 ? 1 : 2;
  for (const Span& sp : split_range(ctx, type, first, count)) {
    PoolSet& s = *sp.s;
    ensure_pos_of(s);
    std::vector<int64_t> pos(s.pos_of.begin() + sp.first, s.pos_of.begin() + sp.first + sp.count);
    DevBuf<int64_t> d_pos;
    DevBuf<double> d_out;
    CU_TRY(ctx, d_pos.upload(pos));
    CU_TRY(ctx, d_out.alloc((size_t)(width * sp.count)));
    const int threads = 256;
    if ((rc = launch(ctx, kNoProf, 1, [&] {
           cfmm::gather_state_kernel<<<(unsigned)((sp.count + threads - 1) / threads), threads, 0, ctx->stream>>>(
               s.d_R.p, s.d_park.p, s.d_active.p, type == CFMM_POOL_UNIV3 ? s.d_first[1].p : nullptr, s.d_gidx.p,
               d_pos.p, sp.count, d_out.p);
         })) != CFMM_OK)
      return rc;
    CU_TRY(ctx, read_back(ctx, state + width * sp.offset, d_out.p, (size_t)(width * sp.count)));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    if (active)
      for (int64_t j = 0; j < sp.count; ++j)
        active[sp.offset + j] = (s.retired.empty() || !s.retired[(size_t)(sp.first + j)]) ? 1 : 0;
  }
  return CFMM_OK;
}

// ---- swaps: quotes and in-order execution (swap_kernels.cuh) ----------------------------
namespace {

// Every argument of cfmm_quote_swaps / cfmm_execute_swaps, checked on the host before any launch.
int check_swaps(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const double* tender,
                const double* received, bool need_received, const char* what) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative row count", what);
  if (q > 0 && (!pool || !tender || (need_received && !received)))
    return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  const int64_t m = type_pools(ctx, type);
  for (int64_t j = 0; j < q; ++j) {
    if (pool[j] < 0 || pool[j] >= m)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: pool %lld outside 0..%lld", what, (long long)j,
                  (long long)pool[j], (long long)m);
    const double x1 = tender[2 * j], x2 = tender[2 * j + 1];
    if (!std::isfinite(x1) || !std::isfinite(x2) || x1 < 0.0 || x2 < 0.0)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: tender (%g, %g) must be finite and >= 0", what,
                  (long long)j, x1, x2);
    if (x1 > 0.0 && x2 > 0.0)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: tender (%g, %g) has both sides > 0", what, (long long)j,
                  x1, x2);
  }
  return CFMM_OK;
}

cfmm::SwapSet swap_set(PoolSet& s) {
  cfmm::SwapSet w;
  w.R = s.d_R.p;
  w.gam = s.d_gam.p;
  w.w = s.d_w.p;
  w.gidx = s.d_gidx.p;
  w.active = s.d_active.p;
  w.u = univ3_state(s);
  return w;
}

// The rows of one call that fall in one set (main or tail): row index and device position.
struct SetRows {
  PoolSet* s;
  std::vector<int64_t> row, pos;
};

std::vector<SetRows> rows_by_set(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool) {
  std::vector<SetRows> out{{&ctx->sets[type], {}, {}}, {&ctx->tails[type], {}, {}}};
  const int64_t m_main = ctx->sets[type].m;
  for (SetRows& r : out) ensure_pos_of(*r.s);
  for (int64_t j = 0; j < q; ++j) {
    SetRows& r = out[pool[j] < m_main ? 0 : 1];
    r.row.push_back(j);
    r.pos.push_back(r.s->pos_of[(size_t)(pool[j] < m_main ? pool[j] : pool[j] - m_main)]);
  }
  return out;
}

// A stable group by key: key[g] is the g-th distinct key (ascending), rows[off[g] .. off[g+1]) the
// values of its entries in batch order: val[j] for entry j (j itself when val is null).  Keys lie in
// -1 .. n_keys - 1, and every entry of key -1 is a group of its own.  A counting sort on the key
// when the batch is large against the key range, a stable comparison sort otherwise.
struct Groups {
  std::vector<int64_t> key, off, rows;
};

Groups group_by_key(const std::vector<int64_t>& key, int64_t n_keys, const std::vector<int64_t>* val = nullptr) {
  const int64_t n = (int64_t)key.size();
  const auto value = [&](int64_t j) { return val ? (*val)[(size_t)j] : j; };
  Groups g;
  g.rows.resize((size_t)n);
  if (n * 8 >= n_keys) {
    // slot s = key + 1; start[s + 1] counts the slot's entries, then start[s] is its first row
    std::vector<int64_t> start((size_t)n_keys + 2, 0);
    for (int64_t j = 0; j < n; ++j) start[(size_t)(key[(size_t)j] + 2)]++;
    for (int64_t s = 0; s <= n_keys; ++s) {
      const int64_t c = start[(size_t)s + 1];
      for (int64_t i = 0; i < c; i += s == 0 ? 1 : c) {
        g.key.push_back(s - 1);
        g.off.push_back(start[(size_t)s] + i);
      }
      start[(size_t)s + 1] += start[(size_t)s];
    }
    for (int64_t j = 0; j < n; ++j) g.rows[(size_t)start[(size_t)(key[(size_t)j] + 1)]++] = value(j);
  } else {
    std::vector<int64_t> idx((size_t)n);
    std::iota(idx.begin(), idx.end(), (int64_t)0);
    std::stable_sort(idx.begin(), idx.end(), [&](int64_t a, int64_t b) { return key[(size_t)a] < key[(size_t)b]; });
    for (int64_t j = 0; j < n; ++j) {
      const int64_t k = key[(size_t)idx[(size_t)j]];
      if (j == 0 || k < 0 || k != g.key.back()) {
        g.key.push_back(k);
        g.off.push_back(j);
      }
      g.rows[(size_t)j] = value(idx[(size_t)j]);
    }
  }
  g.off.push_back(n);
  return g;
}

// The rows of one set grouped by pool: key[g] is the g-th touched device position, rows the call's
// row indices.
Groups group_by_pool(const SetRows& r, int64_t m_padded) { return group_by_key(r.pos, m_padded, &r.row); }

// After an execute kernel on set s: the derived state of the UniV3 pools it listed in d_moved
// (d_n_moved of them) is rebuilt as after cfmm_apply_trades; for two-coin sets a raised d_flag
// (a reserve left the guard-free range) clears in_fast_range, and the fixed-point scale follows.
int swap_bookkeeping(cfmm_ctx* ctx, PoolSet& s, int type, const int64_t* d_moved,
                     const unsigned long long* d_n_moved, const int* d_flag) {
  int rc = CFMM_OK;
  unsigned long long h_moved = 0;
  int h_flag = 0;
  CU_TRY(ctx, read_back(ctx, &h_moved, d_n_moved, 1));
  CU_TRY(ctx, read_back(ctx, &h_flag, d_flag, 1));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (type == CFMM_POOL_UNIV3) {
    if (h_moved > 0) {  // the derived state of the pools that moved, as after cfmm_apply_trades
      std::vector<int64_t> moved((size_t)h_moved);
      CU_TRY(ctx, cudaMemcpy(moved.data(), d_moved, (size_t)h_moved * sizeof(int64_t), cudaMemcpyDeviceToHost));
      std::sort(moved.begin(), moved.end());
      moved.erase(std::unique(moved.begin(), moved.end()), moved.end());  // (a pool crossed by several paths)
      if ((rc = univ3_update_listed(ctx, s, moved, nullptr, nullptr, true)) != CFMM_OK) return rc;
    }
  } else {
    if (h_flag) s.in_fast_range = false;  // later sweeps take the generic (guarded) form
    if (s.tma_ok && (rc = refresh_scale(ctx, s)) != CFMM_OK) return rc;
  }
  return CFMM_OK;
}

// The kinds, amounts and limits of order rows (noun: "row" or "path"); amount and limit may be null
// (amounts checked elsewhere; no limits).
int check_order_row(cfmm_ctx* ctx, const char* what, const char* noun, int64_t j, const uint8_t* kind,
                    const double* amount, const double* limit) {
  if (kind[j] != CFMM_SWAP_EXACT_IN && kind[j] != CFMM_SWAP_EXACT_OUT)
    return fail(ctx, CFMM_ERR_INVALID, "%s: %s %lld: kind %d is neither exact-in (0) nor exact-out (1)", what, noun,
                (long long)j, (int)kind[j]);
  if (amount && (!std::isfinite(amount[j]) || amount[j] < 0.0))
    return fail(ctx, CFMM_ERR_INVALID, "%s: %s %lld: amount %g must be finite and >= 0", what, noun, (long long)j,
                amount[j]);
  if (!limit) return CFMM_OK;
  if (std::isnan(limit[j]) || limit[j] < 0.0)
    return fail(ctx, CFMM_ERR_INVALID, "%s: %s %lld: limit %g must be >= 0", what, noun, (long long)j, limit[j]);
  if (std::isinf(limit[j]) && kind[j] == CFMM_SWAP_EXACT_IN)
    return fail(ctx, CFMM_ERR_INVALID, "%s: %s %lld: an exact-in %s's minimum received must be finite", what, noun,
                (long long)j, noun);
  return CFMM_OK;
}

extern "C++" {  // (templates, inside the file's extern "C" block)

// Launch the swap kernel of the given pool type on `blocks` blocks of 256 threads: kernel(T) is its
// instantiation for pool type T (a std::integral_constant).
template <class Kernel, class... Args>
void swap_launch(int type, Kernel kernel, unsigned blocks, cudaStream_t st, Args... args) {
  const auto k = type == CFMM_POOL_PRODUCT   ? kernel(std::integral_constant<int, 0>{})
                 : type == CFMM_POOL_GEOMEAN ? kernel(std::integral_constant<int, 1>{})
                                             : kernel(std::integral_constant<int, 2>{});
  k<<<blocks, 256, 0, st>>>(args...);
}

// cfmm_quote_swaps and cfmm_quote_swaps_exact_out: rows (pool, in [2]) priced on the current state on
// their own, out [2] per row; one launch per set.
template <class Kernel>
int quote_swap_rows(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const double* in, double* out,
                    Kernel kernel) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  DevBuf<double> d_in, d_out;
  CU_TRY(ctx, d_in.upload(in, (size_t)(2 * q)));
  CU_TRY(ctx, d_out.alloc((size_t)(2 * q)));
  for (SetRows& r : rows_by_set(ctx, type, q, pool)) {
    const int64_t n = (int64_t)r.row.size();
    if (n == 0) continue;
    DevBuf<int64_t> d_row, d_pos;
    CU_TRY(ctx, d_row.upload(r.row));
    CU_TRY(ctx, d_pos.upload(r.pos));
    const cfmm::SwapSet ss = swap_set(*r.s);
    if ((rc = launch(ctx, kProfSwaps, 1, [&] {
           swap_launch(type, kernel, (unsigned)((n + 255) / 256), ctx->stream, ss, d_row.p, d_pos.p, n, d_in.p,
                       d_out.p);
         })) != CFMM_OK)
      return rc;
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // (d_row, d_pos are freed at the end of the block)
  }
  CU_TRY(ctx, read_back(ctx, out, d_out.p, (size_t)(2 * q)));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

// cfmm_execute_swaps and cfmm_execute_swap_orders: per set, the rows grouped by pool (a thread per
// touched pool runs its rows in batch order), one launch with the row arrays `rows`, then
// swap_bookkeeping.
template <class Kernel, class... Rows>
int execute_swap_rows(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, Kernel kernel, Rows... rows) {
  int rc;
  for (SetRows& r : rows_by_set(ctx, type, q, pool)) {
    PoolSet& s = *r.s;
    if (r.row.empty()) continue;
    const Groups seg = group_by_pool(r, s.m_padded);
    const int64_t n_seg = (int64_t)seg.key.size();
    DevBuf<int64_t> d_seg_pos, d_seg_off, d_seg_rows, d_moved;
    DevBuf<unsigned long long> d_n_moved;
    DevBuf<int> d_flag;
    CU_TRY(ctx, d_seg_pos.upload(seg.key));
    CU_TRY(ctx, d_seg_off.upload(seg.off));
    CU_TRY(ctx, d_seg_rows.upload(seg.rows));
    CU_TRY(ctx, d_n_moved.alloc(1));
    CU_TRY(ctx, d_flag.alloc(1));
    if (type == CFMM_POOL_UNIV3) CU_TRY(ctx, d_moved.alloc((size_t)n_seg));
    CU_TRY(ctx, cudaMemsetAsync(d_n_moved.p, 0, sizeof(unsigned long long), ctx->stream));
    CU_TRY(ctx, cudaMemsetAsync(d_flag.p, 0, sizeof(int), ctx->stream));
    const cfmm::SwapSet ss = swap_set(s);
    if ((rc = launch(ctx, kProfSwaps, 1, [&] {
           swap_launch(type, kernel, (unsigned)((n_seg + 255) / 256), ctx->stream, ss, d_seg_pos.p, d_seg_off.p,
                       d_seg_rows.p, n_seg, rows..., d_moved.p, d_n_moved.p, d_flag.p);
         })) != CFMM_OK)
      return rc;
    if ((rc = swap_bookkeeping(ctx, s, type, d_moved.p, d_n_moved.p, d_flag.p)) != CFMM_OK) return rc;
  }
  return CFMM_OK;
}

}  // extern "C++"

}  // namespace

int cfmm_quote_swaps(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const double* tender,
                     double* received) {
  int rc = check_swaps(ctx, type, q, pool, tender, received, true, "quote_swaps");
  if (rc != CFMM_OK || q == 0) return rc;
  return quote_swap_rows(ctx, type, q, pool, tender, received,
                         [](auto t) { return cfmm::swap_quote_kernel<decltype(t)::value>; });
}

int cfmm_quote_swaps_exact_out(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const double* want,
                               double* tender) {
  int rc = check_swaps(ctx, type, q, pool, want, tender, true, "quote_swaps_exact_out");
  if (rc != CFMM_OK || q == 0) return rc;
  return quote_swap_rows(ctx, type, q, pool, want, tender,
                         [](auto t) { return cfmm::swap_quote_exact_out_kernel<decltype(t)::value>; });
}

int cfmm_execute_swaps(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const double* tender,
                       double* received) {
  int rc = check_swaps(ctx, type, q, pool, tender, received, false, "execute_swaps");
  if (rc != CFMM_OK || q == 0) return rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  ctx->state_version++;
  DevBuf<double> d_tender, d_recv;
  CU_TRY(ctx, d_tender.upload(tender, (size_t)(2 * q)));
  CU_TRY(ctx, d_recv.alloc((size_t)(2 * q)));
  if ((rc = execute_swap_rows(ctx, type, q, pool,
                              [](auto t) { return cfmm::swap_execute_kernel<decltype(t)::value>; }, d_tender.p,
                              d_recv.p)) != CFMM_OK)
    return rc;
  CU_TRY(ctx, read_back(ctx, received, d_recv.p, (size_t)(2 * q)));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

// ---- exact-output rows and slippage limits (swap_kernels.cuh) -----------------------------------
namespace {

// The kinds and limits of cfmm_execute_swap_orders (the amounts are checked by check_swaps).
int check_orders(cfmm_ctx* ctx, int64_t q, const uint8_t* kind, const double* limit) {
  if (q > 0 && !kind) return fail(ctx, CFMM_ERR_INVALID, "execute_swap_orders: null kind array");
  for (int64_t j = 0; j < q; ++j) {
    const int rc = check_order_row(ctx, "execute_swap_orders", "row", j, kind, nullptr, limit);
    if (rc != CFMM_OK) return rc;
  }
  return CFMM_OK;
}

}  // namespace

int cfmm_execute_swap_orders(cfmm_ctx* ctx, int type, int64_t q, const int64_t* pool, const uint8_t* kind,
                             const double* amount, const double* limit, double* paid, double* received,
                             uint8_t* status) {
  int rc = check_swaps(ctx, type, q, pool, amount, nullptr, false, "execute_swap_orders");
  if (rc != CFMM_OK) return rc;
  if ((rc = check_orders(ctx, q, kind, limit)) != CFMM_OK || q == 0) return rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  ctx->state_version++;
  DevBuf<double> d_amount, d_limit, d_paid, d_recv;
  DevBuf<uint8_t> d_kind, d_status;
  CU_TRY(ctx, d_amount.upload(amount, (size_t)(2 * q)));
  CU_TRY(ctx, d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, d_limit.upload(limit, (size_t)q));
  CU_TRY(ctx, d_paid.alloc((size_t)(2 * q)));
  CU_TRY(ctx, d_recv.alloc((size_t)(2 * q)));
  CU_TRY(ctx, d_status.alloc((size_t)q));
  if ((rc = execute_swap_rows(ctx, type, q, pool,
                              [](auto t) { return cfmm::swap_execute_orders_kernel<decltype(t)::value>; },
                              d_kind.p, d_amount.p, d_limit.p, d_paid.p, d_recv.p, d_status.p)) != CFMM_OK)
    return rc;
  CU_TRY(ctx, read_back(ctx, paid, d_paid.p, (size_t)(2 * q)));
  CU_TRY(ctx, read_back(ctx, received, d_recv.p, (size_t)(2 * q)));
  CU_TRY(ctx, read_back(ctx, status, d_status.p, (size_t)q));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

// ---- multi-hop swap paths (path_kernels.cuh) ---------------------------------------------------
namespace {

// Set k of the path kernels: 2·type, + 1 for the type's appended pools.
PoolSet& path_set(cfmm_ctx* ctx, int k) { return (k & 1) ? ctx->tails[k >> 1] : ctx->sets[k >> 1]; }

// Every host-side argument of cfmm_quote_paths / cfmm_execute_paths, checked before any launch
// (the token walk is checked on the device, path_check_kernel).
int check_paths(cfmm_ctx* ctx, int64_t q, const int64_t* hop_off, const int* hop_type, const int64_t* hop_pool,
                const int64_t* token_in, const uint8_t* kind, const double* amount, const double* limit,
                const char* what) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative path count", what);
  if (q == 0) return CFMM_OK;
  if (!hop_off || !hop_type || !hop_pool || !token_in || !kind || !amount)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  if (hop_off[0] != 0) return fail(ctx, CFMM_ERR_INVALID, "%s: hop_off[0] must be 0", what);
  for (int64_t j = 0; j < q; ++j) {
    const int64_t n = hop_off[j + 1] - hop_off[j];
    if (n < 1 || n > CFMM_PATH_MAX_HOPS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld has %lld hops (hop_off must rise by 1..%d per path)", what,
                  (long long)j, (long long)n, CFMM_PATH_MAX_HOPS);
  }
  for (int64_t j = 0; j < q; ++j) {
    for (int64_t h = hop_off[j]; h < hop_off[j + 1]; ++h) {
      const int t = hop_type[h];
      if (t != CFMM_POOL_PRODUCT && t != CFMM_POOL_GEOMEAN && t != CFMM_POOL_UNIV3)
        return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld hop %lld: unknown pool type %d", what, (long long)j,
                    (long long)(h - hop_off[j]), t);
      if (hop_pool[h] < 0 || hop_pool[h] >= type_pools(ctx, t))
        return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld hop %lld: pool %lld outside 0..%lld", what, (long long)j,
                    (long long)(h - hop_off[j]), (long long)hop_pool[h], (long long)type_pools(ctx, t));
      for (int64_t g = hop_off[j]; g < h; ++g)
        if (hop_type[g] == t && hop_pool[g] == hop_pool[h])
          return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld: hops %lld and %lld are the same pool", what, (long long)j,
                      (long long)(g - hop_off[j]), (long long)(h - hop_off[j]));
    }
    if (token_in[j] < 1 || token_in[j] > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld: token_in %lld outside 1..%lld", what, (long long)j,
                  (long long)token_in[j], (long long)ctx->n_tokens);
    if ((rc = check_order_row(ctx, what, "path", j, kind, amount, limit)) != CFMM_OK) return rc;
  }
  return CFMM_OK;
}

// The pool sets the path and order kernels see (on the device), and on execute the flags they
// raise: out_of_range [6], touched [6], and per UniV3 set the moved list.  The order kernels list a
// pool once (listed flags; the lists hold m_padded entries), the path kernels once per hop that
// crossed it (moved_len: the lists' lengths, no listed flags).
struct OrderSets {
  cfmm::PathSets P{};
  cfmm::SplitMoved mv{};
  DevBuf<int> flags;
  DevBuf<unsigned long long> n_moved;
  DevBuf<int64_t> moved[2];
  DevBuf<uint8_t> listed[2];
  DevBuf<cfmm::PathSets> d_P;
};

int order_sets(cfmm_ctx* ctx, bool exec, OrderSets& os, const int64_t* moved_len = nullptr) {
  cfmm::PathSets& P = os.P;
  for (int k = 0; k < cfmm::kPathSets; ++k) {
    PoolSet& s = path_set(ctx, k);
    P.s[k] = swap_set(s);
    P.Ai[k] = s.d_Ai.p;
  }
  if (exec) {
    CU_TRY(ctx, os.flags.alloc(2 * cfmm::kPathSets));
    CU_TRY(ctx, os.n_moved.alloc(2));
    CU_TRY(ctx, cudaMemsetAsync(os.flags.p, 0, 2 * cfmm::kPathSets * sizeof(int), ctx->stream));
    CU_TRY(ctx, cudaMemsetAsync(os.n_moved.p, 0, 2 * sizeof(unsigned long long), ctx->stream));
    for (int u = 0; u < 2; ++u) {
      if (moved_len) {
        CU_TRY(ctx, os.moved[u].alloc((size_t)moved_len[u]));
      } else {
        const size_t m = (size_t)path_set(ctx, 2 * CFMM_POOL_UNIV3 + u).m_padded;
        CU_TRY(ctx, os.moved[u].alloc(m));
        CU_TRY(ctx, os.listed[u].alloc(m));
        if (m) CU_TRY(ctx, cudaMemsetAsync(os.listed[u].p, 0, m, ctx->stream));
        os.mv.flag[u] = os.listed[u].p;
      }
      P.moved[u] = os.moved[u].p;
    }
    P.out_of_range = os.flags.p;
    P.touched = os.flags.p + cfmm::kPathSets;
    P.n_moved = os.n_moved.p;
  }
  CU_TRY(ctx, os.d_P.upload(&P, 1));
  return CFMM_OK;
}

// After an execute: the bookkeeping of cfmm_execute_swaps on every set a filled row touched.
int order_bookkeeping(cfmm_ctx* ctx, OrderSets& os) {
  int rc;
  int touched[cfmm::kPathSets];
  CU_TRY(ctx, read_back(ctx, touched, os.P.touched, cfmm::kPathSets));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < cfmm::kPathSets; ++k) {
    if (!touched[k]) continue;
    const int t = k >> 1;
    if ((rc = swap_bookkeeping(ctx, path_set(ctx, k), t, t == CFMM_POOL_UNIV3 ? os.moved[k & 1].p : nullptr,
                               os.n_moved.p + (k & 1), os.flags.p + k)) != CFMM_OK)
      return rc;
  }
  return CFMM_OK;
}

// One path call on the device: the hops resolved to (set, device position) as rows_by_set
// resolves rows, the path arrays, the pool sets and the per-hop outputs.
struct PathCall {
  int64_t q = 0, H = 0;
  std::vector<uint8_t> set;
  std::vector<int64_t> pos;
  DevBuf<int64_t> d_off, d_pos, d_token;
  DevBuf<uint8_t> d_set, d_tok1, d_kind, d_status;
  DevBuf<double> d_amount, d_tender, d_recv;
  OrderSets os;
};

// Upload a checked call, walk its tokens on the device (path_check_kernel) and reject it, before
// anything is written, when some hop's pool does not hold the token that reaches it.
int path_prepare(cfmm_ctx* ctx, PathCall& c, bool exec, int64_t q, const int64_t* hop_off, const int* hop_type,
                 const int64_t* hop_pool, const int64_t* token_in, const uint8_t* kind, const double* amount,
                 const char* what) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  c.q = q;
  c.H = hop_off[q];
  for (int k = 0; k < cfmm::kPathSets; ++k) ensure_pos_of(path_set(ctx, k));
  c.set.resize((size_t)c.H);
  c.pos.resize((size_t)c.H);
  int64_t univ3_hops[2] = {0, 0};
  for (int64_t h = 0; h < c.H; ++h) {
    const int t = hop_type[h];
    const int64_t m_main = ctx->sets[t].m;
    const bool tail = hop_pool[h] >= m_main;
    c.set[(size_t)h] = (uint8_t)(2 * t + (tail ? 1 : 0));
    c.pos[(size_t)h] = path_set(ctx, 2 * t + (tail ? 1 : 0)).pos_of[(size_t)(tail ? hop_pool[h] - m_main : hop_pool[h])];
    if (t == CFMM_POOL_UNIV3) univ3_hops[tail ? 1 : 0]++;
  }
  CU_TRY(ctx, c.d_off.upload(hop_off, (size_t)q + 1));
  CU_TRY(ctx, c.d_token.upload(token_in, (size_t)q));
  CU_TRY(ctx, c.d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, c.d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, c.d_set.upload(c.set));
  CU_TRY(ctx, c.d_pos.upload(c.pos));
  CU_TRY(ctx, c.d_tok1.alloc((size_t)c.H));
  CU_TRY(ctx, c.d_tender.alloc((size_t)c.H));
  CU_TRY(ctx, c.d_recv.alloc((size_t)c.H));
  CU_TRY(ctx, c.d_status.alloc((size_t)q));
  if ((rc = order_sets(ctx, exec, c.os, univ3_hops)) != CFMM_OK) return rc;
  DevBuf<unsigned long long> d_bad;
  CU_TRY(ctx, d_bad.alloc(1));
  CU_TRY(ctx, cudaMemsetAsync(d_bad.p, 0xff, sizeof(unsigned long long), ctx->stream));
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::path_check_kernel<<<(unsigned)((q + 255) / 256), 256, 0, ctx->stream>>>(
             c.os.d_P.p, q, c.d_off.p, c.d_set.p, c.d_pos.p, c.d_token.p, c.d_tok1.p, d_bad.p);
       })) != CFMM_OK)
    return rc;
  unsigned long long bad = 0;
  CU_TRY(ctx, read_back(ctx, &bad, d_bad.p, 1));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (bad != ~0ull) {
    const int64_t j = (int64_t)(std::upper_bound(hop_off, hop_off + q + 1, (int64_t)bad) - hop_off) - 1;
    int64_t t = token_in[j];
    for (int64_t h = hop_off[j]; h < (int64_t)bad; ++h) {  // the token that reached the bad hop
      int2 ai;
      CU_TRY(ctx, cudaMemcpy(&ai, path_set(ctx, c.set[(size_t)h]).d_Ai.p + c.pos[(size_t)h], sizeof(int2),
                             cudaMemcpyDeviceToHost));
      t = (t - 1 == ai.x ? ai.y : ai.x) + 1;
    }
    return fail(ctx, CFMM_ERR_INVALID, "%s: path %lld hop %lld: pool %lld of type %d does not hold token %lld", what,
                (long long)j, (long long)(bad - hop_off[j]), (long long)hop_pool[bad], hop_type[bad], (long long)t);
  }
  return CFMM_OK;
}

int path_outputs(cfmm_ctx* ctx, const PathCall& c, double* hop_tender, double* hop_received, uint8_t* status) {
  CU_TRY(ctx, read_back(ctx, hop_tender, c.d_tender.p, (size_t)c.H));
  CU_TRY(ctx, read_back(ctx, hop_received, c.d_recv.p, (size_t)c.H));
  CU_TRY(ctx, read_back(ctx, status, c.d_status.p, (size_t)c.q));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

// The last level a resource of one table was given in this call (0 = none yet): a dense array when
// the call's uses of the table are many against its size, a hash otherwise (group_by_key's rule).
struct LevelTable {
  std::vector<int> dense;
  std::unordered_map<int64_t, int> sparse;
  int& at(int64_t p) { return dense.empty() ? sparse[p] : dense[(size_t)p]; }
};

// Execution order of the execute calls that run conflicting rows apart (paths, routed orders): row
// j's level is 1 + the largest level of an earlier row sharing one of its resources, so the rows of
// one level touch disjoint resources and every resource sees its rows in batch order.  A resource is
// an index into one of the tables (size[k] entries, uses[k] of them named by the call);
// for_each(j, visit) calls visit(k, index) on every resource of row j.  order: the rows sorted stably
// by (level, batch index); the rows of level L (1-based) are order[level_off[L-1] .. level_off[L]).
extern "C++" template <class ForEach>
void conflict_levels(int64_t q, int n_tables, const int64_t* size, const int64_t* uses, ForEach for_each,
                     std::vector<int64_t>& order, std::vector<int64_t>& level_off) {
  std::vector<LevelTable> tab((size_t)n_tables);
  for (int k = 0; k < n_tables; ++k) {
    if (uses[k] > 0 && uses[k] * 8 >= size[k])
      tab[(size_t)k].dense.assign((size_t)size[k], 0);
    else
      tab[(size_t)k].sparse.reserve((size_t)uses[k]);
  }
  std::vector<int> lev((size_t)q);
  int n_levels = 0;
  for (int64_t j = 0; j < q; ++j) {
    int L = 0;
    for_each(j, [&](int k, int64_t p) { L = std::max(L, tab[(size_t)k].at(p)); });
    ++L;
    for_each(j, [&](int k, int64_t p) { tab[(size_t)k].at(p) = L; });
    lev[(size_t)j] = L;
    n_levels = std::max(n_levels, L);
  }
  level_off.assign((size_t)n_levels + 1, 0);
  for (int64_t j = 0; j < q; ++j) level_off[(size_t)lev[(size_t)j]]++;
  for (int L = 1; L <= n_levels; ++L) level_off[(size_t)L] += level_off[(size_t)L - 1];
  std::vector<int64_t> next(level_off.begin(), level_off.end() - 1);
  order.resize((size_t)q);
  for (int64_t j = 0; j < q; ++j) order[(size_t)next[(size_t)lev[(size_t)j] - 1]++] = j;
}

}  // namespace

int cfmm_quote_paths(cfmm_ctx* ctx, int64_t q, const int64_t* hop_off, const int* hop_type, const int64_t* hop_pool,
                     const int64_t* token_in, const uint8_t* kind, const double* amount, double* hop_tender,
                     double* hop_received, uint8_t* status) {
  int rc = check_paths(ctx, q, hop_off, hop_type, hop_pool, token_in, kind, amount, nullptr, "quote_paths");
  if (rc != CFMM_OK || q == 0) return rc;
  if (!hop_tender || !hop_received || !status) return fail(ctx, CFMM_ERR_INVALID, "quote_paths: null array argument");
  PathCall c;
  if ((rc = path_prepare(ctx, c, false, q, hop_off, hop_type, hop_pool, token_in, kind, amount, "quote_paths")) !=
      CFMM_OK)
    return rc;
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::path_quote_kernel<<<(unsigned)((q + 255) / 256), 256, 0, ctx->stream>>>(
             c.os.d_P.p, q, c.d_off.p, c.d_set.p, c.d_pos.p, c.d_tok1.p, c.d_kind.p, c.d_amount.p, c.d_tender.p,
             c.d_recv.p, c.d_status.p);
       })) != CFMM_OK)
    return rc;
  return path_outputs(ctx, c, hop_tender, hop_received, status);
}

int cfmm_execute_paths(cfmm_ctx* ctx, int64_t q, const int64_t* hop_off, const int* hop_type, const int64_t* hop_pool,
                       const int64_t* token_in, const uint8_t* kind, const double* amount, const double* limit,
                       double* hop_tender, double* hop_received, uint8_t* status) {
  int rc = check_paths(ctx, q, hop_off, hop_type, hop_pool, token_in, kind, amount, limit, "execute_paths");
  if (rc != CFMM_OK || q == 0) return rc;
  PathCall c;
  if ((rc = path_prepare(ctx, c, true, q, hop_off, hop_type, hop_pool, token_in, kind, amount, "execute_paths")) !=
      CFMM_OK)
    return rc;
  ctx->state_version++;
  DevBuf<double> d_limit;
  CU_TRY(ctx, d_limit.upload(limit, (size_t)q));
  // levels over the hops' pools: one table per set
  int64_t size[cfmm::kPathSets], uses[cfmm::kPathSets] = {};
  for (int k = 0; k < cfmm::kPathSets; ++k) size[k] = path_set(ctx, k).m_padded;
  for (int64_t h = 0; h < c.H; ++h) uses[c.set[(size_t)h]]++;
  std::vector<int64_t> order, level_off;
  conflict_levels(
      q, cfmm::kPathSets, size, uses,
      [&](int64_t j, auto&& visit) {
        for (int64_t h = hop_off[j]; h < hop_off[j + 1]; ++h) visit(c.set[(size_t)h], c.pos[(size_t)h]);
      },
      order, level_off);
  DevBuf<int64_t> d_order;
  CU_TRY(ctx, d_order.upload(order));
  for (size_t L = 1; L < level_off.size(); ++L) {
    const int64_t n = level_off[L] - level_off[L - 1];
    if ((rc = launch(ctx, kProfSwaps, 1, [&] {
           cfmm::path_execute_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
               c.os.d_P.p, d_order.p + level_off[L - 1], n, c.d_off.p, c.d_set.p, c.d_pos.p, c.d_tok1.p, c.d_kind.p,
               c.d_amount.p, d_limit.p, c.d_tender.p, c.d_recv.p, c.d_status.p);
         })) != CFMM_OK)
      return rc;
  }
  if ((rc = order_bookkeeping(ctx, c.os)) != CFMM_OK) return rc;
  return path_outputs(ctx, c, hop_tender, hop_received, status);
}

// ---- orders split across the pools of their token pair (split_kernels.cuh) --------------------
namespace {

// The pair index on the device: keys per pool in global insertion order (pair_key_kernel), a stable
// radix sort, a run-length pass and the CSR offsets.  Kept until the pools move.
int ensure_pair_index(cfmm_ctx* ctx) {
  auto& ix = ctx->pairs;
  if (ix.built) return CFMM_OK;
  const int64_t n = ctx->n_pools, nt = ctx->n_tokens;
  if (n > INT32_MAX) return fail(ctx, CFMM_ERR_INVALID, "pair index: more than 2^31 - 1 pools");
  ix.adj_built = false;
  ix.adj_off.release();
  ix.adj_nbr.release();
  ix.adj_pair.release();
  ix.adj_off_host.clear();
  ix.keys.release();
  ix.off.release();
  ix.pool.release();
  ix.n_pairs = 0;
  if (n > 0) {
    cudaStream_t st = ctx->stream;
    DevBuf<int64_t> keys_in, ent_in, keys_sorted, run_len;
    DevBuf<int> d_runs;
    DevBuf<unsigned char> temp;
    CU_TRY(ctx, keys_in.alloc((size_t)n));
    CU_TRY(ctx, ent_in.alloc((size_t)n));
    CU_TRY(ctx, keys_sorted.alloc((size_t)n));
    CU_TRY(ctx, run_len.alloc((size_t)n + 1));
    CU_TRY(ctx, d_runs.alloc(1));
    CU_TRY(ctx, ix.pool.alloc((size_t)n));
    CU_TRY(ctx, ix.keys.alloc((size_t)n));
    CU_TRY(ctx, ix.off.alloc((size_t)n + 1));
    int end_bit = 1;  // keys < n_tokens²
    while (end_bit < 63 && (1ll << end_bit) < nt * nt) ++end_bit;
    const int items = (int)n;
    size_t b1 = 0, b2 = 0, b3 = 0;
    CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, b1, keys_in.p, keys_sorted.p, ent_in.p, ix.pool.p, items, 0,
                                                end_bit, st));
    CU_TRY(ctx, cub::DeviceRunLengthEncode::Encode(nullptr, b2, keys_sorted.p, ix.keys.p, run_len.p, d_runs.p, items, st));
    CU_TRY(ctx, cub::DeviceScan::ExclusiveSum(nullptr, b3, run_len.p, ix.off.p, items + 1, st));
    CU_TRY(ctx, temp.alloc(std::max(b1, std::max(b2, b3))));
    int n_sets = 0;
    for (int k = 0; k < cfmm::kPathSets; ++k) n_sets += path_set(ctx, k).m > 0;
    int rc = launch(ctx, kProfSwaps, n_sets + 3, [&]() -> int {
      for (int k = 0; k < cfmm::kPathSets; ++k) {
        PoolSet& s = path_set(ctx, k);
        if (s.m == 0) continue;
        cfmm::pair_key_kernel<<<(unsigned)((s.m_padded + 255) / 256), 256, 0, st>>>(s.d_Ai.p, s.d_gidx.p, s.m_padded, k,
                                                                                   nt, keys_in.p, ent_in.p);
      }
      size_t bytes = temp.n;
      CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(temp.p, bytes, keys_in.p, keys_sorted.p, ent_in.p, ix.pool.p, items, 0,
                                                  end_bit, st));
      CU_TRY(ctx, cudaMemsetAsync(run_len.p, 0, ((size_t)n + 1) * sizeof(int64_t), st));
      bytes = temp.n;
      CU_TRY(ctx, cub::DeviceRunLengthEncode::Encode(temp.p, bytes, keys_sorted.p, ix.keys.p, run_len.p, d_runs.p, items,
                                                     st));
      bytes = temp.n;
      CU_TRY(ctx, cub::DeviceScan::ExclusiveSum(temp.p, bytes, run_len.p, ix.off.p, items + 1, st));
      return CFMM_OK;
    });
    if (rc != CFMM_OK) return rc;
    int runs = 0;
    CU_TRY(ctx, read_back(ctx, &runs, d_runs.p, 1));
    CU_TRY(ctx, cudaStreamSynchronize(st));
    ix.n_pairs = runs;
  }
  ix.built = true;
  return CFMM_OK;
}

// Tokens of rows naming a pair: 1-based, in range, distinct.
int check_pair_tokens(cfmm_ctx* ctx, int64_t q, const int64_t* a, const int64_t* b, const char* what) {
  for (int64_t j = 0; j < q; ++j) {
    if (a[j] < 1 || a[j] > ctx->n_tokens || b[j] < 1 || b[j] > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: tokens (%lld, %lld) outside 1..%lld", what, (long long)j,
                  (long long)a[j], (long long)b[j], (long long)ctx->n_tokens);
    if (a[j] == b[j])
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: the two tokens are both %lld", what, (long long)j,
                  (long long)a[j]);
  }
  return CFMM_OK;
}

// The rows' pairs on the device (index into the pair index, -1 = none) and their pool counts on
// the host; the tokens are uploaded to d_a / d_b.
int pair_lookup(cfmm_ctx* ctx, int64_t q, const int64_t* a, const int64_t* b, DevBuf<int64_t>& d_a,
                DevBuf<int64_t>& d_b, DevBuf<int64_t>& d_pair, std::vector<int64_t>& count) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  if ((rc = ensure_pair_index(ctx)) != CFMM_OK) return rc;
  DevBuf<int64_t> d_count;
  CU_TRY(ctx, d_a.upload(a, (size_t)q));
  CU_TRY(ctx, d_b.upload(b, (size_t)q));
  CU_TRY(ctx, d_pair.alloc((size_t)q));
  CU_TRY(ctx, d_count.alloc((size_t)q));
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::pair_lookup_kernel<<<(unsigned)((q + 255) / 256), 256, 0, ctx->stream>>>(
             ctx->pairs.keys.p, ctx->pairs.n_pairs, ctx->pairs.off.p, d_a.p, d_b.p, q, ctx->n_tokens, d_pair.p,
             d_count.p);
       })) != CFMM_OK)
    return rc;
  count.resize((size_t)q);
  CU_TRY(ctx, read_back(ctx, count.data(), d_count.p, (size_t)q));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

// Every argument of cfmm_quote_split_orders / cfmm_execute_split_orders, before anything runs.
int check_split(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const uint8_t* kind,
                const double* amount, const double* limit, const char* what) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative row count", what);
  if (q == 0) return CFMM_OK;
  if (!token_in || !token_out || !kind || !amount) return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  if ((rc = check_pair_tokens(ctx, q, token_in, token_out, what)) != CFMM_OK) return rc;
  for (int64_t j = 0; j < q; ++j)
    if ((rc = check_order_row(ctx, what, "row", j, kind, amount, limit)) != CFMM_OK) return rc;
  return CFMM_OK;
}

// One split, routed or arbitrage call on the device: the rows' pair lists looked up in the pair
// index (d_a, d_b, d_pair; one list per split row), the legs of every list (leg_off), the row
// arrays, the per-row outputs and the pool sets.  On execute, pair holds the lists' pairs on the
// host.
struct OrderCall {
  int64_t q = 0, L = 0;
  bool legs = false;  // leg outputs asked for, and some list has a pool
  std::vector<int64_t> pair;
  DevBuf<int64_t> d_a, d_b, d_pair, d_leg_off;
  DevBuf<uint8_t> d_kind, d_status;
  DevBuf<double> d_amount, d_limit, d_paid, d_recv, d_price, d_ld, d_ll;
  OrderSets os;
};

// kind and amount are null for arbitrage rows, limit when there are no limits.
int order_prepare(cfmm_ctx* ctx, OrderCall& c, bool exec, int64_t q, int64_t n_lists, const int64_t* a,
                  const int64_t* b, const uint8_t* kind, const double* amount, const double* limit, bool legs) {
  int rc;
  std::vector<int64_t> count;
  if ((rc = pair_lookup(ctx, n_lists, a, b, c.d_a, c.d_b, c.d_pair, count)) != CFMM_OK) return rc;
  std::vector<int64_t> leg_off((size_t)n_lists + 1, 0);
  for (int64_t j = 0; j < n_lists; ++j) leg_off[(size_t)j + 1] = leg_off[(size_t)j] + count[(size_t)j];
  c.q = q;
  c.L = leg_off[(size_t)n_lists];
  c.legs = legs && c.L > 0;
  CU_TRY(ctx, c.d_leg_off.upload(leg_off));
  CU_TRY(ctx, c.d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, c.d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, c.d_limit.upload(limit, (size_t)q));
  CU_TRY(ctx, c.d_paid.alloc((size_t)q));
  CU_TRY(ctx, c.d_recv.alloc((size_t)q));
  CU_TRY(ctx, c.d_price.alloc((size_t)q));
  CU_TRY(ctx, c.d_status.alloc((size_t)q));
  if (c.legs) {
    CU_TRY(ctx, c.d_ld.alloc((size_t)(2 * c.L)));
    CU_TRY(ctx, c.d_ll.alloc((size_t)(2 * c.L)));
  }
  if ((rc = order_sets(ctx, exec, c.os)) != CFMM_OK) return rc;
  if (exec) {
    ctx->state_version++;
    c.pair.resize((size_t)n_lists);
    CU_TRY(ctx, read_back(ctx, c.pair.data(), c.d_pair.p, (size_t)n_lists));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return CFMM_OK;
}

int order_outputs(cfmm_ctx* ctx, const OrderCall& c, double* paid, double* received, double* price, uint8_t* status,
                  double* leg_delta, double* leg_lambda) {
  CU_TRY(ctx, read_back(ctx, paid, c.d_paid.p, (size_t)c.q));
  CU_TRY(ctx, read_back(ctx, received, c.d_recv.p, (size_t)c.q));
  CU_TRY(ctx, read_back(ctx, price, c.d_price.p, (size_t)c.q));
  CU_TRY(ctx, read_back(ctx, status, c.d_status.p, (size_t)c.q));
  if (c.legs) {
    CU_TRY(ctx, read_back(ctx, leg_delta, c.d_ld.p, (size_t)(2 * c.L)));
    CU_TRY(ctx, read_back(ctx, leg_lambda, c.d_ll.p, (size_t)(2 * c.L)));
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

int split_orders(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_in, const int64_t* token_out,
                 const uint8_t* kind, const double* amount, const double* limit, double* paid, double* received,
                 double* price, uint8_t* status, double* leg_delta, double* leg_lambda) {
  int rc;
  OrderCall c;
  if ((rc = order_prepare(ctx, c, exec, q, q, token_in, token_out, kind, amount, limit, leg_delta || leg_lambda)) !=
      CFMM_OK)
    return rc;
  cfmm::SplitRows R{c.d_a.p,    c.d_b.p,    c.d_kind.p,  c.d_amount.p, c.d_limit.p, c.d_pair.p, c.d_leg_off.p,
                    c.d_paid.p, c.d_recv.p, c.d_price.p, c.d_status.p, c.d_ld.p,    c.d_ll.p};
  const cfmm::PairIndexView ix{ctx->pairs.off.p, ctx->pairs.pool.p};
  const int per_block = cfmm::kSplitThreads / 32;  // a warp per row (quote) or per pair (execute)
  if (!exec) {
    rc = launch(ctx, kProfSwaps, 1, [&] {
      cfmm::split_quote_kernel<<<(unsigned)((q + per_block - 1) / per_block), cfmm::kSplitThreads, 0, ctx->stream>>>(
          c.os.d_P.p, ix, R, q);
    });
    if (rc != CFMM_OK) return rc;
  } else {
    // the rows grouped by pair, batch order kept inside each pair; a row whose pair no pool holds is a
    // group of its own
    const Groups seg = group_by_key(c.pair, ctx->pairs.n_pairs);
    const int64_t n_seg = (int64_t)seg.key.size();
    DevBuf<int64_t> d_seg_off, d_seg_rows;
    CU_TRY(ctx, d_seg_off.upload(seg.off));
    CU_TRY(ctx, d_seg_rows.upload(seg.rows));
    rc = launch(ctx, kProfSwaps, 1, [&] {
      cfmm::split_execute_kernel<<<(unsigned)((n_seg + per_block - 1) / per_block), cfmm::kSplitThreads, 0,
                                   ctx->stream>>>(c.os.d_P.p, ix, R, d_seg_off.p, d_seg_rows.p, n_seg, c.os.mv);
    });
    if (rc != CFMM_OK) return rc;
    if ((rc = order_bookkeeping(ctx, c.os)) != CFMM_OK) return rc;
  }
  return order_outputs(ctx, c, paid, received, price, status, leg_delta, leg_lambda);
}

// ---- orders routed over their pair and two-hop routes through hubs (route_kernels.cuh) ----------

// Every argument of cfmm_quote_routed_orders / cfmm_execute_routed_orders, before anything runs.
int check_hubs(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const int64_t* hub_off,
               const int64_t* hubs, const char* what);

int check_routed(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const uint8_t* kind,
                 const double* amount, const double* limit, const int64_t* hub_off, const int64_t* hubs,
                 const char* what) {
  int rc = check_split(ctx, q, token_in, token_out, kind, amount, limit, what);
  if (rc != CFMM_OK || q == 0) return rc;
  return check_hubs(ctx, q, token_in, token_out, hub_off, hubs, what);
}

// Every argument of cfmm_quote_arbitrage / cfmm_execute_arbitrage: routed rows' tokens and hubs, and
// min_profit (NULL: 0) neither NaN, negative nor +inf (an exact-in row's minimum received).
int check_arbitrage(cfmm_ctx* ctx, int64_t q, const int64_t* base, const int64_t* other, const double* min_profit,
                    const int64_t* hub_off, const int64_t* hubs, const char* what) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative row count", what);
  if (q == 0) return CFMM_OK;
  if (!base || !other) return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  if ((rc = check_pair_tokens(ctx, q, other, base, what)) != CFMM_OK) return rc;
  for (int64_t r = 0; min_profit && r < q; ++r)
    if (!(min_profit[r] >= 0.0) || std::isinf(min_profit[r]))
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: min_profit %g must be finite and >= 0", what, (long long)r,
                  min_profit[r]);
  return check_hubs(ctx, q, other, base, hub_off, hubs, what);
}

// Routed and arbitrage rows' hub lists.
int check_hubs(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const int64_t* hub_off,
               const int64_t* hubs, const char* what) {
  if (!hub_off) return fail(ctx, CFMM_ERR_INVALID, "%s: null hub_off", what);
  if (hub_off[0] != 0) return fail(ctx, CFMM_ERR_INVALID, "%s: hub_off[0] = %lld, not 0", what, (long long)hub_off[0]);
  for (int64_t r = 0; r < q; ++r) {
    const int64_t c = hub_off[r + 1] - hub_off[r];
    if (c < 0 || c > CFMM_ROUTE_MAX_HUBS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld hubs, not 0..%d", what, (long long)r, (long long)c,
                  CFMM_ROUTE_MAX_HUBS);
  }
  if (hub_off[q] > 0 && !hubs) return fail(ctx, CFMM_ERR_INVALID, "%s: null hubs", what);
  for (int64_t r = 0; r < q; ++r) {
    for (int64_t g = hub_off[r]; g < hub_off[r + 1]; ++g) {
      const int64_t h = hubs[g];
      if (h < 1 || h > ctx->n_tokens)
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: hub %lld outside 1..%lld", what, (long long)r, (long long)h,
                    (long long)ctx->n_tokens);
      if (h == token_in[r] || h == token_out[r])
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: hub %lld is one of the row's tokens", what, (long long)r,
                    (long long)h);
      for (int64_t f = hub_off[r]; f < g; ++f)
        if (hubs[f] == h)
          return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: hub %lld listed twice", what, (long long)r, (long long)h);
    }
  }
  return CFMM_OK;
}

// Routed rows, or with arb arbitrage rows (token_in = the other token, token_out = the base token,
// kind and amount null, limit = min_profit, paid = the surplus of the other token, received = profit).
int routed_orders(cfmm_ctx* ctx, bool exec, bool arb, int64_t q, const int64_t* token_in, const int64_t* token_out,
                  const uint8_t* kind, const double* amount, const double* limit, const int64_t* hub_off,
                  const int64_t* hubs, double* paid, double* received, double* price, uint8_t* status,
                  double* hub_price, double* hub_surplus, double* leg_delta, double* leg_lambda) {
  int rc;
  const int64_t nh = hub_off[q];
  // the rows' pair lists: (j, i), then (j, h), (h, i) per hub; row r's start at r + 2·hub_off[r]
  const int64_t n_lists = q + 2 * nh;
  std::vector<int64_t> la((size_t)n_lists), lb((size_t)n_lists);
  int max_hubs = 0;
  for (int64_t r = 0; r < q; ++r) {
    const int64_t base = r + 2 * hub_off[r];
    la[(size_t)base] = token_in[r];
    lb[(size_t)base] = token_out[r];
    for (int64_t g = hub_off[r]; g < hub_off[r + 1]; ++g) {
      const int64_t x = base + 1 + 2 * (g - hub_off[r]);
      la[(size_t)x] = token_in[r];
      lb[(size_t)x] = hubs[g];
      la[(size_t)x + 1] = hubs[g];
      lb[(size_t)x + 1] = token_out[r];
    }
    max_hubs = std::max(max_hubs, (int)(hub_off[r + 1] - hub_off[r]));
  }
  OrderCall c;
  if ((rc = order_prepare(ctx, c, exec, q, n_lists, la.data(), lb.data(), kind, amount, limit,
                          leg_delta || leg_lambda)) != CFMM_OK)
    return rc;
  DevBuf<int64_t> d_in, d_out, d_hub_off, d_hubs;
  DevBuf<double> d_hp, d_hs;
  CU_TRY(ctx, d_in.upload(token_in, (size_t)q));
  CU_TRY(ctx, d_out.upload(token_out, (size_t)q));
  CU_TRY(ctx, d_hub_off.upload(hub_off, (size_t)q + 1));
  CU_TRY(ctx, d_hubs.upload(hubs, (size_t)nh));
  CU_TRY(ctx, d_hp.alloc((size_t)nh));
  CU_TRY(ctx, d_hs.alloc((size_t)nh));
  cfmm::RouteRows R{d_in.p,     d_out.p,    c.d_kind.p,  c.d_amount.p, c.d_limit.p, d_hub_off.p,
                    d_hubs.p,   c.d_pair.p, c.d_leg_off.p, c.d_paid.p, c.d_recv.p,  c.d_price.p,
                    c.d_status.p, d_hp.p,   d_hs.p,      c.d_ld.p,     c.d_ll.p};
  const cfmm::PairIndexView ix{ctx->pairs.off.p, ctx->pairs.pool.p};
  const unsigned threads = 32u * (1u + (unsigned)max_hubs);  // warp 0: the direct pools, warp 1 + h: hub h
  if (!exec) {
    rc = launch(ctx, kProfSwaps, 1, [&] {
      if (arb)
        cfmm::arb_quote_kernel<<<(unsigned)q, threads, 0, ctx->stream>>>(c.os.d_P.p, ix, R);
      else
        cfmm::route_quote_kernel<<<(unsigned)q, threads, 0, ctx->stream>>>(c.os.d_P.p, ix, R);
    });
    if (rc != CFMM_OK) return rc;
  } else {
    // levels over the rows' pairs (a pool belongs to one pair); pairs no pool holds conflict with
    // nothing
    const int64_t n_pairs = ctx->pairs.n_pairs;
    std::vector<int64_t> order, level_off;
    conflict_levels(
        q, 1, &n_pairs, &n_lists,
        [&](int64_t r, auto&& visit) {
          for (int64_t x = r + 2 * hub_off[r]; x < r + 1 + 2 * hub_off[r + 1]; ++x)
            if (c.pair[(size_t)x] >= 0) visit(0, c.pair[(size_t)x]);
        },
        order, level_off);
    DevBuf<int64_t> d_rows;
    CU_TRY(ctx, d_rows.upload(order));
    for (size_t l = 1; l < level_off.size(); ++l) {
      const int64_t n = level_off[l] - level_off[l - 1];
      const int64_t* rows = d_rows.p + level_off[l - 1];
      rc = launch(ctx, kProfSwaps, 1, [&] {
        if (arb)
          cfmm::arb_execute_kernel<<<(unsigned)n, threads, 0, ctx->stream>>>(c.os.d_P.p, ix, R, rows, c.os.mv);
        else
          cfmm::route_execute_kernel<<<(unsigned)n, threads, 0, ctx->stream>>>(c.os.d_P.p, ix, R, rows, c.os.mv);
      });
      if (rc != CFMM_OK) return rc;
    }
    if ((rc = order_bookkeeping(ctx, c.os)) != CFMM_OK) return rc;
  }
  CU_TRY(ctx, read_back(ctx, hub_price, d_hp.p, (size_t)nh));
  CU_TRY(ctx, read_back(ctx, hub_surplus, d_hs.p, (size_t)nh));
  return order_outputs(ctx, c, paid, received, price, status, leg_delta, leg_lambda);
}

// ---- arbitrage cycles through base tokens (arb_scan_kernels.cuh) --------------------------------

// Every argument of cfmm_scan_arbitrage, before anything runs.
int check_scan(cfmm_ctx* ctx, int64_t nb, const int64_t* base, const double* min_profit, int max_hubs, int64_t cap,
               const int64_t* found, const int64_t* row_base, const int64_t* row_other, const int64_t* hub_count,
               const int64_t* hubs, const double* profit, const double* price) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (nb < 0) return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: negative base count");
  if (cap < 0) return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: negative cap");
  if (!found) return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: null found");
  if (max_hubs < 0 || max_hubs > CFMM_ROUTE_MAX_HUBS)
    return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: max_hubs %d, not 0..%d", max_hubs, CFMM_ROUTE_MAX_HUBS);
  if (cap > 0 && (!row_base || !row_other || !hub_count || !hubs || !profit || !price))
    return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: null output with cap > 0");
  if (nb == 0) return CFMM_OK;
  if (!base || !min_profit) return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: null array argument");
  for (int64_t b = 0; b < nb; ++b) {
    if (base[b] < 1 || base[b] > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: base %lld: token %lld outside 1..%lld", (long long)b,
                  (long long)base[b], (long long)ctx->n_tokens);
    if (!(min_profit[b] > 0.0) || std::isinf(min_profit[b]))
      return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: base %lld: min_profit %g must be finite and > 0",
                  (long long)b, min_profit[b]);
  }
  std::vector<int64_t> sorted(base, base + nb);
  std::sort(sorted.begin(), sorted.end());
  for (int64_t b = 1; b < nb; ++b)
    if (sorted[(size_t)b] == sorted[(size_t)b - 1])
      return fail(ctx, CFMM_ERR_INVALID, "scan_arbitrage: base token %lld listed twice", (long long)sorted[(size_t)b]);
  return CFMM_OK;
}

// The token adjacency (arb_scan_kernels.cuh), built from the pair index's keys and kept with it.
int ensure_adjacency(cfmm_ctx* ctx) {
  int rc;
  if ((rc = ensure_pair_index(ctx)) != CFMM_OK) return rc;
  auto& ix = ctx->pairs;
  if (ix.adj_built) return CFMM_OK;
  const int64_t nt = ctx->n_tokens, np = ix.n_pairs, m = 2 * np;
  if (nt >= INT32_MAX || m > INT32_MAX)
    return fail(ctx, CFMM_ERR_INVALID, "token adjacency: more than 2^31 - 1 tokens or entries");
  cudaStream_t st = ctx->stream;
  CU_TRY(ctx, ix.adj_off.alloc((size_t)nt + 1));
  CU_TRY(ctx, ix.adj_nbr.alloc((size_t)m));
  CU_TRY(ctx, ix.adj_pair.alloc((size_t)m));
  DevBuf<int64_t> kin, kout;
  DevBuf<int32_t> vin;
  DevBuf<unsigned char> temp;
  size_t bytes = 0;
  int end_bit = 1;  // keys < n_tokens²
  while (end_bit < 63 && (1ll << end_bit) < nt * nt) ++end_bit;
  if (m > 0) {
    CU_TRY(ctx, kin.alloc((size_t)m));
    CU_TRY(ctx, kout.alloc((size_t)m));
    CU_TRY(ctx, vin.alloc((size_t)m));
    CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin.p, kout.p, vin.p, ix.adj_pair.p, (int)m, 0, end_bit,
                                                st));
    CU_TRY(ctx, temp.alloc(bytes));
  }
  int rc2 = launch(ctx, kProfSwaps, m > 0 ? 3 : 1, [&]() -> int {
    if (m > 0) {
      cfmm::adj_entries_kernel<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(ix.keys.p, np, nt, kin.p, vin.p);
      CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(temp.p, bytes, kin.p, kout.p, vin.p, ix.adj_pair.p, (int)m, 0,
                                                  end_bit, st));
    }
    const int64_t th = std::max(m, nt + 1);
    cfmm::adj_finish_kernel<<<(unsigned)((th + 255) / 256), 256, 0, st>>>(kout.p, m, nt, ix.adj_nbr.p, ix.adj_off.p);
    return CFMM_OK;
  });
  if (rc2 != CFMM_OK) return rc2;
  ix.adj_off_host.resize((size_t)nt + 1);
  CU_TRY(ctx, read_back(ctx, ix.adj_off_host.data(), ix.adj_off.p, (size_t)nt + 1));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  ix.adj_built = true;
  return CFMM_OK;
}

int scan_arbitrage(cfmm_ctx* ctx, int64_t nb, const int64_t* base, const double* min_profit, int max_hubs, int64_t cap,
                   int64_t* found, int64_t* row_base, int64_t* row_other, int64_t* hub_count, int64_t* hubs,
                   double* profit, double* price) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  if ((rc = ensure_adjacency(ctx)) != CFMM_OK) return rc;
  auto& ix = ctx->pairs;
  cudaStream_t st = ctx->stream;
  const int64_t np = ix.n_pairs;
  // slots: (base b, its e-th neighbour), base after base
  std::vector<int64_t> slot_off((size_t)nb + 1, 0);
  for (int64_t b = 0; b < nb; ++b)
    slot_off[(size_t)b + 1] =
        slot_off[(size_t)b] + ix.adj_off_host[(size_t)base[b]] - ix.adj_off_host[(size_t)base[b] - 1];
  const int64_t ns = slot_off[(size_t)nb];
  if (ns == 0) return CFMM_OK;
  DevBuf<unsigned char> temp;
  const auto cub_scan = [&](const int64_t* in, int64_t* out, int64_t n) {
    size_t b = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, b, in, out, (int)n, st);
    if (e == cudaSuccess && b > temp.n) e = temp.alloc(b);
    return e == cudaSuccess ? cub::DeviceScan::ExclusiveSum(temp.p, b, in, out, (int)n, st) : e;
  };
  const auto blocks = [](int64_t threads) { return (unsigned)((threads + 255) / 256); };
  OrderSets os;
  if ((rc = order_sets(ctx, false, os)) != CFMM_OK) return rc;
  // rates
  DevBuf<long long> rate;
  CU_TRY(ctx, rate.alloc((size_t)(2 * np)));
  CU_TRY(ctx, cudaMemsetAsync(rate.p, 0, (size_t)(2 * np) * sizeof(long long), st));
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::arb_rates_kernel<<<blocks(ctx->n_pools), 256, 0, st>>>(os.d_P.p, ix.off.p, ix.pool.p, ix.keys.p, np,
                                                                      ctx->n_tokens, rate.p);
       })) != CFMM_OK)
    return rc;
  // candidates, one warp per slot, then their rows in slot order
  DevBuf<int64_t> d_base, d_slot_off, flag, nhub, row_pos, hub_pos;
  DevBuf<int32_t> slot_hub, slot_lists;
  DevBuf<double> d_min;
  CU_TRY(ctx, d_base.upload(base, (size_t)nb));
  CU_TRY(ctx, d_min.upload(min_profit, (size_t)nb));
  CU_TRY(ctx, d_slot_off.upload(slot_off));
  CU_TRY(ctx, flag.alloc((size_t)ns + 1));
  CU_TRY(ctx, nhub.alloc((size_t)ns + 1));
  CU_TRY(ctx, row_pos.alloc((size_t)ns + 1));
  CU_TRY(ctx, hub_pos.alloc((size_t)ns + 1));
  CU_TRY(ctx, slot_hub.alloc((size_t)(cfmm::kRouteMaxHubs * ns)));
  CU_TRY(ctx, slot_lists.alloc((size_t)((1 + 2 * cfmm::kRouteMaxHubs) * ns)));
  CU_TRY(ctx, cudaMemsetAsync(flag.p, 0, ((size_t)ns + 1) * sizeof(int64_t), st));
  CU_TRY(ctx, cudaMemsetAsync(nhub.p, 0, ((size_t)ns + 1) * sizeof(int64_t), st));
  const cfmm::AdjView A{ix.adj_off.p, ix.adj_nbr.p, ix.adj_pair.p};
  if ((rc = launch(ctx, kProfSwaps, 3, [&]() -> int {
         cfmm::arb_candidates_kernel<<<blocks(32 * ns), 256, 0, st>>>(A, reinterpret_cast<const double*>(rate.p),
                                                                       d_base.p, d_slot_off.p, nb, max_hubs, flag.p,
                                                                       nhub.p, slot_hub.p, slot_lists.p);
         CU_TRY(ctx, cub_scan(flag.p, row_pos.p, ns + 1));
         CU_TRY(ctx, cub_scan(nhub.p, hub_pos.p, ns + 1));
         return CFMM_OK;
       })) != CFMM_OK)
    return rc;
  int64_t q = 0, nh = 0;
  CU_TRY(ctx, read_back(ctx, &q, row_pos.p + ns, 1));
  CU_TRY(ctx, read_back(ctx, &nh, hub_pos.p + ns, 1));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  if (q == 0) return CFMM_OK;
  DevBuf<int64_t> tin, tout, row_b, hub_off, d_hubs, pair;
  DevBuf<double> surplus, d_profit, d_price;
  DevBuf<uint8_t> status;
  CU_TRY(ctx, tin.alloc((size_t)q));
  CU_TRY(ctx, tout.alloc((size_t)q));
  CU_TRY(ctx, row_b.alloc((size_t)q));
  CU_TRY(ctx, hub_off.alloc((size_t)q + 1));
  CU_TRY(ctx, d_hubs.alloc((size_t)nh));
  CU_TRY(ctx, pair.alloc((size_t)(q + 2 * nh)));
  CU_TRY(ctx, surplus.alloc((size_t)q));
  CU_TRY(ctx, d_profit.alloc((size_t)q));
  CU_TRY(ctx, d_price.alloc((size_t)q));
  CU_TRY(ctx, status.alloc((size_t)q));
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::arb_rows_kernel<<<blocks(ns + 1), 256, 0, st>>>(A, d_base.p, d_slot_off.p, nb, flag.p, nhub.p,
                                                               slot_hub.p, slot_lists.p, row_pos.p, hub_pos.p, tin.p,
                                                               tout.p, row_b.p, hub_off.p, d_hubs.p, pair.p);
       })) != CFMM_OK)
    return rc;
  // solve: every candidate as an arbitrage row on the current state
  const cfmm::PairIndexView pv{ix.off.p, ix.pool.p};
  cfmm::RouteRows R{tin.p,     tout.p,  nullptr,    nullptr,     nullptr, hub_off.p, d_hubs.p, pair.p, nullptr,
                    surplus.p, d_profit.p, d_price.p, status.p, nullptr, nullptr,   nullptr,  nullptr};
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::arb_quote_kernel<<<(unsigned)q, 32u * (1u + (unsigned)max_hubs), 0, st>>>(os.d_P.p, pv, R);
       })) != CFMM_OK)
    return rc;
  // select: filled rows with profit >= their base's minimum, then (base index, profit desc, x asc) by
  // two stable sorts of the (base index, x)-ordered rows: on the complemented profit bits, then the base
  DevBuf<int64_t> keep, keep_pos;
  DevBuf<uint64_t> key;
  CU_TRY(ctx, keep.alloc((size_t)q + 1));
  CU_TRY(ctx, keep_pos.alloc((size_t)q + 1));
  CU_TRY(ctx, key.alloc((size_t)q));
  if ((rc = launch(ctx, kProfSwaps, 2, [&]() -> int {
         cfmm::arb_keep_kernel<<<blocks(q + 1), 256, 0, st>>>(status.p, d_profit.p, row_b.p, d_min.p, q, keep.p,
                                                              key.p);
         CU_TRY(ctx, cub_scan(keep.p, keep_pos.p, q + 1));
         return CFMM_OK;
       })) != CFMM_OK)
    return rc;
  int64_t n_sel = 0;
  CU_TRY(ctx, read_back(ctx, &n_sel, keep_pos.p + q, 1));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  *found = n_sel;
  const int64_t n_out = std::min(n_sel, cap);
  if (n_out == 0) return CFMM_OK;
  DevBuf<int64_t> sel, v1, v2;
  DevBuf<uint64_t> sel_key, key_s;
  DevBuf<uint32_t> b1, b_s;
  CU_TRY(ctx, sel.alloc((size_t)n_sel));
  CU_TRY(ctx, v1.alloc((size_t)n_sel));
  CU_TRY(ctx, v2.alloc((size_t)n_sel));
  CU_TRY(ctx, sel_key.alloc((size_t)n_sel));
  CU_TRY(ctx, key_s.alloc((size_t)n_sel));
  CU_TRY(ctx, b1.alloc((size_t)n_sel));
  CU_TRY(ctx, b_s.alloc((size_t)n_sel));
  int b_bits = 1;
  while (b_bits < 32 && (1ll << b_bits) < nb) ++b_bits;
  size_t s1 = 0, s2 = 0;
  CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, s1, sel_key.p, key_s.p, sel.p, v1.p, (int)n_sel, 0, 64, st));
  CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(nullptr, s2, b1.p, b_s.p, v1.p, v2.p, (int)n_sel, 0, b_bits, st));
  if (std::max(s1, s2) > temp.n) CU_TRY(ctx, temp.alloc(std::max(s1, s2)));
  DevBuf<int64_t> o_base, o_other, o_count, o_hubs;
  DevBuf<double> o_profit, o_price;
  CU_TRY(ctx, o_base.alloc((size_t)n_out));
  CU_TRY(ctx, o_other.alloc((size_t)n_out));
  CU_TRY(ctx, o_count.alloc((size_t)n_out));
  CU_TRY(ctx, o_hubs.alloc((size_t)(cfmm::kRouteMaxHubs * n_out)));
  CU_TRY(ctx, o_profit.alloc((size_t)n_out));
  CU_TRY(ctx, o_price.alloc((size_t)n_out));
  if ((rc = launch(ctx, kProfSwaps, 5, [&]() -> int {
         cfmm::arb_select_kernel<<<blocks(q), 256, 0, st>>>(keep_pos.p, key.p, q, sel.p, sel_key.p);
         s1 = temp.n;
         CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(temp.p, s1, sel_key.p, key_s.p, sel.p, v1.p, (int)n_sel, 0, 64,
                                                     st));
         cfmm::arb_base_key_kernel<<<blocks(n_sel), 256, 0, st>>>(v1.p, n_sel, row_b.p, b1.p);
         s2 = temp.n;
         CU_TRY(ctx, cub::DeviceRadixSort::SortPairs(temp.p, s2, b1.p, b_s.p, v1.p, v2.p, (int)n_sel, 0, b_bits, st));
         cfmm::arb_output_kernel<<<blocks(n_out), 256, 0, st>>>(v2.p, n_out, tin.p, tout.p, hub_off.p, d_hubs.p,
                                                                d_profit.p, d_price.p, o_base.p, o_other.p,
                                                                o_count.p, o_hubs.p, o_profit.p, o_price.p);
         return CFMM_OK;
       })) != CFMM_OK)
    return rc;
  const size_t n = (size_t)n_out;
  CU_TRY(ctx, read_back(ctx, row_base, o_base.p, n));
  CU_TRY(ctx, read_back(ctx, row_other, o_other.p, n));
  CU_TRY(ctx, read_back(ctx, hub_count, o_count.p, n));
  CU_TRY(ctx, read_back(ctx, hubs, o_hubs.p, n * cfmm::kRouteMaxHubs));
  CU_TRY(ctx, read_back(ctx, profit, o_profit.p, n));
  CU_TRY(ctx, read_back(ctx, price, o_price.p, n));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  return CFMM_OK;
}

// ---- hubs chosen for order rows (hub_kernels.cuh) -----------------------------------------------

// Every argument of cfmm_choose_order_hubs, before anything runs: split orders' rows, max_hubs, and
// the two CSR outputs.
int check_choose_hubs(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                      const uint8_t* kind, const double* amount, int max_hubs, const int64_t* hub_off,
                      const int64_t* hubs) {
  int rc = check_split(ctx, q, token_in, token_out, kind, amount, nullptr, "choose_order_hubs");
  if (rc != CFMM_OK) return rc;
  if (max_hubs < 0 || max_hubs > CFMM_ROUTE_MAX_HUBS)
    return fail(ctx, CFMM_ERR_INVALID, "choose_order_hubs: max_hubs %d, not 0..%d", max_hubs, CFMM_ROUTE_MAX_HUBS);
  if (q > 0 && (!hub_off || !hubs)) return fail(ctx, CFMM_ERR_INVALID, "choose_order_hubs: null hub_off or hubs");
  return CFMM_OK;
}

int choose_order_hubs(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                      const uint8_t* kind, const double* amount, int max_hubs, const uint8_t* allowed,
                      int64_t* hub_off, int64_t* hubs, double* hub_score, int64_t* n_eligible) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  if ((rc = ensure_adjacency(ctx)) != CFMM_OK) return rc;
  auto& ix = ctx->pairs;
  cudaStream_t st = ctx->stream;
  OrderSets os;
  if ((rc = order_sets(ctx, false, os)) != CFMM_OK) return rc;
  const size_t slots = (size_t)q * (size_t)max_hubs;
  DevBuf<int64_t> d_in, d_out, d_nhub, d_hub, d_elig;
  DevBuf<uint8_t> d_kind, d_allowed;
  DevBuf<double> d_amount, d_score;
  CU_TRY(ctx, d_in.upload(token_in, (size_t)q));
  CU_TRY(ctx, d_out.upload(token_out, (size_t)q));
  CU_TRY(ctx, d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, d_allowed.upload(allowed, (size_t)ctx->n_tokens));
  CU_TRY(ctx, d_nhub.alloc((size_t)q));
  CU_TRY(ctx, d_elig.alloc((size_t)q));
  CU_TRY(ctx, d_hub.alloc(slots));
  CU_TRY(ctx, d_score.alloc(slots));
  const cfmm::PairIndexView pv{ix.off.p, ix.pool.p};
  const cfmm::AdjView A{ix.adj_off.p, ix.adj_nbr.p, ix.adj_pair.p};
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::hub_choice_kernel<<<(unsigned)((32 * q + 255) / 256), 256, 0, st>>>(
             os.d_P.p, pv, A, d_in.p, d_out.p, d_kind.p, d_amount.p, q, max_hubs, d_allowed.p, d_nhub.p, d_hub.p,
             d_score.p, d_elig.p);
       })) != CFMM_OK)
    return rc;
  std::vector<int64_t> nhub((size_t)q), hub(slots);
  std::vector<double> score(hub_score ? slots : 0);
  CU_TRY(ctx, read_back(ctx, nhub.data(), d_nhub.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, hub.data(), d_hub.p, slots));
  CU_TRY(ctx, read_back(ctx, hub_score ? score.data() : nullptr, d_score.p, slots));
  CU_TRY(ctx, read_back(ctx, n_eligible, d_elig.p, (size_t)q));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  // pack each row's first nhub[r] slots
  hub_off[0] = 0;
  for (int64_t r = 0; r < q; ++r) {
    const int64_t g = hub_off[r];
    for (int64_t h = 0; h < nhub[(size_t)r]; ++h) {
      hubs[g + h] = hub[(size_t)(max_hubs * r + h)];
      if (hub_score) hub_score[g + h] = score[(size_t)(max_hubs * r + h)];
    }
    hub_off[r + 1] = g + nhub[(size_t)r];
  }
  return CFMM_OK;
}

// ---- best paths through allowed tokens (best_path_kernels.cuh) ----------------------------------

// Pool p of path set k as cfmm_pair_pools reports it: its index in its type's insertion order.
int64_t pool_id(cfmm_ctx* ctx, int k, int64_t p) {
  return path_set(ctx, k).order[(size_t)p] + ((k & 1) ? ctx->sets[k >> 1].m : 0);
}

// The walks of a path search, H hop slots per entry (a row, or a requested walk): nhop per entry, and
// per slot the set, device position, tendered side, delivered token (1-based), tender and received.
struct HopSlots {
  int64_t k = 0;
  int H = 0;
  DevBuf<int32_t> nhop;
  DevBuf<uint8_t> set, tok1;
  DevBuf<int64_t> pos, token;
  DevBuf<double> tender, received;

  int alloc(cfmm_ctx* ctx, int64_t entries, int max_hops) {
    k = entries;
    H = max_hops;
    const size_t slots = (size_t)k * (size_t)H;
    CU_TRY(ctx, nhop.alloc((size_t)k));
    CU_TRY(ctx, set.alloc(slots));
    CU_TRY(ctx, pos.alloc(slots));
    CU_TRY(ctx, tok1.alloc(slots));
    CU_TRY(ctx, token.alloc(slots));
    CU_TRY(ctx, tender.alloc(slots));
    CU_TRY(ctx, received.alloc(slots));
    return CFMM_OK;
  }

  // After the launches, with the call's other read-backs enqueued: each entry's first nhop slots as
  // cfmm_execute_paths' CSR, pools as cfmm_pair_pools reports them.  Synchronises the stream.
  int pack(cfmm_ctx* ctx, int64_t* hop_off, int* hop_type, int64_t* hop_pool, int64_t* hop_token, double* hop_tender,
           double* hop_received) {
    const size_t slots = (size_t)k * (size_t)H;
    std::vector<int32_t> n((size_t)k);
    std::vector<uint8_t> s(slots);
    std::vector<int64_t> p(slots), t(slots);
    std::vector<double> x(hop_tender ? slots : 0), y(hop_received ? slots : 0);
    CU_TRY(ctx, read_back(ctx, n.data(), nhop.p, (size_t)k));
    CU_TRY(ctx, read_back(ctx, s.data(), set.p, slots));
    CU_TRY(ctx, read_back(ctx, p.data(), pos.p, slots));
    CU_TRY(ctx, read_back(ctx, t.data(), token.p, slots));
    CU_TRY(ctx, read_back(ctx, hop_tender ? x.data() : nullptr, tender.p, slots));
    CU_TRY(ctx, read_back(ctx, hop_received ? y.data() : nullptr, received.p, slots));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    hop_off[0] = 0;
    for (int64_t e = 0; e < k; ++e) {
      const int64_t g = hop_off[e];
      for (int64_t h = 0; h < n[(size_t)e]; ++h) {
        const size_t w = (size_t)(H * e + h);
        hop_type[g + h] = s[w] >> 1;
        hop_pool[g + h] = pool_id(ctx, s[w], p[w]);
        hop_token[g + h] = t[w];
        if (hop_tender) hop_tender[g + h] = x[w];
        if (hop_received) hop_received[g + h] = y[w];
      }
      hop_off[e + 1] = g + n[(size_t)e];
    }
    return CFMM_OK;
  }
};

// The call's allowed tokens; a row's tokens besides its own are these less the row's own among them.
int64_t count_allowed(const cfmm_ctx* ctx, const uint8_t* allowed) {
  int64_t n = 0;
  for (int64_t t = 0; t < ctx->n_tokens; ++t) n += allowed[t] != 0;
  return n;
}

// Every argument of cfmm_find_order_paths, before anything runs: split orders' rows, max_hops, the
// mask (required) and each row's |B| (the allowed tokens other than its two), and the CSR outputs.
int check_find_paths(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                     const uint8_t* kind, const double* amount, int max_hops, const uint8_t* allowed,
                     const int64_t* hop_off, const int* hop_type, const int64_t* hop_pool, const int64_t* hop_token,
                     const char* what = "find_order_paths") {
  int rc = check_split(ctx, q, token_in, token_out, kind, amount, nullptr, what);
  if (rc != CFMM_OK) return rc;
  if (max_hops < 1 || max_hops > CFMM_PATH_MAX_HOPS)
    return fail(ctx, CFMM_ERR_INVALID, "%s: max_hops %d, not 1..%d", what, max_hops, CFMM_PATH_MAX_HOPS);
  if (!allowed) return fail(ctx, CFMM_ERR_INVALID, "%s: null allowed (the intermediate tokens are required)", what);
  if (q == 0) return CFMM_OK;
  if (!hop_off || !hop_type || !hop_pool || !hop_token)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null hop_off, hop_type, hop_pool or hop_token", what);
  const int64_t n_allowed = count_allowed(ctx, allowed);
  for (int64_t r = 0; r < q; ++r) {
    const int64_t nb = n_allowed - (allowed[token_in[r] - 1] != 0) - (allowed[token_out[r] - 1] != 0);
    if (nb > CFMM_BEST_PATH_MAX_TOKENS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld intermediate tokens, more than %d", what, (long long)r,
                  (long long)nb, CFMM_BEST_PATH_MAX_TOKENS);
  }
  return CFMM_OK;
}

// The per-hop costs of the _net calls: n of them, each >= 0 (+inf allowed), before anything runs.
int check_hop_cost(cfmm_ctx* ctx, const double* hop_cost, int64_t n, const char* what) {
  if (n > 0 && !hop_cost) return fail(ctx, CFMM_ERR_INVALID, "%s: null hop_cost", what);
  for (int64_t k = 0; k < n; ++k)
    if (!(hop_cost[k] >= 0.0))
      return fail(ctx, CFMM_ERR_INVALID, "%s: hop_cost[%lld] %g, not >= 0", what, (long long)k, hop_cost[k]);
  return CFMM_OK;
}

// hop_cost (cfmm_find_order_paths_net): the best filled max_hops = L result net of hop_cost[r] per
// hop, its net into net (NULL: not written); null: cfmm_find_order_paths.
int find_order_paths(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const uint8_t* kind,
                     const double* amount, int max_hops, const uint8_t* allowed, int64_t* hop_off, int* hop_type,
                     int64_t* hop_pool, int64_t* hop_token, double* hop_tender, double* hop_received, double* value,
                     uint8_t* status, const double* hop_cost = nullptr, double* net = nullptr) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  if ((rc = ensure_adjacency(ctx)) != CFMM_OK) return rc;
  auto& ix = ctx->pairs;
  cudaStream_t st = ctx->stream;
  OrderSets os;
  if ((rc = order_sets(ctx, false, os)) != CFMM_OK) return rc;
  // the call's slots: the allowed tokens, ascending
  std::vector<int32_t> tok, slot_of((size_t)ctx->n_tokens, -1);
  for (int64_t t = 0; t < ctx->n_tokens; ++t)
    if (allowed[t]) {
      slot_of[(size_t)t] = (int32_t)tok.size();
      tok.push_back((int32_t)t);
    }
  const int nB = (int)tok.size(), H = max_hops;
  const size_t nn = (size_t)nB * (size_t)nB;
  DevBuf<int64_t> d_in, d_out;
  DevBuf<int32_t> d_tok, d_slot, d_deg, d_gpair;
  DevBuf<int16_t> d_gnbr;
  DevBuf<uint8_t> d_kind, d_status;
  DevBuf<double> d_amount, d_value, d_cost, d_net;
  HopSlots hs;
  CU_TRY(ctx, d_in.upload(token_in, (size_t)q));
  CU_TRY(ctx, d_out.upload(token_out, (size_t)q));
  CU_TRY(ctx, d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, d_tok.upload(tok));
  CU_TRY(ctx, d_slot.upload(slot_of));
  CU_TRY(ctx, d_deg.alloc((size_t)nB));
  CU_TRY(ctx, d_gnbr.alloc(nn));
  CU_TRY(ctx, d_gpair.alloc(nn));
  if ((rc = hs.alloc(ctx, q, H)) != CFMM_OK) return rc;
  CU_TRY(ctx, d_value.alloc((size_t)q));
  CU_TRY(ctx, d_status.alloc((size_t)q));
  if (hop_cost) {
    CU_TRY(ctx, d_cost.upload(hop_cost, (size_t)q));
    CU_TRY(ctx, d_net.alloc((size_t)q));
  }
  const size_t smem = cfmm::best_path_smem(nB, H);
  const auto kernel = hop_cost ? cfmm::best_path_kernel<true> : cfmm::best_path_kernel<false>;
  CU_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const cfmm::PairIndexView pv{ix.off.p, ix.pool.p};
  const cfmm::AdjView A{ix.adj_off.p, ix.adj_nbr.p, ix.adj_pair.p};
  const cfmm::BestPathGraph G{d_tok.p, d_slot.p, d_deg.p, d_gnbr.p, d_gpair.p, nB};
  if ((rc = launch(ctx, kProfSwaps, nB > 0 ? 2 : 1, [&] {
         if (nB > 0)
           cfmm::best_path_graph_kernel<<<(unsigned)((32 * (int64_t)nB + 255) / 256), 256, 0, st>>>(
               A, d_tok.p, d_slot.p, nB, d_deg.p, d_gnbr.p, d_gpair.p);
         kernel<<<(unsigned)q, cfmm::kBestPathThreads, smem, st>>>(
             os.d_P.p, pv, A, G, d_in.p, d_out.p, d_kind.p, d_amount.p, H, hs.nhop.p, hs.set.p, hs.pos.p, hs.tok1.p,
             hs.token.p, hs.tender.p, hs.received.p, d_value.p, d_status.p, d_cost.p, d_net.p);
       })) != CFMM_OK)
    return rc;
  CU_TRY(ctx, read_back(ctx, value, d_value.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, status, d_status.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, hop_cost ? net : nullptr, d_net.p, (size_t)q));
  return hs.pack(ctx, hop_off, hop_type, hop_pool, hop_token, hop_tender, hop_received);
}

// ---- token values from one root over the whole pool graph (token_value_kernels.cuh) -------------

// Every argument of cfmm_quote_token_values, before anything runs.
int check_token_values(cfmm_ctx* ctx, int64_t q, const int64_t* root, const uint8_t* kind, const double* amount,
                       int max_hops, const double* value, int64_t n_req, const int64_t* req_row,
                       const int64_t* req_token, const int64_t* hop_off, const int* hop_type, const int64_t* hop_pool,
                       const int64_t* hop_token, const char* what = "quote_token_values") {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative row count", what);
  if (n_req < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative request count", what);
  if (max_hops < 1 || max_hops > CFMM_PATH_MAX_HOPS)
    return fail(ctx, CFMM_ERR_INVALID, "%s: max_hops %d, not 1..%d", what, max_hops, CFMM_PATH_MAX_HOPS);
  if (ctx->n_tokens > INT32_MAX || ctx->n_pools > INT32_MAX)
    return fail(ctx, CFMM_ERR_INVALID, "%s: more than 2^31 - 1 tokens or pools", what);
  if (q == 0) return CFMM_OK;
  if (!root || !kind || !amount || !value)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null root, kind, amount or value", what);
  for (int64_t r = 0; r < q; ++r) {
    if (root[r] < 1 || root[r] > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: root %lld outside 1..%lld", what, (long long)r,
                  (long long)root[r], (long long)ctx->n_tokens);
    if (kind[r] > 1) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: kind %d, not 0 or 1", what, (long long)r, kind[r]);
    if (!(amount[r] > 0.0) || !std::isfinite(amount[r]))
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: amount %g, not finite and > 0", what, (long long)r, amount[r]);
  }
  if (n_req == 0) return CFMM_OK;
  if (!req_row || !req_token || !hop_off || !hop_type || !hop_pool || !hop_token)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null req_row, req_token, hop_off, hop_type, hop_pool or hop_token", what);
  for (int64_t j = 0; j < n_req; ++j) {
    if (req_row[j] < 0 || req_row[j] >= q)
      return fail(ctx, CFMM_ERR_INVALID, "%s: request %lld: row %lld outside 0..%lld", what, (long long)j,
                  (long long)req_row[j], (long long)(q - 1));
    if (req_token[j] < 1 || req_token[j] > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "%s: request %lld: token %lld outside 1..%lld", what, (long long)j,
                  (long long)req_token[j], (long long)ctx->n_tokens);
  }
  return CFMM_OK;
}

// Per-row bytes of the token-value workspace: val, best, lvl and H levels of predecessors; with net,
// also the selected level's value, net and level.
size_t token_value_row_bytes(int64_t n, int H, bool with_net) {
  return (size_t)n * (sizeof(double) + sizeof(unsigned __int128) + 1 + (size_t)H * sizeof(uint64_t) +
                      (with_net ? 2 * sizeof(double) + 1 : 0));
}
constexpr size_t kTokenValueBudget = size_t(512) << 20;  // workspace bytes the rows of one group may take

// hop_cost (cfmm_quote_token_values_net): per (row, token) the best filled max_hops = L result net
// of hop_cost[t] per hop, its net into net (NULL: not written); null: cfmm_quote_token_values.
int quote_token_values(cfmm_ctx* ctx, int64_t q, const int64_t* root, const uint8_t* kind, const double* amount,
                       int max_hops, const uint8_t* allowed, double* value, uint8_t* hops, uint8_t* status,
                       int64_t* frontier, int64_t n_req, const int64_t* req_row, const int64_t* req_token,
                       int64_t* hop_off, int* hop_type, int64_t* hop_pool, int64_t* hop_token, double* hop_tender,
                       double* hop_received, uint8_t* req_status, const double* hop_cost = nullptr,
                       double* net = nullptr) {
  int rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  cudaStream_t st = ctx->stream;
  OrderSets os;
  if ((rc = order_sets(ctx, false, os)) != CFMM_OK) return rc;
  const int64_t n = ctx->n_tokens;
  const int H = max_hops;
  cfmm::TvSets S{};
  for (int k = 0; k < cfmm::kPathSets; ++k) {
    const PoolSet& s = path_set(ctx, k);
    S.start[k + 1] = S.start[k] + (s.m > 0 ? s.m_padded : 0);
  }
  const int64_t positions = S.start[cfmm::kPathSets];
  // the group: up to kTvMaxGroup rows, as many as the budget holds (at least one)
  const size_t row_bytes = token_value_row_bytes(n, H, hop_cost != nullptr);
  const int G = (int)std::max<int64_t>(
      1, std::min<int64_t>({q, (int64_t)cfmm::kTvMaxGroup, (int64_t)(kTokenValueBudget / row_bytes)}));
  // workspace: [G][n] best (16-byte slots first), val, [G][H][n] pred, [2][n] fmask, [G][H+1] cnt,
  // [H+1] tot, [G][n] lvl; kept on the context and grown when a call needs more
  const size_t gn = (size_t)G * (size_t)n;
  const size_t b_best = 0, b_val = b_best + gn * 16, b_pred = b_val + gn * 8, b_fmask = b_pred + gn * H * 8,
               b_cnt = b_fmask + 2 * (size_t)n * 8, b_tot = b_cnt + (size_t)G * (H + 1) * 4,
               b_lvl = (b_tot + (size_t)(H + 1) * 4 + 15) & ~(size_t)15, b_end = b_lvl + gn;
  // with net: [G][n] selected value and net, [G][n] selected level, after the rest
  const size_t b_nval = (b_end + 15) & ~(size_t)15, b_nnet = b_nval + gn * 8, b_nlvl = b_nnet + gn * 8,
               b_all = hop_cost ? b_nlvl + gn : b_end;
  if (ctx->tv_ws.n < b_all) CU_TRY(ctx, ctx->tv_ws.alloc(b_all));
  unsigned char* ws = ctx->tv_ws.p;
  DevBuf<int64_t> d_root, d_req_row, d_req_tok, d_entry;
  DevBuf<uint8_t> d_kind, d_allowed, d_hops, d_status, d_rstatus;
  DevBuf<double> d_amount, d_value, d_cost, d_net;
  HopSlots hs;
  CU_TRY(ctx, d_root.upload(root, (size_t)q));
  CU_TRY(ctx, d_kind.upload(kind, (size_t)q));
  CU_TRY(ctx, d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, d_allowed.upload(allowed, (size_t)n));
  CU_TRY(ctx, d_value.alloc(gn));
  CU_TRY(ctx, d_hops.alloc(gn));
  CU_TRY(ctx, d_status.alloc(gn));
  if (hop_cost) {
    CU_TRY(ctx, d_cost.upload(hop_cost, (size_t)n));
    CU_TRY(ctx, d_net.alloc(gn));
  }
  // no selection without costs: every output from the last level a token changed at
  const cfmm::TvNet N = hop_cost ? cfmm::TvNet{d_cost.p, reinterpret_cast<double*>(ws + b_nval),
                                               reinterpret_cast<double*>(ws + b_nnet), ws + b_nlvl}
                                 : cfmm::TvNet{};
  if (n_req > 0) {
    CU_TRY(ctx, d_req_row.upload(req_row, (size_t)n_req));
    CU_TRY(ctx, d_req_tok.upload(req_token, (size_t)n_req));
    CU_TRY(ctx, d_entry.alloc((size_t)std::max<int64_t>(ctx->n_pools, 1)));
    CU_TRY(ctx, d_rstatus.alloc((size_t)n_req));
    if ((rc = hs.alloc(ctx, n_req, H)) != CFMM_OK) return rc;
    if ((rc = launch(ctx, kProfSwaps, 1, [&] {
           if (positions > 0)
             cfmm::tv_entry_kernel<<<(unsigned)((positions + 255) / 256), 256, 0, st>>>(os.d_P.p, S, d_entry.p);
         })) != CFMM_OK)
      return rc;
  }
  std::vector<int32_t> cnt((size_t)G * (H + 1));
  const unsigned tok_grid = (unsigned)((n + cfmm::kTvThreads - 1) / cfmm::kTvThreads);
  const unsigned pool_grid = (unsigned)((positions + cfmm::kTvThreads - 1) / cfmm::kTvThreads);
  for (int64_t r0 = 0; r0 < q; r0 += G) {
    const int g = (int)std::min<int64_t>(G, q - r0);
    const size_t gn_g = (size_t)g * (size_t)n;
    cfmm::TvWork W{d_root.p + r0,
                   d_kind.p + r0,
                   d_amount.p + r0,
                   allowed ? d_allowed.p : nullptr,
                   g,
                   H,
                   n,
                   reinterpret_cast<double*>(ws + b_val),
                   reinterpret_cast<unsigned __int128*>(ws + b_best),
                   ws + b_lvl,
                   reinterpret_cast<uint64_t*>(ws + b_pred),
                   reinterpret_cast<uint64_t*>(ws + b_fmask),
                   reinterpret_cast<int32_t*>(ws + b_cnt),
                   reinterpret_cast<int32_t*>(ws + b_tot)};
    bool any_req = false;
    for (int64_t j = 0; j < n_req && !any_req; ++j) any_req = req_row[j] >= r0 && req_row[j] < r0 + g;
    const unsigned gn_grid = (unsigned)((gn_g + 255) / 256);
    const int64_t n_launch = 2 + (pool_grid > 0 ? 2 : 1) * H + (hop_cost ? H : 0) + (any_req ? 1 : 0);
    if ((rc = launch(ctx, kProfSwaps, n_launch, [&] {
           cfmm::tv_init_kernel<<<tok_grid, cfmm::kTvThreads, 0, st>>>(W);
           for (int h = 1; h <= H; ++h) {
             if (pool_grid > 0) cfmm::tv_relax_kernel<<<pool_grid, cfmm::kTvThreads, 0, st>>>(os.d_P.p, S, W, h);
             cfmm::tv_finalize_kernel<<<tok_grid, cfmm::kTvThreads, 0, st>>>(W, h);
             if (hop_cost) cfmm::tv_select_kernel<<<gn_grid, 256, 0, st>>>(W, N, h);
           }
           cfmm::tv_rebuild_kernel<<<gn_grid, 256, 0, st>>>(W, N, d_value.p, d_hops.p, d_status.p, d_net.p);
           if (any_req)
             cfmm::tv_path_kernel<<<(unsigned)((n_req + 127) / 128), 128, 0, st>>>(
                 os.d_P.p, W, N, r0, d_entry.p, n_req, d_req_row.p, d_req_tok.p, hs.nhop.p, hs.set.p, hs.pos.p,
                 hs.tok1.p, hs.token.p, hs.tender.p, hs.received.p, d_rstatus.p);
         })) != CFMM_OK)
      return rc;
    CU_TRY(ctx, read_back(ctx, value + r0 * n, d_value.p, gn_g));
    CU_TRY(ctx, read_back(ctx, hops ? hops + r0 * n : nullptr, d_hops.p, gn_g));
    CU_TRY(ctx, read_back(ctx, status ? status + r0 * n : nullptr, d_status.p, gn_g));
    CU_TRY(ctx, read_back(ctx, frontier ? cnt.data() : nullptr, W.cnt, (size_t)g * (H + 1)));
    CU_TRY(ctx, read_back(ctx, hop_cost && net ? net + r0 * n : nullptr, d_net.p, gn_g));
    CU_TRY(ctx, cudaStreamSynchronize(st));
    if (frontier)
      for (int r = 0; r < g; ++r)
        for (int h = 1; h <= H; ++h) frontier[(r0 + r) * H + h - 1] = cnt[(size_t)r * (H + 1) + h];
  }
  if (n_req == 0) return CFMM_OK;
  CU_TRY(ctx, read_back(ctx, req_status, d_rstatus.p, (size_t)n_req));
  return hs.pack(ctx, hop_off, hop_type, hop_pool, hop_token, hop_tender, hop_received);
}

}  // namespace

int cfmm_quote_token_values(cfmm_ctx* ctx, int64_t q, const int64_t* root, const uint8_t* kind, const double* amount,
                            int max_hops, const uint8_t* allowed, double* value, uint8_t* hops, uint8_t* status,
                            int64_t* frontier, int64_t n_req, const int64_t* req_row, const int64_t* req_token,
                            int64_t* hop_off, int* hop_type, int64_t* hop_pool, int64_t* hop_token,
                            double* hop_tender, double* hop_received, uint8_t* req_status) {
  int rc = check_token_values(ctx, q, root, kind, amount, max_hops, value, n_req, req_row, req_token, hop_off,
                              hop_type, hop_pool, hop_token);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (hop_off) hop_off[0] = 0;
    return CFMM_OK;
  }
  return quote_token_values(ctx, q, root, kind, amount, max_hops, allowed, value, hops, status, frontier, n_req,
                            req_row, req_token, hop_off, hop_type, hop_pool, hop_token, hop_tender, hop_received,
                            req_status);
}

int cfmm_quote_token_values_net(cfmm_ctx* ctx, int64_t q, const int64_t* root, const uint8_t* kind,
                                const double* amount, int max_hops, const uint8_t* allowed, const double* hop_cost,
                                double* value, uint8_t* hops, uint8_t* status, double* net, int64_t* frontier,
                                int64_t n_req, const int64_t* req_row, const int64_t* req_token, int64_t* hop_off,
                                int* hop_type, int64_t* hop_pool, int64_t* hop_token, double* hop_tender,
                                double* hop_received, uint8_t* req_status) {
  const char* what = "quote_token_values_net";
  int rc = check_token_values(ctx, q, root, kind, amount, max_hops, value, n_req, req_row, req_token, hop_off,
                              hop_type, hop_pool, hop_token, what);
  if (rc != CFMM_OK || (rc = check_hop_cost(ctx, hop_cost, ctx->n_tokens, what)) != CFMM_OK) return rc;
  if (q == 0) {
    if (hop_off) hop_off[0] = 0;
    return CFMM_OK;
  }
  return quote_token_values(ctx, q, root, kind, amount, max_hops, allowed, value, hops, status, frontier, n_req,
                            req_row, req_token, hop_off, hop_type, hop_pool, hop_token, hop_tender, hop_received,
                            req_status, hop_cost, net);
}

int cfmm_pair_pools(cfmm_ctx* ctx, int64_t q, const int64_t* token_a, const int64_t* token_b, int64_t* count,
                    int64_t cap, int* type_out, int64_t* pool_out, uint8_t* active_out) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "pair_pools: negative row count");
  if (q == 0) return CFMM_OK;
  if (!token_a || !token_b || !count) return fail(ctx, CFMM_ERR_INVALID, "pair_pools: null array argument");
  if ((rc = check_pair_tokens(ctx, q, token_a, token_b, "pair_pools")) != CFMM_OK) return rc;
  DevBuf<int64_t> d_a, d_b, d_pair;
  std::vector<int64_t> cnt;
  if ((rc = pair_lookup(ctx, q, token_a, token_b, d_a, d_b, d_pair, cnt)) != CFMM_OK) return rc;
  std::vector<int64_t> cum((size_t)q, 0);
  int64_t total = 0;
  for (int64_t j = 0; j < q; ++j) {
    count[j] = cnt[(size_t)j];
    cum[(size_t)j] = total;
    total += cnt[(size_t)j];
  }
  if (total == 0 || total > cap || (!type_out && !pool_out && !active_out)) return CFMM_OK;
  DevBuf<int64_t> d_cum, d_ent;
  CU_TRY(ctx, d_cum.upload(cum));
  CU_TRY(ctx, d_ent.alloc((size_t)total));
  if ((rc = launch(ctx, kProfSwaps, 1, [&] {
         cfmm::pair_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(
             ctx->pairs.off.p, ctx->pairs.pool.p, d_pair.p, d_cum.p, q, total, d_ent.p);
       })) != CFMM_OK)
    return rc;
  std::vector<int64_t> ent((size_t)total);
  CU_TRY(ctx, read_back(ctx, ent.data(), d_ent.p, (size_t)total));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  for (int64_t t = 0; t < total; ++t) {  // (set, device position) -> (type, index in the type's insertion order)
    const int k = (int)(ent[(size_t)t] >> cfmm::kPairSetShift);
    const int64_t p = ent[(size_t)t] & cfmm::kPairPosMask;
    PoolSet& s = path_set(ctx, k);
    const int64_t i = s.order[(size_t)p];
    if (type_out) type_out[t] = k >> 1;
    if (pool_out) pool_out[t] = i + ((k & 1) ? ctx->sets[k >> 1].m : 0);
    if (active_out) active_out[t] = (s.retired.empty() || !s.retired[(size_t)i]) ? 1 : 0;
  }
  return CFMM_OK;
}

int cfmm_quote_split_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                            const uint8_t* kind, const double* amount, double* paid, double* received, double* price,
                            uint8_t* status, double* leg_delta, double* leg_lambda) {
  int rc = check_split(ctx, q, token_in, token_out, kind, amount, nullptr, "quote_split_orders");
  if (rc != CFMM_OK || q == 0) return rc;
  return split_orders(ctx, false, q, token_in, token_out, kind, amount, nullptr, paid, received, price, status,
                      leg_delta, leg_lambda);
}

int cfmm_execute_split_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                              const uint8_t* kind, const double* amount, const double* limit, double* paid,
                              double* received, double* price, uint8_t* status, double* leg_delta,
                              double* leg_lambda) {
  int rc = check_split(ctx, q, token_in, token_out, kind, amount, limit, "execute_split_orders");
  if (rc != CFMM_OK || q == 0) return rc;
  return split_orders(ctx, true, q, token_in, token_out, kind, amount, limit, paid, received, price, status,
                      leg_delta, leg_lambda);
}

int cfmm_quote_routed_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                             const uint8_t* kind, const double* amount, const int64_t* hub_off, const int64_t* hubs,
                             double* paid, double* received, double* price, uint8_t* status, double* hub_price,
                             double* hub_surplus, double* leg_delta, double* leg_lambda) {
  int rc = check_routed(ctx, q, token_in, token_out, kind, amount, nullptr, hub_off, hubs, "quote_routed_orders");
  if (rc != CFMM_OK || q == 0) return rc;
  return routed_orders(ctx, false, false, q, token_in, token_out, kind, amount, nullptr, hub_off, hubs, paid, received, price,
                       status, hub_price, hub_surplus, leg_delta, leg_lambda);
}

int cfmm_execute_routed_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                               const uint8_t* kind, const double* amount, const double* limit, const int64_t* hub_off,
                               const int64_t* hubs, double* paid, double* received, double* price, uint8_t* status,
                               double* hub_price, double* hub_surplus, double* leg_delta, double* leg_lambda) {
  int rc = check_routed(ctx, q, token_in, token_out, kind, amount, limit, hub_off, hubs, "execute_routed_orders");
  if (rc != CFMM_OK || q == 0) return rc;
  return routed_orders(ctx, true, false, q, token_in, token_out, kind, amount, limit, hub_off, hubs, paid, received,
                       price, status, hub_price, hub_surplus, leg_delta, leg_lambda);
}

int cfmm_quote_arbitrage(cfmm_ctx* ctx, int64_t q, const int64_t* base, const int64_t* other, const int64_t* hub_off,
                         const int64_t* hubs, double* profit, double* surplus_in, double* price, uint8_t* status,
                         double* hub_price, double* hub_surplus, double* leg_delta, double* leg_lambda) {
  int rc = check_arbitrage(ctx, q, base, other, nullptr, hub_off, hubs, "quote_arbitrage");
  if (rc != CFMM_OK || q == 0) return rc;
  return routed_orders(ctx, false, true, q, other, base, nullptr, nullptr, nullptr, hub_off, hubs, surplus_in, profit,
                       price, status, hub_price, hub_surplus, leg_delta, leg_lambda);
}

int cfmm_execute_arbitrage(cfmm_ctx* ctx, int64_t q, const int64_t* base, const int64_t* other,
                           const double* min_profit, const int64_t* hub_off, const int64_t* hubs, double* profit,
                           double* surplus_in, double* price, uint8_t* status, double* hub_price, double* hub_surplus,
                           double* leg_delta, double* leg_lambda) {
  int rc = check_arbitrage(ctx, q, base, other, min_profit, hub_off, hubs, "execute_arbitrage");
  if (rc != CFMM_OK || q == 0) return rc;
  return routed_orders(ctx, true, true, q, other, base, nullptr, nullptr, min_profit, hub_off, hubs, surplus_in,
                       profit, price, status, hub_price, hub_surplus, leg_delta, leg_lambda);
}

int cfmm_scan_arbitrage(cfmm_ctx* ctx, int64_t nb, const int64_t* base, const double* min_profit, int max_hubs,
                        int64_t cap, int64_t* found, int64_t* row_base, int64_t* row_other, int64_t* hub_count,
                        int64_t* hubs, double* profit, double* price) {
  int rc = check_scan(ctx, nb, base, min_profit, max_hubs, cap, found, row_base, row_other, hub_count, hubs, profit,
                      price);
  if (rc != CFMM_OK) return rc;
  *found = 0;
  if (nb == 0) return CFMM_OK;
  return scan_arbitrage(ctx, nb, base, min_profit, max_hubs, cap, found, row_base, row_other, hub_count, hubs, profit,
                        price);
}

int cfmm_choose_order_hubs(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                           const uint8_t* kind, const double* amount, int max_hubs, const uint8_t* allowed,
                           int64_t* hub_off, int64_t* hubs, double* hub_score, int64_t* n_eligible) {
  int rc = check_choose_hubs(ctx, q, token_in, token_out, kind, amount, max_hubs, hub_off, hubs);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (hub_off) hub_off[0] = 0;
    return CFMM_OK;
  }
  return choose_order_hubs(ctx, q, token_in, token_out, kind, amount, max_hubs, allowed, hub_off, hubs, hub_score,
                           n_eligible);
}

int cfmm_find_order_paths(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                          const uint8_t* kind, const double* amount, int max_hops, const uint8_t* allowed,
                          int64_t* hop_off, int* hop_type, int64_t* hop_pool, int64_t* hop_token, double* hop_tender,
                          double* hop_received, double* value, uint8_t* status) {
  int rc = check_find_paths(ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_off, hop_type, hop_pool,
                            hop_token);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (hop_off) hop_off[0] = 0;
    return CFMM_OK;
  }
  return find_order_paths(ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_off, hop_type, hop_pool,
                          hop_token, hop_tender, hop_received, value, status);
}

int cfmm_find_order_paths_net(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                              const uint8_t* kind, const double* amount, int max_hops, const uint8_t* allowed,
                              const double* hop_cost, int64_t* hop_off, int* hop_type, int64_t* hop_pool,
                              int64_t* hop_token, double* hop_tender, double* hop_received, double* value,
                              uint8_t* status, double* net) {
  const char* what = "find_order_paths_net";
  int rc = check_find_paths(ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_off, hop_type, hop_pool,
                            hop_token, what);
  if (rc != CFMM_OK || (rc = check_hop_cost(ctx, hop_cost, q, what)) != CFMM_OK) return rc;
  if (q == 0) {
    if (hop_off) hop_off[0] = 0;
    return CFMM_OK;
  }
  return find_order_paths(ctx, q, token_in, token_out, kind, amount, max_hops, allowed, hop_off, hop_type, hop_pool,
                          hop_token, hop_tender, hop_received, value, status, hop_cost, net);
}

// ---- orders routed over every pool among their allowed tokens (subgraph_kernels.cuh) ------------
namespace {

// The allowed tokens of a subgraph, basket or limit call: one mask over the tokens (mask), or a per-row
// CSR (off [q+1], tok 1-based; the _rows calls).  n_mask: the mask's count, set by the checks.
struct Allowed {
  const uint8_t* mask;
  bool per_row = false;
  const int64_t* off = nullptr;
  const int64_t* tok = nullptr;
  int64_t n_mask = 0;
  bool rows() const { return per_row; }
  int64_t count(int64_t r) const { return off ? off[r + 1] - off[r] : n_mask; }
  // whether row r allows token t (1-based)
  bool has(int64_t r, int64_t t) const {
    if (!off) return mask[t - 1] != 0;
    return std::find(tok + off[r], tok + off[r + 1], t) != tok + off[r + 1];
  }
};

// The context, the row count, the allowed tokens and the options of a basket or subgraph call.  A
// per-row CSR: allow_off non-null, from 0 and not decreasing, allow_token non-null when it lists any
// token, every token in 1..n_tokens and none twice in one row.
int check_row_opts(cfmm_ctx* ctx, int64_t q, Allowed& M, const cfmm_subgraph_opts& o, const char* what) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: negative row count", what);
  if (!M.rows() && !M.mask)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null allowed (the intermediate tokens are required)", what);
  if (M.rows()) {
    if (!M.off) return fail(ctx, CFMM_ERR_INVALID, "%s: null allow_off", what);
    if (M.off[0] != 0) return fail(ctx, CFMM_ERR_INVALID, "%s: allow_off[0] is %lld, not 0", what, (long long)M.off[0]);
    for (int64_t r = 0; r < q; ++r)
      if (M.off[r + 1] < M.off[r]) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: allow_off decreases", what, (long long)r);
    if (M.off[q] > 0 && !M.tok) return fail(ctx, CFMM_ERR_INVALID, "%s: null allow_token", what);
    std::vector<int64_t> seen((size_t)ctx->n_tokens, -1);  // the last row that listed each token
    for (int64_t r = 0; r < q; ++r) {
      for (int64_t k = M.off[r]; k < M.off[r + 1]; ++k) {
        const int64_t t = M.tok[k];
        if (t < 1 || t > ctx->n_tokens)
          return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: allowed token %lld outside 1..%lld", what, (long long)r,
                      (long long)t, (long long)ctx->n_tokens);
        if (seen[(size_t)(t - 1)] == r)
          return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: allowed token %lld listed twice", what, (long long)r,
                      (long long)t);
        seen[(size_t)(t - 1)] = r;
      }
    }
  } else {
    M.n_mask = count_allowed(ctx, M.mask);
  }
  if (o.max_iter < 1 || o.max_fun < 1)
    return fail(ctx, CFMM_ERR_INVALID, "%s: max_iter %d and max_fun %d must be >= 1", what, o.max_iter, o.max_fun);
  if (!(std::isfinite(o.rtol) && o.rtol > 0.0)) return fail(ctx, CFMM_ERR_INVALID, "%s: rtol %g must be finite and > 0", what, o.rtol);
  if (!(std::isfinite(o.factr) && o.factr >= 0.0))
    return fail(ctx, CFMM_ERR_INVALID, "%s: factr %g must be finite and >= 0", what, o.factr);
  return CFMM_OK;
}

int check_limit(cfmm_ctx* ctx, const double* limit, int64_t r, const char* what) {
  if (limit && !(std::isfinite(limit[r]) && limit[r] >= 0.0))
    return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: limit %g must be finite and >= 0", what, (long long)r, limit[r]);
  return CFMM_OK;
}

// Every argument of cfmm_quote_subgraph_swap_orders / cfmm_execute_subgraph_swap_orders, before
// anything runs.  kind null: every row exact-in.
int check_subgraph(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out, const uint8_t* kind,
                   const double* amount, const double* limit, Allowed& M, const cfmm_subgraph_opts& o,
                   const char* what) {
  int rc = check_row_opts(ctx, q, M, o, what);
  if (rc != CFMM_OK || q == 0) return rc;
  if (!token_in || !token_out || !amount) return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  if ((rc = check_pair_tokens(ctx, q, token_in, token_out, what)) != CFMM_OK) return rc;
  for (int64_t j = 0; j < q; ++j) {
    if (kind && kind[j] > CFMM_SWAP_EXACT_OUT)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: kind %d is neither 0 (exact-in) nor 1 (exact-out)", what,
                  (long long)j, (int)kind[j]);
    if (!std::isfinite(amount[j]) || amount[j] < 0.0)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: amount %g must be finite and >= 0", what, (long long)j,
                  amount[j]);
    if (kind && kind[j] == CFMM_SWAP_EXACT_OUT) {  // the maximum paid: +inf allowed
      if (limit && !(limit[j] >= 0.0))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: exact-out limit %g must be >= 0", what, (long long)j,
                    limit[j]);
    } else if ((rc = check_limit(ctx, limit, j, what)) != CFMM_OK) {
      return rc;
    }
  }
  for (int64_t r = 0; r < q; ++r) {
    const int64_t nb = M.count(r) - M.has(r, token_in[r]) - M.has(r, token_out[r]);
    if (nb > CFMM_SUBGRAPH_MAX_TOKENS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld intermediate tokens, more than %d", what, (long long)r,
                  (long long)nb, CFMM_SUBGRAPH_MAX_TOKENS);
  }
  return CFMM_OK;
}

// Whether row r of a basket call is a buy row: at least one entry of kind CFMM_SWAP_EXACT_OUT.
bool basket_buy_row(const int64_t* basket_off, const uint8_t* kind, int64_t r) {
  return kind && std::find(kind + basket_off[r], kind + basket_off[r + 1], (uint8_t)CFMM_SWAP_EXACT_OUT) !=
                     kind + basket_off[r + 1];
}

// Every argument of cfmm_quote/execute_basket_orders (kind null) and cfmm_quote/execute_basket_swap_orders,
// before anything runs.
int check_basket(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                 const int64_t* basket_token, const uint8_t* kind, const double* basket_amount, const double* limit,
                 Allowed& M, const cfmm_subgraph_opts& o, const char* what) {
  int rc = check_row_opts(ctx, q, M, o, what);
  if (rc != CFMM_OK || q == 0) return rc;
  if (!token_out || !basket_off || !basket_token || !basket_amount)
    return fail(ctx, CFMM_ERR_INVALID, "%s: null array argument", what);
  if (basket_off[0] != 0) return fail(ctx, CFMM_ERR_INVALID, "%s: basket_off[0] is %lld, not 0", what, (long long)basket_off[0]);
  for (int64_t r = 0; r < q; ++r) {
    const int64_t b0 = basket_off[r], K = basket_off[r + 1] - b0, i = token_out[r];
    if (K < 0) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: basket_off decreases", what, (long long)r);
    if (K < 1 || K > CFMM_BASKET_MAX_TOKENS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld basket entries, not 1..%d", what, (long long)r,
                  (long long)K, CFMM_BASKET_MAX_TOKENS);
    if (i < 1 || i > ctx->n_tokens)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: token_out %lld outside 1..%lld", what, (long long)r,
                  (long long)i, (long long)ctx->n_tokens);
    int64_t n_other = M.count(r) - M.has(r, i);  // the row's tokens other than i
    for (int64_t k = b0; k < b0 + K; ++k) {
      const int64_t t = basket_token[k];
      const double a = basket_amount[k];
      if (t < 1 || t > ctx->n_tokens)
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: basket token %lld outside 1..%lld", what, (long long)r,
                    (long long)t, (long long)ctx->n_tokens);
      if (t == i) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: token_out %lld is in the basket", what, (long long)r, (long long)i);
      for (int64_t l = b0; l < k; ++l)
        if (basket_token[l] == t)
          return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: basket token %lld appears twice", what, (long long)r,
                      (long long)t);
      if (!std::isfinite(a) || a < 0.0)
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: amount %g must be finite and >= 0", what, (long long)r, a);
      if (kind && kind[k] > CFMM_SWAP_EXACT_OUT)
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: entry kind %d is neither 0 (sold) nor 1 (bought)", what,
                    (long long)r, (int)kind[k]);
      n_other += !M.has(r, t);
    }
    if (n_other > CFMM_SUBGRAPH_MAX_TOKENS + 1)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld tokens besides token_out, more than %d", what,
                  (long long)r, (long long)n_other, CFMM_SUBGRAPH_MAX_TOKENS + 1);
    if (basket_buy_row(basket_off, kind, r)) {  // the minimum net of token_out: negative and −inf allowed
      if (limit && !(limit[r] < INFINITY))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: buy-row limit %g must not be NaN or +inf", what,
                    (long long)r, limit[r]);
    } else if ((rc = check_limit(ctx, limit, r, what)) != CFMM_OK) {
      return rc;
    }
  }
  return CFMM_OK;
}

// The occupancy of a row kernel, cached per context.  A family with dynamic shared memory (basket rows,
// dyn: its kernels) may take most_dyn (that of the longest basket over the most slots; per-row masks add
// the row graph's kRowGraphBytes), beyond the 48 KB default:
// the attribute of each of its kernels is set once per context to that one value (so concurrent calls
// never lower it), and the occupancy taken there.
int row_occupancy(cfmm_ctx* ctx, const void* kernel, std::initializer_list<const void*> dyn, const char* name,
                  int& occ, size_t most_dyn = cfmm::bk_dyn_bytes(cfmm::kBasketMaxTokens, cfmm::kSubgraphSlots)) {
  int& c = ctx->occupancy[kernel];
  if (c == 0) {
    const int most = dyn.size() ? (int)most_dyn : 0;
    for (const void* f : dyn) CU_TRY(ctx, cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    CU_TRY(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, kernel, cfmm::kSubgraphThreads, (size_t)most));
    if (c < 1) return fail(ctx, CFMM_ERR_CUDA, "%s does not fit on an SM", name);
  }
  occ = c;
  return CFMM_OK;
}

extern "C++" template <class K>
const void* kernel_ptr(K* k) {
  return reinterpret_cast<const void*>(k);
}

// One subgraph or basket call after its checks, on the device of ctx with its inputs uploaded (R's input
// pointers and options).  The family gives what differs:
//   occ, occ2     the occupancy of its two row kernels (occ2 0 when no row takes the second);
//   n2, second    the number of rows second(r) sends to the second kernel (exact-out rows, buy rows);
//   K             its longest basket (0: subgraph rows), which sizes the dynamic shared memory;
//   n_paid        the length of paid (q, or basket_off[q]);
//   plan(...)     the plan launch; rows(exec_tag, second, ...) a launch of one row kernel;
//   visit(r, v)   the tokens row r visits besides the slots (a token visited twice changes nothing),
//                 and uses their count over the call, for the conflict levels of an execute;
//   all_slots     every row also visits every slot (subgraph and basket rows: B is the whole mask, or
//                 with per-row masks the row's own list).
// The driver builds the call's slots and their B-graph (per-row masks: uploads the lists and sizes the
// per-CTA row graphs, which each row's CTA builds), runs the plan, sizes the outputs and the per-CTA
// workspace, runs the rows (a level's rows, or a quote's, split between the two kernels), and reads back.
// plan and rows get both the call's graph and the per-row masks (RM.off null with one mask).
extern "C++" template <class Rows, class Out, class Plan, class RowLaunch, class Second, class Visit>
int row_orders(cfmm_ctx* ctx, bool exec, int64_t q, const Allowed& M, Rows R, const Out& O, int occ, int occ2,
               int64_t n2, int K, int64_t n_paid, int64_t uses, bool all_slots, const char* what, Plan plan,
               RowLaunch rows,
               Second second, Visit visit) {
  int rc;
  auto& ix = ctx->pairs;
  cudaStream_t st = ctx->stream;
  // the call's slots: the allowed tokens, ascending; their filtered adjacency and its activity (none
  // with per-row masks)
  std::vector<int32_t> tok, slot_of(M.rows() ? 0 : (size_t)ctx->n_tokens, -1);
  for (int64_t t = 0; !M.rows() && t < ctx->n_tokens; ++t)
    if (M.mask[t]) {
      slot_of[(size_t)t] = (int32_t)tok.size();
      tok.push_back((int32_t)t);
    }
  const int nB = (int)tok.size();
  // per-row masks: the longest list sizes each CTA's row graph; its tokens and degrees go after the
  // basket rows' dynamic shared memory
  int64_t bmax = 0;
  for (int64_t r = 0; M.rows() && r < q; ++r) bmax = std::max(bmax, M.count(r));
  const size_t nn = (size_t)nB * (size_t)nB, goff = K > 0 ? cfmm::bk_dyn_bytes(K, M.rows() ? (int)bmax : nB) : 0,
               dyn = goff + (M.rows() ? (size_t)cfmm::kRowGraphBytes : 0);
  DevBuf<int64_t> d_ntok, d_npool;
  DevBuf<int32_t> d_tok, d_slot, d_deg, d_gpair;
  DevBuf<int16_t> d_gnbr;
  DevBuf<uint8_t> d_act;
  CU_TRY(ctx, d_tok.upload(tok));
  CU_TRY(ctx, d_slot.upload(slot_of));
  CU_TRY(ctx, d_deg.alloc((size_t)nB));
  CU_TRY(ctx, d_gnbr.alloc(nn));
  CU_TRY(ctx, d_gpair.alloc(nn));
  CU_TRY(ctx, d_act.alloc(nn));
  CU_TRY(ctx, d_ntok.alloc((size_t)q));
  CU_TRY(ctx, d_npool.alloc((size_t)q));
  OrderSets os;
  if ((rc = order_sets(ctx, false, os)) != CFMM_OK) return rc;
  const cfmm::PairIndexView pv{ix.off.p, ix.pool.p};
  const cfmm::AdjView A{ix.adj_off.p, ix.adj_nbr.p, ix.adj_pair.p};
  const cfmm::BestPathGraph G{d_tok.p, d_slot.p, d_deg.p, d_gnbr.p, d_gpair.p, nB};
  // a persistent grid: one wave of resident CTAs of each kernel that runs
  const int64_t wave = (int64_t)ctx->sm_count * occ, wave2 = (int64_t)ctx->sm_count * occ2;
  const unsigned plan_grid = (unsigned)std::min<int64_t>(q, wave);
  const int64_t grid = std::min<int64_t>(q, std::max(wave, wave2));  // the workspaces
  DevBuf<int64_t> d_aoff, d_atok;
  DevBuf<int16_t> d_rnbr;
  DevBuf<int32_t> d_rpair;
  DevBuf<uint8_t> d_ract;
  cfmm::RowMasks RM{};
  if (M.rows()) {
    const size_t cells = (size_t)(bmax * bmax) * (size_t)grid;
    CU_TRY(ctx, d_aoff.upload(M.off, (size_t)q + 1));
    CU_TRY(ctx, d_atok.upload(M.tok, (size_t)M.off[q]));
    CU_TRY(ctx, d_rnbr.alloc(cells));
    CU_TRY(ctx, d_rpair.alloc(cells));
    CU_TRY(ctx, d_ract.alloc(cells));
    RM = cfmm::RowMasks{d_aoff.p, d_atok.p, d_rnbr.p, d_rpair.p, d_ract.p, bmax * bmax, (int)goff};
  }
  if ((rc = launch(ctx, kProfSwaps, nB > 0 ? 3 : 1, [&] {
         if (nB > 0) {
           cfmm::best_path_graph_kernel<<<(unsigned)((32 * (int64_t)nB + 255) / 256), 256, 0, st>>>(
               A, d_tok.p, d_slot.p, nB, d_deg.p, d_gnbr.p, d_gpair.p);
           cfmm::subgraph_act_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(os.d_P.p, pv, G, d_act.p);
         }
         plan(plan_grid, dyn, st, os.d_P.p, pv, A, G, d_act.p, RM, d_ntok.p, d_npool.p);
       })) != CFMM_OK)
    return rc;
  std::vector<int64_t> ntok((size_t)q), npool((size_t)q);
  CU_TRY(ctx, read_back(ctx, ntok.data(), d_ntok.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, npool.data(), d_npool.p, (size_t)q));
  CU_TRY(ctx, cudaStreamSynchronize(st));
  std::vector<int64_t> tok_off((size_t)q + 1, 0), leg_off((size_t)q + 1, 0);
  int64_t max_pool = 0;
  for (int64_t r = 0; r < q; ++r) {
    tok_off[(size_t)r + 1] = tok_off[(size_t)r] + ntok[(size_t)r];
    leg_off[(size_t)r + 1] = leg_off[(size_t)r] + npool[(size_t)r];
    max_pool = std::max(max_pool, npool[(size_t)r]);
  }
  const int64_t NT = tok_off[(size_t)q], L = leg_off[(size_t)q];
  if (O.tok_off) std::copy(tok_off.begin(), tok_off.end(), O.tok_off);
  if (O.leg_off) std::copy(leg_off.begin(), leg_off.end(), O.leg_off);
  const bool want_tok = O.token || O.nu || O.psi, want_leg = O.leg_type || O.leg_pool || O.leg_delta || O.leg_lambda;
  if (exec && ((want_tok && NT > O.tok_cap) || (want_leg && L > O.leg_cap)))
    return fail(ctx, CFMM_ERR_INVALID,
                "%s: the outputs need %lld token and %lld leg entries, above tok_cap %lld or leg_cap %lld", what,
                (long long)NT, (long long)L, (long long)O.tok_cap, (long long)O.leg_cap);
  const bool toks = want_tok && NT > 0 && NT <= O.tok_cap, legs = want_leg && L > 0 && L <= O.leg_cap;
  // a size query (no per-row output, and no token or leg output that fits) runs no solve
  if (!exec && !toks && !legs && !O.paid && !O.received && !O.status && !O.solver_status && !O.iterations &&
      !O.fun_evals && !O.merit)
    return CFMM_OK;
  // outputs and the per-CTA workspace
  DevBuf<int64_t> d_tok_off, d_leg_off, d_token, d_entry;
  DevBuf<double> d_paid, d_recv, d_merit, d_nu, d_psi, d_ld, d_ll;
  DevBuf<uint8_t> d_status;
  DevBuf<int32_t> d_sst, d_iter, d_fev;
  CU_TRY(ctx, d_tok_off.upload(tok_off));
  CU_TRY(ctx, d_leg_off.upload(leg_off));
  CU_TRY(ctx, d_paid.alloc((size_t)n_paid));
  CU_TRY(ctx, d_recv.alloc((size_t)q));
  CU_TRY(ctx, d_merit.alloc((size_t)q));
  CU_TRY(ctx, d_status.alloc((size_t)q));
  CU_TRY(ctx, d_sst.alloc((size_t)q));
  CU_TRY(ctx, d_iter.alloc((size_t)q));
  CU_TRY(ctx, d_fev.alloc((size_t)q));
  if (toks) {
    CU_TRY(ctx, d_token.alloc((size_t)NT));
    CU_TRY(ctx, d_nu.alloc((size_t)NT));
    CU_TRY(ctx, d_psi.alloc((size_t)NT));
  }
  if (legs) {
    CU_TRY(ctx, d_entry.alloc((size_t)L));
    CU_TRY(ctx, d_ld.alloc((size_t)(2 * L)));
    CU_TRY(ctx, d_ll.alloc((size_t)(2 * L)));
  }
  int64_t cap = 1;
  while (cap < max_pool) cap <<= 1;
  DevBuf<int64_t> w64;
  DevBuf<int32_t> w32;
  DevBuf<double> wd;
  CU_TRY(ctx, w64.alloc((size_t)(2 * cap * grid)));
  CU_TRY(ctx, w32.alloc((size_t)(4 * cap * grid)));
  CU_TRY(ctx, wd.alloc((size_t)(2 * cap * grid)));
  const cfmm::SubgraphWork W{w64.p, w64.p + cap * grid, w32.p, w32.p + cap * grid, w32.p + 2 * cap * grid,
                             wd.p, wd.p + cap * grid, cap};
  R.tok_off = d_tok_off.p;
  R.leg_off = d_leg_off.p;
  R.paid = d_paid.p;
  R.received = d_recv.p;
  R.status = d_status.p;
  R.solver_status = d_sst.p;
  R.iterations = d_iter.p;
  R.fun_evals = d_fev.p;
  R.merit = d_merit.p;
  R.token = d_token.p;
  R.nu = d_nu.p;
  R.psi = d_psi.p;
  R.leg_entry = d_entry.p;
  R.leg_delta = d_ld.p;
  R.leg_lambda = d_ll.p;
  // rows[0 .. n1) to the first kernel, rows[n1 .. n) to the second: one launch of each kernel that has
  // rows (rows null: every row to the first)
  const auto run = [&](auto exec_tag, const cfmm::PathSets* P, const cfmm::SplitMoved& mv, const int64_t* rows_,
                       int64_t n1, int64_t n) {
    return launch(ctx, kProfSwaps, (n1 > 0) + (n > n1), [&] {
      if (n1 > 0)
        rows(exec_tag, false, (unsigned)std::min(n1, wave), dyn, st, P, pv, A, G, d_act.p, RM, R, W, mv, rows_, n1);
      if (n > n1)
        rows(exec_tag, true, (unsigned)std::min(n - n1, wave2), dyn, st, P, pv, A, G, d_act.p, RM, R, W, mv,
             rows_ + n1, n - n1);
    });
  };
  const auto first = [&](int64_t r) { return !second(r); };
  OrderSets xs;
  if (!exec && n2 == 0) {
    if ((rc = run(std::false_type{}, os.d_P.p, cfmm::SplitMoved{}, nullptr, q, q)) != CFMM_OK) return rc;
  } else if (!exec) {
    std::vector<int64_t> order((size_t)q);
    std::iota(order.begin(), order.end(), (int64_t)0);
    std::stable_partition(order.begin(), order.end(), first);
    DevBuf<int64_t> d_rows;
    CU_TRY(ctx, d_rows.upload(order));
    if ((rc = run(std::false_type{}, os.d_P.p, cfmm::SplitMoved{}, d_rows.p, q - n2, q)) != CFMM_OK) return rc;
  } else {
    if ((rc = order_sets(ctx, true, xs)) != CFMM_OK) return rc;
    ctx->state_version++;
    // levels over the tokens the rows visit and B (one table of n_tokens entries; per-row masks: each
    // row's own list)
    int64_t size = ctx->n_tokens, use = uses + (all_slots ? (M.rows() ? M.off[q] : q * (int64_t)nB) : 0);
    std::vector<int64_t> order, level_off;
    conflict_levels(
        q, 1, &size, &use,
        [&](int64_t r, auto&& v) {
          visit(r, v);
          if (all_slots && M.rows())
            for (int64_t k = M.off[r]; k < M.off[r + 1]; ++k) v(0, M.tok[k] - 1);
          else if (all_slots)
            for (int32_t t : tok) v(0, t);
        },
        order, level_off);
    // a level's rows share no token, so their order does not matter: its first kernel's rows go first
    DevBuf<int64_t> d_order;
    std::vector<int64_t> level_first(level_off.size(), 0);
    for (size_t Lv = 1; Lv < level_off.size(); ++Lv) {
      const auto b = order.begin() + level_off[Lv - 1], e = order.begin() + level_off[Lv];
      level_first[Lv] = n2 > 0 ? std::stable_partition(b, e, first) - b : e - b;
    }
    CU_TRY(ctx, d_order.upload(order));
    for (size_t Lv = 1; Lv < level_off.size(); ++Lv)
      if ((rc = run(std::true_type{}, xs.d_P.p, xs.mv, d_order.p + level_off[Lv - 1], level_first[Lv],
                    level_off[Lv] - level_off[Lv - 1])) != CFMM_OK)
        return rc;
    if ((rc = order_bookkeeping(ctx, xs)) != CFMM_OK) return rc;
  }
  CU_TRY(ctx, read_back(ctx, O.paid, d_paid.p, (size_t)n_paid));
  CU_TRY(ctx, read_back(ctx, O.received, d_recv.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, O.status, d_status.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, O.solver_status, d_sst.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, O.iterations, d_iter.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, O.fun_evals, d_fev.p, (size_t)q));
  CU_TRY(ctx, read_back(ctx, O.merit, d_merit.p, (size_t)q));
  std::vector<int64_t> ent(legs && (O.leg_type || O.leg_pool) ? (size_t)L : 0);
  if (toks) {
    CU_TRY(ctx, read_back(ctx, O.token, d_token.p, (size_t)NT));
    CU_TRY(ctx, read_back(ctx, O.nu, d_nu.p, (size_t)NT));
    CU_TRY(ctx, read_back(ctx, O.psi, d_psi.p, (size_t)NT));
  }
  if (legs) {
    CU_TRY(ctx, read_back(ctx, ent.empty() ? nullptr : ent.data(), d_entry.p, (size_t)L));
    CU_TRY(ctx, read_back(ctx, O.leg_delta, d_ld.p, (size_t)(2 * L)));
    CU_TRY(ctx, read_back(ctx, O.leg_lambda, d_ll.p, (size_t)(2 * L)));
  }
  CU_TRY(ctx, cudaStreamSynchronize(st));
  for (size_t t = 0; t < ent.size(); ++t) {  // (set, device position) -> (type, index in the type's order)
    const int k = (int)(ent[t] >> cfmm::kPairSetShift);
    const int64_t p = ent[t] & cfmm::kPairPosMask;
    if (O.leg_type) O.leg_type[t] = k >> 1;
    if (O.leg_pool) O.leg_pool[t] = pool_id(ctx, k, p);
  }
  return CFMM_OK;
}

// The device, the stream and the token adjacency of a subgraph or basket call.
int row_begin(cfmm_ctx* ctx) {
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  int rc = use_stream(ctx, ctx->stream);
  return rc != CFMM_OK ? rc : ensure_adjacency(ctx);
}

int subgraph_orders(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_in, const int64_t* token_out,
                    const uint8_t* kind, const double* amount, const double* limit, const Allowed& M,
                    const cfmm_subgraph_opts& o, cfmm_subgraph_out* out) {
  int rc;
  if ((rc = row_begin(ctx)) != CFMM_OK) return rc;
  cfmm_subgraph_out none{};
  DevBuf<int64_t> d_in, d_out;
  DevBuf<double> d_amount, d_limit;
  CU_TRY(ctx, d_in.upload(token_in, (size_t)q));
  CU_TRY(ctx, d_out.upload(token_out, (size_t)q));
  CU_TRY(ctx, d_amount.upload(amount, (size_t)q));
  CU_TRY(ctx, d_limit.upload(limit, (size_t)q));
  int occ = 0, occ_out = 0;
  const char* name = "a subgraph row kernel";
  const int64_t n_out = kind ? std::count(kind, kind + q, (uint8_t)CFMM_SWAP_EXACT_OUT) : 0;
  if (M.rows()) {  // per-row masks: the row graph's dynamic shared memory
    if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::subgraph_rows_kernel<false, false>),
                            {kernel_ptr(&cfmm::subgraph_rows_plan_kernel), kernel_ptr(&cfmm::subgraph_rows_kernel<false, false>),
                             kernel_ptr(&cfmm::subgraph_rows_kernel<true, false>)},
                            name, occ, cfmm::kRowGraphBytes)) != CFMM_OK)
      return rc;
    if (n_out > 0 && (rc = row_occupancy(ctx, kernel_ptr(&cfmm::subgraph_rows_kernel<false, true>),
                                         {kernel_ptr(&cfmm::subgraph_rows_kernel<false, true>),
                                          kernel_ptr(&cfmm::subgraph_rows_kernel<true, true>)},
                                         name, occ_out, cfmm::kRowGraphBytes)) != CFMM_OK)
      return rc;
  } else {
    if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::subgraph_kernel<false>), {}, name, occ)) != CFMM_OK) return rc;
    if (n_out > 0 && (rc = row_occupancy(ctx, kernel_ptr(&cfmm::subgraph_out_kernel<false>), {}, name, occ_out)) != CFMM_OK)
      return rc;
  }
  cfmm::SubgraphRows R{d_in.p, d_out.p, d_amount.p, d_limit.p, o.max_iter, o.max_fun, o.rtol, o.factr};
  return row_orders(
      ctx, exec, q, M, R, out ? *out : none, occ, occ_out, n_out, 0, q, 2 * q, true, "execute_subgraph_orders",
      [&](unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P, cfmm::PairIndexView pv, cfmm::AdjView A,
          const cfmm::BestPathGraph& G, const uint8_t* act, const cfmm::RowMasks& RM, int64_t* ntok, int64_t* npool) {
        if (RM.off)
          cfmm::subgraph_rows_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, d_in.p, d_out.p, q,
                                                                                     ntok, npool);
        else
          cfmm::subgraph_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, d_in.p, d_out.p, q,
                                                                                ntok, npool);
      },
      [&](auto exec_tag, bool second, unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P,
          cfmm::PairIndexView pv, cfmm::AdjView A, const cfmm::BestPathGraph& G, const uint8_t* act,
          const cfmm::RowMasks& RM, const cfmm::SubgraphRows& R, const cfmm::SubgraphWork& W, const cfmm::SplitMoved& mv,
          const int64_t* rows, int64_t n) {
        constexpr bool X = decltype(exec_tag)::value;
        if (RM.off && second)
          cfmm::subgraph_rows_kernel<X, true><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, R, W, mv, rows, n);
        else if (RM.off)
          cfmm::subgraph_rows_kernel<X, false><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, R, W, mv, rows, n);
        else if (second)
          cfmm::subgraph_out_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, R, W, mv, rows, n);
        else
          cfmm::subgraph_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, R, W, mv, rows, n);
      },
      [&](int64_t r) { return kind[r] == CFMM_SWAP_EXACT_OUT; },
      [&](int64_t r, auto&& visit) {
        visit(0, token_in[r] - 1);
        visit(0, token_out[r] - 1);
      });
}

// kind null: every row sell-only (cfmm_quote/execute_basket_orders).  limit_price set (kind null): every
// row a limit row (cfmm_quote/execute_limit_orders), run by basket_limit_kernel.
int basket_orders(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                  const int64_t* basket_token, const uint8_t* kind, const double* basket_amount,
                  const double* limit_price, const double* limit, const Allowed& M, const cfmm_subgraph_opts& o,
                  const cfmm_basket_out& O, const char* what) {
  int rc;
  if ((rc = row_begin(ctx)) != CFMM_OK) return rc;
  const int64_t NE = basket_off[q];
  int K = 0;
  for (int64_t r = 0; r < q; ++r) K = std::max<int>(K, (int)(basket_off[r + 1] - basket_off[r]));
  DevBuf<int64_t> d_out, d_boff, d_btok;
  DevBuf<uint8_t> d_kind;
  DevBuf<double> d_bamt, d_limit, d_price;
  CU_TRY(ctx, d_out.upload(token_out, (size_t)q));
  CU_TRY(ctx, d_boff.upload(basket_off, (size_t)q + 1));
  if (kind) CU_TRY(ctx, d_kind.upload(kind, (size_t)NE));
  CU_TRY(ctx, d_btok.upload(basket_token, (size_t)NE));
  CU_TRY(ctx, d_bamt.upload(basket_amount, (size_t)NE));
  if (limit_price) CU_TRY(ctx, d_price.upload(limit_price, (size_t)NE));
  CU_TRY(ctx, d_limit.upload(limit, (size_t)q));
  int occ = 0, occ_buy = 0;
  int64_t n_buy = 0;
  for (int64_t r = 0; r < q; ++r) n_buy += basket_buy_row(basket_off, kind, r);
  if (M.rows()) {  // per-row masks: basket_rows_kernel, with the row graph after the basket's bytes
    const size_t most = cfmm::bk_dyn_bytes(cfmm::kBasketMaxTokens, cfmm::kSubgraphSlots) + cfmm::kRowGraphBytes;
    const void* plan = kernel_ptr(&cfmm::basket_rows_plan_kernel);
    if (limit_price) {
      if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_rows_kernel<false, false, true>),
                              {plan, kernel_ptr(&cfmm::basket_rows_kernel<false, false, true>),
                               kernel_ptr(&cfmm::basket_rows_kernel<true, false, true>)},
                              "basket_rows_kernel", occ, most)) != CFMM_OK)
        return rc;
    } else if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_rows_kernel<false, false, false>),
                                   {plan, kernel_ptr(&cfmm::basket_rows_kernel<false, false, false>),
                                    kernel_ptr(&cfmm::basket_rows_kernel<true, false, false>)},
                                   "basket_rows_kernel", occ, most)) != CFMM_OK) {
      return rc;
    }
    if (n_buy > 0 && (rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_rows_kernel<false, true, false>),
                                         {kernel_ptr(&cfmm::basket_rows_kernel<false, true, false>),
                                          kernel_ptr(&cfmm::basket_rows_kernel<true, true, false>)},
                                         "basket_rows_kernel", occ_buy, most)) != CFMM_OK)
      return rc;
  } else if (limit_price) {
    if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_limit_kernel<false>),
                            {kernel_ptr(&cfmm::basket_plan_kernel), kernel_ptr(&cfmm::basket_limit_kernel<false>),
                             kernel_ptr(&cfmm::basket_limit_kernel<true>)},
                            "basket_limit_kernel", occ)) != CFMM_OK)
      return rc;
  } else if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_kernel<false>),
                                 {kernel_ptr(&cfmm::basket_plan_kernel), kernel_ptr(&cfmm::basket_kernel<false>),
                                  kernel_ptr(&cfmm::basket_kernel<true>)},
                                 "basket_kernel", occ)) != CFMM_OK) {
    return rc;
  }
  // buy rows run basket_buy_kernel (sized the same way, once per context, when a call first has them)
  if (!M.rows() && n_buy > 0 &&
      (rc = row_occupancy(ctx, kernel_ptr(&cfmm::basket_buy_kernel<false>),
                          {kernel_ptr(&cfmm::basket_buy_kernel<false>), kernel_ptr(&cfmm::basket_buy_kernel<true>)},
                          "basket_buy_kernel", occ_buy)) != CFMM_OK)
    return rc;
  // (basket_kernel and basket_buy_kernel take the BasketRows part of R)
  cfmm::LimitRows R{{d_out.p, d_boff.p, d_btok.p, d_bamt.p, d_limit.p, o.max_iter, o.max_fun, o.rtol, o.factr},
                    d_price.p};
  return row_orders(
      ctx, exec, q, M, R, O, occ, occ_buy, n_buy, K, NE, q + NE, true, what,
      [&](unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P, cfmm::PairIndexView pv, cfmm::AdjView A,
          const cfmm::BestPathGraph& G, const uint8_t* act, const cfmm::RowMasks& RM, int64_t* ntok, int64_t* npool) {
        if (RM.off)
          cfmm::basket_rows_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, d_boff.p, d_btok.p,
                                                                                   d_out.p, q, ntok, npool);
        else
          cfmm::basket_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, d_boff.p, d_btok.p,
                                                                              d_out.p, q, ntok, npool);
      },
      [&](auto exec_tag, bool second, unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P,
          cfmm::PairIndexView pv, cfmm::AdjView A, const cfmm::BestPathGraph& G, const uint8_t* act,
          const cfmm::RowMasks& RM, const cfmm::LimitRows& R, const cfmm::SubgraphWork& W, const cfmm::SplitMoved& mv,
          const int64_t* rows, int64_t n) {
        constexpr bool X = decltype(exec_tag)::value;
        const cfmm::BasketRows& B = R;
        if (RM.off && limit_price)
          cfmm::basket_rows_kernel<X, false, true><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, R, nullptr, W,
                                                                                             mv, rows, n);
        else if (RM.off && second)
          cfmm::basket_rows_kernel<X, true, false><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, B, d_kind.p,
                                                                                             W, mv, rows, n);
        else if (RM.off)
          cfmm::basket_rows_kernel<X, false, false><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, B, nullptr,
                                                                                              W, mv, rows, n);
        else if (limit_price)
          cfmm::basket_limit_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, R, W, mv, rows, n);
        else if (second)
          cfmm::basket_buy_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, R, d_kind.p, W, mv,
                                                                                rows, n);
        else
          cfmm::basket_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, G, act, R, W, mv, rows, n);
      },
      [&](int64_t r) { return basket_buy_row(basket_off, kind, r); },
      [&](int64_t r, auto&& visit) {
        visit(0, token_out[r] - 1);
        for (int64_t k = basket_off[r]; k < basket_off[r + 1]; ++k) visit(0, basket_token[k] - 1);
      });
}

cfmm_subgraph_opts subgraph_opts(const cfmm_subgraph_opts* in) {
  if (in) return *in;
  cfmm_subgraph_opts o;
  o.max_iter = 1000;
  o.max_fun = 4000;
  o.rtol = 1e-4;
  o.factr = 0.0;
  return o;
}

int basket_call(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                const int64_t* basket_token, const uint8_t* kind, const double* basket_amount, const double* limit,
                Allowed M, const cfmm_subgraph_opts* opts, cfmm_basket_out* out, const char* what) {
  const cfmm_subgraph_opts o = subgraph_opts(opts);
  int rc = check_basket(ctx, q, token_out, basket_off, basket_token, kind, basket_amount, limit, M, o, what);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (out && out->tok_off) out->tok_off[0] = 0;
    if (out && out->leg_off) out->leg_off[0] = 0;
    return CFMM_OK;
  }
  const cfmm_basket_out none{};
  return basket_orders(ctx, exec, q, token_out, basket_off, basket_token, kind, basket_amount, nullptr, limit, M, o,
                       out ? *out : none, what);
}

// cfmm_quote/execute_limit_orders: the basket calls' checks, then every limit price finite and >= 0,
// before anything runs; the rows through basket_orders; then each row's surplus on the host.
int limit_call(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_out, const int64_t* basket_off,
               const int64_t* basket_token, const double* basket_amount, const double* limit_price,
               const double* min_received, Allowed M, const cfmm_subgraph_opts* opts, cfmm_limit_out* out,
               const char* what) {
  const cfmm_subgraph_opts o = subgraph_opts(opts);
  int rc = check_basket(ctx, q, token_out, basket_off, basket_token, nullptr, basket_amount, min_received, M, o, what);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (out && out->tok_off) out->tok_off[0] = 0;
    if (out && out->leg_off) out->leg_off[0] = 0;
    return CFMM_OK;
  }
  if (!limit_price) return fail(ctx, CFMM_ERR_INVALID, "%s: null limit_price", what);
  for (int64_t r = 0; r < q; ++r)
    for (int64_t k = basket_off[r]; k < basket_off[r + 1]; ++k)
      if (!(std::isfinite(limit_price[k]) && limit_price[k] >= 0.0))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: limit price %g must be finite and >= 0", what,
                    (long long)r, limit_price[k]);
  cfmm_basket_out O{};
  if (out) {
    O.paid = out->paid;
    O.received = out->received;
    O.status = out->status;
    O.solver_status = out->solver_status;
    O.iterations = out->iterations;
    O.fun_evals = out->fun_evals;
    O.merit = out->merit;
    O.tok_off = out->tok_off;
    O.tok_cap = out->tok_cap;
    O.token = out->token;
    O.nu = out->nu;
    O.psi = out->psi;
    O.leg_off = out->leg_off;
    O.leg_cap = out->leg_cap;
    O.leg_type = out->leg_type;
    O.leg_pool = out->leg_pool;
    O.leg_delta = out->leg_delta;
    O.leg_lambda = out->leg_lambda;
  }
  // the surplus needs paid and received, whether or not the caller asked for them
  const bool surplus = out && out->surplus;
  std::vector<double> paid(surplus && !O.paid ? (size_t)basket_off[q] : 0),
      recv(surplus && !O.received ? (size_t)q : 0);
  if (!paid.empty()) O.paid = paid.data();
  if (!recv.empty()) O.received = recv.data();
  if ((rc = basket_orders(ctx, exec, q, token_out, basket_off, basket_token, nullptr, basket_amount, limit_price,
                          min_received, M, o, O, what)) != CFMM_OK)
    return rc;
  // S = received − Σ_k c_k·paid_k in entry order: a multiply, then a subtract (no fma)
  if (surplus)
    for (int64_t r = 0; r < q; ++r) {
      double s = O.received[r];
      for (int64_t k = basket_off[r]; k < basket_off[r + 1]; ++k) {
        const volatile double cp = limit_price[k] * O.paid[k];
        s = s - cp;
      }
      out->surplus[r] = s;
    }
  return CFMM_OK;
}

// ---- arbitrage against external prices over every pool among allowed tokens (price_arb_kernels.cuh)

// Every argument of cfmm_quote/execute_price_arbitrage, before anything runs.
int check_price_arb(cfmm_ctx* ctx, int64_t q, const double* price, const double* min_profit, const uint8_t* allowed,
                    const cfmm_subgraph_opts& o, const char* what) {
  Allowed M{allowed};
  int rc = check_row_opts(ctx, q, M, o, what);
  if (rc != CFMM_OK || q == 0) return rc;
  if (!price) return fail(ctx, CFMM_ERR_INVALID, "%s: null price", what);
  const int64_t nA = count_allowed(ctx, allowed);
  if (nA > CFMM_PRICE_ARB_MAX_TOKENS)
    return fail(ctx, CFMM_ERR_INVALID, "%s: %lld allowed tokens, more than %d", what, (long long)nA,
                CFMM_PRICE_ARB_MAX_TOKENS);
  for (int64_t r = 0; r < q; ++r) {
    bool any = false;
    for (int64_t k = 0; k < nA; ++k) {
      const double c = price[r * nA + k];
      if (!(std::isfinite(c) && c >= 0.0))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: price %g of allowed token %lld must be finite and >= 0",
                    what, (long long)r, c, (long long)k + 1);
      any |= c > 0.0;
    }
    if (!any) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: no positive price", what, (long long)r);
    if (min_profit && !(std::isfinite(min_profit[r]) && min_profit[r] >= 0.0))
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: min_profit %g must be finite and >= 0", what, (long long)r,
                  min_profit[r]);
  }
  return CFMM_OK;
}

// The family's outputs as row_orders takes them: the profit in received, no paid.
cfmm_subgraph_out price_arb_outputs(const cfmm_price_arb_out& out) {
  cfmm_subgraph_out O{};
  O.received = out.profit;
  O.status = out.status;
  O.solver_status = out.solver_status;
  O.iterations = out.iterations;
  O.fun_evals = out.fun_evals;
  O.merit = out.merit;
  O.tok_off = out.tok_off;
  O.tok_cap = out.tok_cap;
  O.token = out.token;
  O.nu = out.nu;
  O.psi = out.psi;
  O.leg_off = out.leg_off;
  O.leg_cap = out.leg_cap;
  O.leg_type = out.leg_type;
  O.leg_pool = out.leg_pool;
  O.leg_delta = out.leg_delta;
  O.leg_lambda = out.leg_lambda;
  return O;
}

// The profit of a price row through row_orders.
int price_arbitrage(cfmm_ctx* ctx, bool exec, int64_t q, const double* price, const double* min_profit,
                    const uint8_t* allowed, const cfmm_subgraph_opts& o, const cfmm_price_arb_out& out,
                    const char* what) {
  int rc;
  if ((rc = row_begin(ctx)) != CFMM_OK) return rc;
  std::vector<int64_t> tokA;  // the columns of price: the allowed tokens, ascending (0-based)
  for (int64_t t = 0; t < ctx->n_tokens; ++t)
    if (allowed[t]) tokA.push_back(t);
  const int64_t nA = (int64_t)tokA.size();
  DevBuf<double> d_price, d_min;
  CU_TRY(ctx, d_price.upload(price, (size_t)(q * nA)));
  CU_TRY(ctx, d_min.upload(min_profit, (size_t)q));
  int occ = 0;
  if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::price_arb_kernel<false>), {}, "price_arb_kernel", occ)) != CFMM_OK)
    return rc;
  int64_t uses = 0;  // the priced tokens over the call
  for (int64_t e = 0; e < q * nA; ++e) uses += price[e] > 0.0;
  cfmm::PriceArbRows R{d_price.p, d_min.p, o.max_iter, o.max_fun, o.rtol, o.factr};
  // a row's T lies in its priced tokens: rows whose priced tokens are disjoint share no pool
  return row_orders(
      ctx, exec, q, Allowed{allowed}, R, price_arb_outputs(out), occ, 0, 0, 0, 0, uses, false, what,
      [&](unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets*, cfmm::PairIndexView pv, cfmm::AdjView,
          const cfmm::BestPathGraph& G, const uint8_t* act, const cfmm::RowMasks&, int64_t* ntok, int64_t* npool) {
        cfmm::price_arb_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(pv, G, act, d_price.p, q, ntok, npool);
      },
      [&](auto exec_tag, bool, unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P,
          cfmm::PairIndexView pv, cfmm::AdjView, const cfmm::BestPathGraph& G, const uint8_t* act,
          const cfmm::RowMasks&, const cfmm::PriceArbRows& R, const cfmm::SubgraphWork& W, const cfmm::SplitMoved& mv, const int64_t* rows,
          int64_t n) {
        constexpr bool X = decltype(exec_tag)::value;
        cfmm::price_arb_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, G, act, R, W, mv, rows, n);
      },
      [](int64_t) { return false; },
      [&](int64_t r, auto&& visit) {
        for (int64_t k = 0; k < nA; ++k)
          if (price[r * nA + k] > 0.0) visit(0, tokA[(size_t)k]);
      });
}

int price_arb_call(cfmm_ctx* ctx, bool exec, int64_t q, const double* price, const double* min_profit,
                   const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_price_arb_out* out, const char* what) {
  const cfmm_subgraph_opts o = subgraph_opts(opts);
  int rc = check_price_arb(ctx, q, price, min_profit, allowed, o, what);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (out && out->tok_off) out->tok_off[0] = 0;
    if (out && out->leg_off) out->leg_off[0] = 0;
    return CFMM_OK;
  }
  const cfmm_price_arb_out none{};
  return price_arbitrage(ctx, exec, q, price, min_profit, allowed, o, out ? *out : none, what);
}

// ---- inventory rows: one token list per row, with holdings (price_arb_kernels.cuh, InvRule)

// Every argument of cfmm_quote/execute_price_arbitrage_rows, before anything runs.
int check_price_arb_rows(cfmm_ctx* ctx, int64_t q, Allowed& M, const double* price, const double* holding,
                         const double* min_profit, const cfmm_price_arb_opts& po, const char* what) {
  const cfmm_subgraph_opts o{po.max_iter, po.max_fun, po.rtol, po.factr};
  int rc = check_row_opts(ctx, q, M, o, what);
  if (rc != CFMM_OK) return rc;
  if (!(std::isfinite(po.atol) && po.atol >= 0.0))
    return fail(ctx, CFMM_ERR_INVALID, "%s: atol %g must be finite and >= 0", what, po.atol);
  if (q == 0) return CFMM_OK;
  if (!price) return fail(ctx, CFMM_ERR_INVALID, "%s: null price", what);
  for (int64_t r = 0; r < q; ++r) {
    const int64_t n = M.count(r);
    if (n < 1 || n > CFMM_PRICE_ARB_MAX_TOKENS)
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: %lld listed tokens, not 1..%d", what, (long long)r,
                  (long long)n, CFMM_PRICE_ARB_MAX_TOKENS);
    bool any = false;
    for (int64_t k = M.off[r]; k < M.off[r + 1]; ++k) {
      if (!(std::isfinite(price[k]) && price[k] >= 0.0))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: price %g of token %lld must be finite and >= 0", what,
                    (long long)r, price[k], (long long)M.tok[k]);
      if (holding && !(std::isfinite(holding[k]) && holding[k] >= 0.0))
        return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: holding %g of token %lld must be finite and >= 0", what,
                    (long long)r, holding[k], (long long)M.tok[k]);
      any |= price[k] > 0.0;
    }
    if (!any) return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: no positive price", what, (long long)r);
    if (min_profit && !(std::isfinite(min_profit[r]) && min_profit[r] >= 0.0))
      return fail(ctx, CFMM_ERR_INVALID, "%s: row %lld: min_profit %g must be finite and >= 0", what, (long long)r,
                  min_profit[r]);
  }
  return CFMM_OK;
}

int price_arb_rows_call(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* allow_off, const int64_t* allow_token,
                        const double* price, const double* holding, const double* min_profit,
                        const cfmm_price_arb_opts* opts, cfmm_price_arb_out* out, const char* what) {
  const cfmm_subgraph_opts d = subgraph_opts(nullptr);
  const cfmm_price_arb_opts po = opts ? *opts : cfmm_price_arb_opts{d.max_iter, d.max_fun, d.rtol, d.factr, 0.0};
  Allowed M{nullptr, true, allow_off, allow_token};
  int rc = check_price_arb_rows(ctx, q, M, price, holding, min_profit, po, what);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (out && out->tok_off) out->tok_off[0] = 0;
    if (out && out->leg_off) out->leg_off[0] = 0;
    return CFMM_OK;
  }
  if ((rc = row_begin(ctx)) != CFMM_OK) return rc;
  const size_t NL = (size_t)allow_off[q];
  DevBuf<double> d_price, d_hold, d_min;
  CU_TRY(ctx, d_price.upload(price, NL));
  CU_TRY(ctx, d_hold.upload(holding, NL));
  CU_TRY(ctx, d_min.upload(min_profit, (size_t)q));
  int occ = 0;
  if ((rc = row_occupancy(ctx, kernel_ptr(&cfmm::price_arb_rows_kernel<false>),
                          {kernel_ptr(&cfmm::price_arb_rows_plan_kernel), kernel_ptr(&cfmm::price_arb_rows_kernel<false>),
                           kernel_ptr(&cfmm::price_arb_rows_kernel<true>)},
                          "price_arb_rows_kernel", occ, cfmm::kRowGraphBytes)) != CFMM_OK)
    return rc;
  const cfmm_price_arb_out none{};
  cfmm::InvArbRows R{{d_price.p, d_min.p, po.max_iter, po.max_fun, po.rtol, po.factr}, d_hold.p, po.atol};
  // a row's T lies in its list: rows on disjoint lists share no pool
  return row_orders(
      ctx, exec, q, M, R, price_arb_outputs(out ? *out : none), occ, 0, 0, 0, 0, 0, true, what,
      [&](unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P, cfmm::PairIndexView pv, cfmm::AdjView A,
          const cfmm::BestPathGraph&, const uint8_t*, const cfmm::RowMasks& RM, int64_t* ntok, int64_t* npool) {
        cfmm::price_arb_rows_plan_kernel<<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, q, ntok, npool);
      },
      [&](auto exec_tag, bool, unsigned grid, size_t dyn, cudaStream_t st, const cfmm::PathSets* P,
          cfmm::PairIndexView pv, cfmm::AdjView A, const cfmm::BestPathGraph&, const uint8_t*,
          const cfmm::RowMasks& RM, const cfmm::InvArbRows& R, const cfmm::SubgraphWork& W, const cfmm::SplitMoved& mv,
          const int64_t* rows, int64_t n) {
        constexpr bool X = decltype(exec_tag)::value;
        cfmm::price_arb_rows_kernel<X><<<grid, cfmm::kSubgraphThreads, dyn, st>>>(P, pv, A, RM, R, W, mv, rows, n);
      },
      [](int64_t) { return false; }, [](int64_t, auto&&) {});
}

}  // namespace

namespace {

int subgraph_call(cfmm_ctx* ctx, bool exec, int64_t q, const int64_t* token_in, const int64_t* token_out,
                  const uint8_t* kind, const double* amount, const double* limit, Allowed M,
                  const cfmm_subgraph_opts* opts, cfmm_subgraph_out* out, const char* what) {
  const cfmm_subgraph_opts o = subgraph_opts(opts);
  int rc = check_subgraph(ctx, q, token_in, token_out, kind, amount, limit, M, o, what);
  if (rc != CFMM_OK) return rc;
  if (q == 0) {
    if (out && out->tok_off) out->tok_off[0] = 0;
    if (out && out->leg_off) out->leg_off[0] = 0;
    return CFMM_OK;
  }
  return subgraph_orders(ctx, exec, q, token_in, token_out, kind, amount, limit, M, o, out);
}

}  // namespace

int cfmm_quote_subgraph_swap_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                                    const uint8_t* kind, const double* amount, const uint8_t* allowed,
                                    const cfmm_subgraph_opts* opts, cfmm_subgraph_out* out) {
  return subgraph_call(ctx, false, q, token_in, token_out, kind, amount, nullptr, Allowed{allowed}, opts, out,
                       "quote_subgraph_orders");
}

int cfmm_execute_subgraph_swap_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                                      const uint8_t* kind, const double* amount, const double* limit,
                                      const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_subgraph_out* out) {
  return subgraph_call(ctx, true, q, token_in, token_out, kind, amount, limit, Allowed{allowed}, opts, out,
                       "execute_subgraph_orders");
}

int cfmm_quote_subgraph_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                               const double* amount, const uint8_t* allowed, const cfmm_subgraph_opts* opts,
                               cfmm_subgraph_out* out) {
  return cfmm_quote_subgraph_swap_orders(ctx, q, token_in, token_out, nullptr, amount, allowed, opts, out);
}

int cfmm_execute_subgraph_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                                 const double* amount, const double* limit, const uint8_t* allowed,
                                 const cfmm_subgraph_opts* opts, cfmm_subgraph_out* out) {
  return cfmm_execute_subgraph_swap_orders(ctx, q, token_in, token_out, nullptr, amount, limit, allowed, opts, out);
}

int cfmm_quote_basket_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                             const int64_t* basket_token, const double* basket_amount, const uint8_t* allowed,
                             const cfmm_subgraph_opts* opts, cfmm_basket_out* out) {
  return basket_call(ctx, false, q, token_out, basket_off, basket_token, nullptr, basket_amount, nullptr,
                     Allowed{allowed}, opts, out, "quote_basket_orders");
}

int cfmm_execute_basket_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                               const int64_t* basket_token, const double* basket_amount, const double* limit,
                               const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_basket_out* out) {
  return basket_call(ctx, true, q, token_out, basket_off, basket_token, nullptr, basket_amount, limit,
                     Allowed{allowed}, opts, out, "execute_basket_orders");
}

int cfmm_quote_basket_swap_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                                  const int64_t* basket_token, const uint8_t* entry_kind, const double* basket_amount,
                                  const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_basket_out* out) {
  return basket_call(ctx, false, q, token_out, basket_off, basket_token, entry_kind, basket_amount, nullptr,
                     Allowed{allowed}, opts, out, "quote_basket_swap_orders");
}

int cfmm_execute_basket_swap_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                                    const int64_t* basket_token, const uint8_t* entry_kind,
                                    const double* basket_amount, const double* limit, const uint8_t* allowed,
                                    const cfmm_subgraph_opts* opts, cfmm_basket_out* out) {
  return basket_call(ctx, true, q, token_out, basket_off, basket_token, entry_kind, basket_amount, limit,
                     Allowed{allowed}, opts, out, "execute_basket_swap_orders");
}

int cfmm_quote_limit_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                            const int64_t* basket_token, const double* basket_amount, const double* limit_price,
                            const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_limit_out* out) {
  return limit_call(ctx, false, q, token_out, basket_off, basket_token, basket_amount, limit_price, nullptr,
                    Allowed{allowed}, opts, out, "quote_limit_orders");
}

int cfmm_execute_limit_orders(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                              const int64_t* basket_token, const double* basket_amount, const double* limit_price,
                              const double* min_received, const uint8_t* allowed, const cfmm_subgraph_opts* opts,
                              cfmm_limit_out* out) {
  return limit_call(ctx, true, q, token_out, basket_off, basket_token, basket_amount, limit_price, min_received,
                    Allowed{allowed}, opts, out, "execute_limit_orders");
}

// ---- per-row masks: the calls above with one allowed list per row (the rows' own slot graphs)

int cfmm_quote_subgraph_swap_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_in, const int64_t* token_out,
                                         const uint8_t* kind, const double* amount, const int64_t* allow_off,
                                         const int64_t* allow_token, const cfmm_subgraph_opts* opts,
                                         cfmm_subgraph_out* out) {
  return subgraph_call(ctx, false, q, token_in, token_out, kind, amount, nullptr, Allowed{nullptr, true, allow_off, allow_token},
                       opts, out, "quote_subgraph_orders_rows");
}

int cfmm_execute_subgraph_swap_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_in,
                                           const int64_t* token_out, const uint8_t* kind, const double* amount,
                                           const double* limit, const int64_t* allow_off, const int64_t* allow_token,
                                           const cfmm_subgraph_opts* opts, cfmm_subgraph_out* out) {
  return subgraph_call(ctx, true, q, token_in, token_out, kind, amount, limit, Allowed{nullptr, true, allow_off, allow_token},
                       opts, out, "execute_subgraph_orders_rows");
}

int cfmm_quote_basket_swap_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                                       const int64_t* basket_token, const uint8_t* entry_kind,
                                       const double* basket_amount, const int64_t* allow_off,
                                       const int64_t* allow_token, const cfmm_subgraph_opts* opts,
                                       cfmm_basket_out* out) {
  return basket_call(ctx, false, q, token_out, basket_off, basket_token, entry_kind, basket_amount, nullptr,
                     Allowed{nullptr, true, allow_off, allow_token}, opts, out, "quote_basket_swap_orders_rows");
}

int cfmm_execute_basket_swap_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_out,
                                         const int64_t* basket_off, const int64_t* basket_token,
                                         const uint8_t* entry_kind, const double* basket_amount, const double* limit,
                                         const int64_t* allow_off, const int64_t* allow_token,
                                         const cfmm_subgraph_opts* opts, cfmm_basket_out* out) {
  return basket_call(ctx, true, q, token_out, basket_off, basket_token, entry_kind, basket_amount, limit,
                     Allowed{nullptr, true, allow_off, allow_token}, opts, out, "execute_basket_swap_orders_rows");
}

int cfmm_quote_limit_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                                 const int64_t* basket_token, const double* basket_amount, const double* limit_price,
                                 const int64_t* allow_off, const int64_t* allow_token, const cfmm_subgraph_opts* opts,
                                 cfmm_limit_out* out) {
  return limit_call(ctx, false, q, token_out, basket_off, basket_token, basket_amount, limit_price, nullptr,
                    Allowed{nullptr, true, allow_off, allow_token}, opts, out, "quote_limit_orders_rows");
}

int cfmm_execute_limit_orders_rows(cfmm_ctx* ctx, int64_t q, const int64_t* token_out, const int64_t* basket_off,
                                   const int64_t* basket_token, const double* basket_amount,
                                   const double* limit_price, const double* min_received, const int64_t* allow_off,
                                   const int64_t* allow_token, const cfmm_subgraph_opts* opts, cfmm_limit_out* out) {
  return limit_call(ctx, true, q, token_out, basket_off, basket_token, basket_amount, limit_price, min_received,
                    Allowed{nullptr, true, allow_off, allow_token}, opts, out, "execute_limit_orders_rows");
}

int cfmm_quote_price_arbitrage(cfmm_ctx* ctx, int64_t q, const double* price, const uint8_t* allowed,
                               const cfmm_subgraph_opts* opts, cfmm_price_arb_out* out) {
  return price_arb_call(ctx, false, q, price, nullptr, allowed, opts, out, "quote_price_arbitrage");
}

int cfmm_execute_price_arbitrage(cfmm_ctx* ctx, int64_t q, const double* price, const double* min_profit,
                                 const uint8_t* allowed, const cfmm_subgraph_opts* opts, cfmm_price_arb_out* out) {
  return price_arb_call(ctx, true, q, price, min_profit, allowed, opts, out, "execute_price_arbitrage");
}

int cfmm_quote_price_arbitrage_rows(cfmm_ctx* ctx, int64_t q, const int64_t* allow_off, const int64_t* allow_token,
                                    const double* price, const double* holding, const cfmm_price_arb_opts* opts,
                                    cfmm_price_arb_out* out) {
  return price_arb_rows_call(ctx, false, q, allow_off, allow_token, price, holding, nullptr, opts, out,
                             "quote_price_arbitrage_rows");
}

int cfmm_execute_price_arbitrage_rows(cfmm_ctx* ctx, int64_t q, const int64_t* allow_off, const int64_t* allow_token,
                                      const double* price, const double* holding, const double* min_profit,
                                      const cfmm_price_arb_opts* opts, cfmm_price_arb_out* out) {
  return price_arb_rows_call(ctx, true, q, allow_off, allow_token, price, holding, min_profit, opts, out,
                             "execute_price_arbitrage_rows");
}

// ---- UniV3 liquidity changes: mint / burn rows, ladders that grow (univ3_state.cuh) ----------
namespace {

int check_liquidity_rows(cfmm_ctx* ctx, int64_t q, const int64_t* pool, const double* range, const double* dL) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if (q < 0) return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: negative row count");
  if (q > 0 && (!pool || !range || !dL)) return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: null array argument");
  const int64_t m = type_pools(ctx, CFMM_POOL_UNIV3);
  for (int64_t j = 0; j < q; ++j) {
    if (pool[j] < 0 || pool[j] >= m)
      return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: row %lld: pool %lld outside 0..%lld", (long long)j,
                  (long long)pool[j], (long long)m);
    const double lo = range[2 * j], hi = range[2 * j + 1];
    if (!std::isfinite(lo) || !std::isfinite(hi) || !(lo > 0.0) || !(lo < hi))
      return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: row %lld: range (%g, %g) needs 0 < lo < hi, both finite",
                  (long long)j, lo, hi);
    if (!std::isfinite(dL[j]) || dL[j] == 0.0)
      return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: row %lld: dL %g must be finite and != 0", (long long)j,
                  dL[j]);
  }
  return CFMM_OK;
}

// One set's part of a cfmm_modify_univ3_liquidity call: the touched pools' new ladders (stage A,
// listing order) and, when tick counts change, the set's new CSR arrays (stage B).
struct LiquidityStage {
  PoolSet* s = nullptr;
  Groups g;
  std::vector<int64_t> new_nt, cum;   // per touched pool: new tick count, listing offsets [n + 1]
  std::vector<double> top;            // per touched pool: its highest candidate boundary
  int64_t growth = 0;                 // ticks added to the set
  DevBuf<int64_t> d_pos, d_row_off, d_rows, d_cum;
  DevBuf<double> d_lower, d_liq;      // stage-A ladders
  DevBuf<double> n_lower, n_liq, n_tickdata;  // stage B, growth > 0 only
  DevBuf<int2> n_tick;
};

// Stage A of one set: merge, inherit, apply; nothing of the set is written.
int liquidity_stage(cfmm_ctx* ctx, LiquidityStage& st, const SetRows& r, const double* range,
                    const double* d_range, const double* d_dL, unsigned long long* d_bad) {
  PoolSet& s = *st.s;
  st.g = group_by_pool(r, s.m_padded);
  const int64_t n = (int64_t)st.g.key.size();
  std::vector<int64_t> cand_off(1, 0);
  std::vector<double> cand;
  st.top.resize((size_t)n);
  for (int64_t j = 0; j < n; ++j) {
    const size_t b = cand.size();
    for (int64_t k = st.g.off[(size_t)j]; k < st.g.off[(size_t)j + 1]; ++k) {
      const int64_t row = st.g.rows[(size_t)k];
      cand.push_back(range[2 * row]);
      cand.push_back(range[2 * row + 1]);
    }
    std::sort(cand.begin() + b, cand.end(), std::greater<double>());
    cand.erase(std::unique(cand.begin() + b, cand.end()), cand.end());
    st.top[(size_t)j] = cand[b];
    cand_off.push_back((int64_t)cand.size());
  }
  DevBuf<int64_t> d_cand_off, d_nt;
  DevBuf<double> d_cand;
  CU_TRY(ctx, st.d_pos.upload(st.g.key));
  CU_TRY(ctx, st.d_row_off.upload(st.g.off));
  CU_TRY(ctx, st.d_rows.upload(st.g.rows));
  CU_TRY(ctx, d_cand_off.upload(cand_off));
  CU_TRY(ctx, d_cand.upload(cand));
  CU_TRY(ctx, d_nt.alloc((size_t)n));
  const cfmm::Univ3State u = univ3_state(s);
  const int threads = 256;
  const unsigned pool_blocks = (unsigned)((n + threads - 1) / threads);
  int rc;
  if ((rc = launch(ctx, kNoProf, 1, [&] {
         cfmm::univ3_liq_ladder_kernel<<<pool_blocks, threads, 0, ctx->stream>>>(u, st.d_pos.p, d_cand_off.p, d_cand.p,
                                                                               n, d_nt.p, nullptr, nullptr, nullptr);
       })) != CFMM_OK)
    return rc;
  st.new_nt.resize((size_t)n);
  CU_TRY(ctx, read_back(ctx, st.new_nt.data(), d_nt.p, (size_t)n));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  st.cum.assign((size_t)n + 1, 0);
  for (int64_t j = 0; j < n; ++j) {
    st.cum[(size_t)j + 1] = st.cum[(size_t)j] + st.new_nt[(size_t)j];
    st.growth += st.new_nt[(size_t)j] - s.n_ticks[(size_t)s.order[(size_t)st.g.key[(size_t)j]]];
  }
  if (s.total_ticks + st.growth > (int64_t)0x7fffffff)
    return fail(ctx, CFMM_ERR_INVALID, "modify_univ3_liquidity: more than 2^31-1 ticks in one pool set");
  const int64_t n_ticks = st.cum[(size_t)n];
  CU_TRY(ctx, st.d_cum.upload(st.cum));
  CU_TRY(ctx, st.d_lower.alloc((size_t)n_ticks));
  CU_TRY(ctx, st.d_liq.alloc((size_t)n_ticks));
  if ((rc = launch(ctx, kNoProf, 2, [&] {
         cfmm::univ3_liq_ladder_kernel<<<pool_blocks, threads, 0, ctx->stream>>>(
             u, st.d_pos.p, d_cand_off.p, d_cand.p, n, nullptr, st.d_cum.p, st.d_lower.p, st.d_liq.p);
         cfmm::univ3_liq_apply_kernel<<<(unsigned)((n_ticks + threads - 1) / threads), threads, 0, ctx->stream>>>(
             st.d_cum.p, n, n_ticks, st.d_row_off.p, st.d_rows.p, d_range, d_dL, st.d_lower.p, st.d_liq.p, d_bad);
       })) != CFMM_OK)
    return rc;
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));  // (the candidate arrays are freed on return)
  return CFMM_OK;
}

// Stage B allocations of one set whose tick counts change: all of them before anything is
// released or written, so that a failure leaves the set as it was.
cudaError_t liquidity_alloc(LiquidityStage& st) {
  const PoolSet& s = *st.s;
  const size_t total = (size_t)(s.total_ticks + st.growth);
  cudaError_t e = st.n_lower.alloc(total);
  if (e == cudaSuccess) e = st.n_liq.alloc(total);
  if (e == cudaSuccess) e = st.n_tick.alloc((size_t)s.m);
  if (e == cudaSuccess) e = st.n_tickdata.alloc(total * cfmm::kTickStride);
  return e;
}

// Stage B of one set: commit the new ladders and rebuild the tick records.
int liquidity_commit(cfmm_ctx* ctx, LiquidityStage& st) {
  PoolSet& s = *st.s;
  const int64_t n = (int64_t)st.g.key.size();
  const int threads = 256;
  if (st.growth == 0) {  // same tick counts: the new liquidities go through the update path
    CU_TRY(ctx, univ3_rebuild(ctx, s, st.d_pos.p, st.d_cum.p, n, st.cum[(size_t)n], nullptr, st.d_liq.p, false));
  } else {
    std::vector<int64_t> shift((size_t)n + 1, 0);
    for (int64_t j = 0; j < n; ++j)
      shift[(size_t)j + 1] = shift[(size_t)j] + st.new_nt[(size_t)j] - s.n_ticks[(size_t)s.order[(size_t)st.g.key[(size_t)j]]];
    DevBuf<int64_t> d_shift;
    CU_TRY(ctx, d_shift.upload(shift));
    const int64_t total = s.total_ticks + st.growth;
    const int rc = launch(ctx, kNoProf, 2, [&] {
      cfmm::univ3_splice_offsets_kernel<<<(unsigned)((s.m + threads - 1) / threads), threads, 0, ctx->stream>>>(
          s.d_tick.p, st.n_tick.p, s.m, st.d_pos.p, d_shift.p, n);
      cfmm::univ3_splice_ticks_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, ctx->stream>>>(
          s.d_tick.p, st.n_tick.p, s.m, total, st.d_pos.p, st.d_cum.p, n, st.d_lower.p, st.d_liq.p, s.d_lower.p,
          s.d_liq.p, st.n_lower.p, st.n_liq.p);
    });
    if (rc != CFMM_OK) return rc;
    CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    std::swap(s.d_lower, st.n_lower);
    std::swap(s.d_liq, st.n_liq);
    std::swap(s.d_tick, st.n_tick);
    std::swap(s.d_tickdata, st.n_tickdata);
    s.total_ticks = total;
    CU_TRY(ctx, univ3_rebuild(ctx, s, nullptr, nullptr, s.m, s.total_ticks, nullptr, nullptr, true));
  }
  for (int64_t j = 0; j < n; ++j) {
    const int64_t i = s.order[(size_t)st.g.key[(size_t)j]];
    s.n_ticks[(size_t)i] = st.new_nt[(size_t)j];
    s.first_lower[(size_t)i] = std::max(s.first_lower[(size_t)i], st.top[(size_t)j]);
  }
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  return CFMM_OK;
}

}  // namespace

int cfmm_modify_univ3_liquidity(cfmm_ctx* ctx, int64_t q, const int64_t* pool, const double* range,
                                const double* dL) {
  int rc = check_liquidity_rows(ctx, q, pool, range, dL);
  if (rc != CFMM_OK || q == 0) return rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  DevBuf<double> d_range, d_dL;
  DevBuf<unsigned long long> d_bad;
  CU_TRY(ctx, d_range.upload(range, (size_t)(2 * q)));
  CU_TRY(ctx, d_dL.upload(dL, (size_t)q));
  CU_TRY(ctx, d_bad.alloc(1));
  CU_TRY(ctx, cudaMemsetAsync(d_bad.p, 0xff, sizeof(unsigned long long), ctx->stream));
  // stage A for every set first: a row that fails anywhere rejects the whole call
  std::vector<std::unique_ptr<LiquidityStage>> stages;
  for (SetRows& r : rows_by_set(ctx, CFMM_POOL_UNIV3, q, pool)) {
    if (r.row.empty()) continue;
    stages.push_back(std::make_unique<LiquidityStage>());
    stages.back()->s = r.s;
    if ((rc = liquidity_stage(ctx, *stages.back(), r, range, d_range.p, d_dL.p, d_bad.p)) != CFMM_OK) return rc;
  }
  unsigned long long bad = 0;
  CU_TRY(ctx, read_back(ctx, &bad, d_bad.p, 1));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
  if (bad != ~0ull)
    return fail(ctx, CFMM_ERR_INVALID,
                "modify_univ3_liquidity: row %lld leaves a tick it adds to with liquidity < 0 or not finite",
                (long long)bad);
  for (auto& st : stages) {
    if (st->growth == 0) continue;
    const cudaError_t e = liquidity_alloc(*st);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();  // (an allocation failure is not sticky: clear it for later calls)
      return fail(ctx, e == cudaErrorMemoryAllocation ? CFMM_ERR_NOMEM : CFMM_ERR_CUDA,
                  "modify_univ3_liquidity: allocating the grown tick arrays failed: %s", cudaGetErrorString(e));
    }
  }
  ctx->state_version++;
  for (auto& st : stages)
    if ((rc = liquidity_commit(ctx, *st)) != CFMM_OK) return rc;
  return CFMM_OK;
}

int cfmm_get_univ3_ticks(cfmm_ctx* ctx, int64_t first, int64_t count, int64_t* tick_off, double* lower_ticks,
                         double* liquidity) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_range(ctx, CFMM_POOL_UNIV3, first, count, "get_univ3_ticks")) != CFMM_OK) return rc;
  if (!tick_off) return fail(ctx, CFMM_ERR_INVALID, "get_univ3_ticks: null tick_off");
  tick_off[0] = 0;
  if (count == 0) return CFMM_OK;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  int64_t base = 0;
  for (const Span& sp : split_range(ctx, CFMM_POOL_UNIV3, first, count)) {
    PoolSet& s = *sp.s;
    ensure_pos_of(s);
    std::vector<int64_t> pos(s.pos_of.begin() + sp.first, s.pos_of.begin() + sp.first + sp.count);
    std::vector<int64_t> cum((size_t)sp.count + 1, 0);
    for (int64_t j = 0; j < sp.count; ++j) {
      cum[(size_t)j + 1] = cum[(size_t)j] + s.n_ticks[(size_t)(sp.first + j)];
      tick_off[sp.offset + j + 1] = base + cum[(size_t)j + 1];
    }
    const int64_t n_ticks = cum[(size_t)sp.count];
    if (lower_ticks || liquidity) {
      DevBuf<int64_t> d_pos, d_cum;
      DevBuf<double> d_lo, d_lq;
      CU_TRY(ctx, d_pos.upload(pos));
      CU_TRY(ctx, d_cum.upload(cum));
      CU_TRY(ctx, d_lo.alloc((size_t)n_ticks));
      CU_TRY(ctx, d_lq.alloc((size_t)n_ticks));
      const int threads = 256;
      if ((rc = launch(ctx, kNoProf, 1, [&] {
             cfmm::univ3_gather_ticks_kernel<<<(unsigned)((n_ticks + threads - 1) / threads), threads, 0,
                                               ctx->stream>>>(univ3_state(s), d_pos.p, d_cum.p, sp.count, n_ticks,
                                                              d_lo.p, d_lq.p);
           })) != CFMM_OK)
        return rc;
      CU_TRY(ctx, read_back(ctx, lower_ticks ? lower_ticks + base : nullptr, d_lo.p, (size_t)n_ticks));
      CU_TRY(ctx, read_back(ctx, liquidity ? liquidity + base : nullptr, d_lq.p, (size_t)n_ticks));
      CU_TRY(ctx, cudaStreamSynchronize(ctx->stream));
    }
    base += n_ticks;
  }
  return CFMM_OK;
}

int cfmm_compact(cfmm_ctx* ctx) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  if ((rc = use_stream(ctx, ctx->stream)) != CFMM_OK) return rc;
  for (int t = 0; t < 3; ++t) {
    PoolSet &live = ctx->sets[t], &tail = ctx->tails[t];
    if (live.m + tail.m == 0) continue;
    auto next = std::make_unique<PoolSet>();
    if ((rc = read_back(ctx, t, live, *next)) != CFMM_OK) return rc;
    if ((rc = read_back(ctx, t, tail, *next)) != CFMM_OK) return rc;
    if ((rc = install_set(ctx, t, live, *next, false)) != CFMM_OK) return rc;
    auto empty = std::make_unique<PoolSet>();
    tail.release();
    std::swap(tail, *empty);
  }
  membership_changed(ctx);
  return calibrate(ctx);
}

// Test hook: pools per compact record of the next gradient-only sweep of the main set (see
// compact_record_of; ProductTwoCoin only, 0 for the other types).
int cfmm_debug_compact_record(cfmm_ctx* ctx, int type, int64_t* pools_per_record) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if (!pools_per_record) return fail(ctx, CFMM_ERR_INVALID, "null output");
  const PoolSet& s = ctx->sets[type];
  *pools_per_record = type == CFMM_POOL_PRODUCT && s.tma_ok && ctx->use_tma ? compact_record_of(ctx, s) : 0;
  return CFMM_OK;
}

// Test hook: keep rule of the next gradient-only TMA sweep of the main ProductTwoCoin set (see
// l2_keep_of; 0 for the other types and for sweeps that do not stream the 192-pool records).
int cfmm_debug_l2_keep(cfmm_ctx* ctx, int type, int64_t* keep) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if (!keep) return fail(ctx, CFMM_ERR_INVALID, "null output");
  const PoolSet& s = ctx->sets[type];
  *keep = 0;
  if (type == CFMM_POOL_PRODUCT && s.tma_ok && ctx->use_tma && compact_record_of(ctx, s) == 192)
    *keep = l2_keep_of(ctx, s.n_recs * cfmm::tma_chunk_bytes_c<0, true, cfmm::kTmaL6>());
  return CFMM_OK;
}

// Test hook: info[8] = {main-set pools, tail pools, main-set padded length, TMA layout built,
// fixed-point Ψ slice allowed, compact stream allowed, every reserve in the guard-free range,
// retired pools} of one pool type.
int cfmm_debug_pool_set_info(cfmm_ctx* ctx, int type, int64_t* info) {
  int rc = ready(ctx);
  if (rc != CFMM_OK) return rc;
  if ((rc = check_type(ctx, type)) != CFMM_OK) return rc;
  if (!info) return fail(ctx, CFMM_ERR_INVALID, "null info array");
  const PoolSet &s = ctx->sets[type], &t = ctx->tails[type];
  int64_t retired = 0;
  for (const PoolSet* p : {&s, &t})
    for (uint8_t r : p->retired) retired += r;
  const int64_t v[8] = {s.m, t.m, s.m_padded, s.tma_ok, s.fixed_ok, s.compact_ok, s.in_fast_range, retired};
  memcpy(info, v, sizeof(v));
  return CFMM_OK;
}


int cfmm_set_option(cfmm_ctx* ctx, const char* key, int64_t value) {
  if (!ctx || !key) return CFMM_ERR_INVALID;
  ctx->state_version++;  // captured sweep graphs are stale
  if (!strcmp(key, "sweep_graphs")) {
    ctx->use_graphs = value != 0;
    return CFMM_OK;
  }
  if (!strcmp(key, "exact")) {
    ctx->exact = value != 0;
  } else if (!strcmp(key, "blocks_per_sm")) {
    if (value < 0 || value > 32) return fail(ctx, CFMM_ERR_INVALID, "blocks_per_sm out of range");
    ctx->blocks_per_sm = (int)value;
  } else if (!strcmp(key, "tma_variant")) {
    if (value < -1 || value > 0) return fail(ctx, CFMM_ERR_INVALID, "tma_variant must be 0 (bucketed layout, TMA kernel) or -1");
    if (ctx->finalized)
      return fail(ctx, CFMM_ERR_STATE, "tma_variant fixes the pool layout: set it before cfmm_finalize");
    ctx->tma_variant = (int)value;
  } else if (!strcmp(key, "orient_by_degree")) {
    if (ctx->finalized)
      return fail(ctx, CFMM_ERR_STATE, "orient_by_degree fixes the pool layout: set it before cfmm_finalize");
    ctx->orient_by_degree = value < 0 ? -1 : (value != 0);
  } else if (!strcmp(key, "psi_fixed_point")) {
    ctx->psi_fixed_point = value != 0;
  } else if (!strcmp(key, "compact_stream")) {
    ctx->compact_stream = value != 0;
  } else if (!strcmp(key, "compact_record")) {
    if (value != 0 && value != 96 && value != 192) return fail(ctx, CFMM_ERR_INVALID, "compact_record: 0 (by set size), 96 or 192");
    ctx->compact_record = (int)value;
  } else if (!strcmp(key, "l2_keep")) {
    if (value < -1 || value > (1 << 20)) return fail(ctx, CFMM_ERR_INVALID, "l2_keep: -1 (by L2 size), 0 (no hints) or records per CTA range");
    ctx->l2_keep = (int)value;
  } else if (!strcmp(key, "geomean_tma")) {
    ctx->geomean_tma = value != 0;
  } else if (!strcmp(key, "balance")) {
    ctx->balance = value != 0;
  } else if (!strcmp(key, "trace")) {
    // measurement only: 1 = every TMA sweep records per-CTA phase timestamps (cfmm_debug_read_trace)
    cudaSetDevice(ctx->device);
    if (value) {
      CU_TRY(ctx, ctx->d_trace.alloc((size_t)8 * 4096));
      CU_TRY(ctx, cudaMemset(ctx->d_trace.p, 0, 8 * 4096 * sizeof(unsigned long long)));
      CU_TRY(ctx, cudaStreamSynchronize(cudaStreamLegacy));
    } else {
      cudaStreamSynchronize(ctx->stream);
      ctx->d_trace.release();
    }
  } else if (!strcmp(key, "fused_exchange")) {
    ctx->fused_exchange = value != 0;
  } else if (!strcmp(key, "grid_waves")) {
    ctx->grid_waves = (int)value;
    ctx->state_version++;
  } else if (!strcmp(key, "coop_launch")) {
    ctx->coop_launch = value != 0;
  } else if (!strcmp(key, "exchange_bypass")) {
    ctx->exchange_bypass = value != 0;
  } else if (!strcmp(key, "exchange_two_shot")) {  // the two LL forms (peer_exchange.cuh)
    ctx->exchange_protocol = value != 0 ? 2 : 1;
    ctx->comm.force_mode(ctx->exchange_protocol);
    ctx->state_version++;
  } else if (!strcmp(key, "exchange_protocol")) {
    if (value < 0 || value > 3) return fail(ctx, CFMM_ERR_INVALID, "exchange_protocol: 0 (auto), 1, 2 or 3");
    ctx->exchange_protocol = (int)value;
    ctx->comm.force_mode(ctx->exchange_protocol);
    ctx->state_version++;
  } else if (!strcmp(key, "sweep_events")) {
    ctx->sweep_events = value != 0;
  } else if (!strcmp(key, "gradient_math")) {
    ctx->gradient_math = value != 0;
  } else if (!strcmp(key, "geomean_log2")) {
    ctx->geomean_log2 = value != 0;
  } else if (!strcmp(key, "use_tma")) {
    ctx->use_tma = value != 0;
  } else if (!strcmp(key, "debug_skip")) {
    ctx->debug_skip = (int)(value & 7);
  } else if (!strcmp(key, "profile")) {
    // value = number of kernel launches to time with CUDA events (0 = off)
    if (value < 0 || value > (1 << 22)) return fail(ctx, CFMM_ERR_INVALID, "profile out of range");
    cudaSetDevice(ctx->device);
    for (auto e : ctx->prof.ev) cudaEventDestroy(e);
    ctx->prof.ev.assign((size_t)value * 2, nullptr);
    ctx->prof.type.assign((size_t)value, -1);
    ctx->prof.used = 0;
    for (auto& e : ctx->prof.ev) CU_TRY(ctx, cudaEventCreate(&e));
  } else {
    return fail(ctx, CFMM_ERR_INVALID, "unknown option '%s'", key);
  }
  return CFMM_OK;
}

int cfmm_profile_read(cfmm_ctx* ctx, int type, double* total_ms, int64_t* launches) {
  if (!ctx || !total_ms || !launches) return CFMM_ERR_INVALID;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  double sum = 0.0;
  int64_t cnt = 0;
  for (size_t i = 0; i < ctx->prof.used; ++i) {
    if (ctx->prof.type[i] != type) continue;
    CU_TRY(ctx, cudaEventSynchronize(ctx->prof.ev[2 * i + 1]));
    float ms = 0.f;
    CU_TRY(ctx, cudaEventElapsedTime(&ms, ctx->prof.ev[2 * i], ctx->prof.ev[2 * i + 1]));
    sum += ms;
    ++cnt;
  }
  *total_ms = sum;
  *launches = cnt;
  return CFMM_OK;
}

int cfmm_profile_read_times(cfmm_ctx* ctx, int type, float* ms_out, int64_t cap, int64_t* n_out) {
  if (!ctx || !n_out || cap < 0 || (cap > 0 && !ms_out)) return CFMM_ERR_INVALID;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  int64_t cnt = 0;
  for (size_t i = 0; i < ctx->prof.used; ++i) {
    if (ctx->prof.type[i] != type) continue;
    if (cnt < cap) {
      CU_TRY(ctx, cudaEventSynchronize(ctx->prof.ev[2 * i + 1]));
      CU_TRY(ctx, cudaEventElapsedTime(&ms_out[cnt], ctx->prof.ev[2 * i], ctx->prof.ev[2 * i + 1]));
    }
    ++cnt;
  }
  *n_out = cnt;
  return CFMM_OK;
}

int cfmm_profile_reset(cfmm_ctx* ctx) {
  if (!ctx) return CFMM_ERR_INVALID;
  ctx->prof.used = 0;
  return CFMM_OK;
}

void* cfmm_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
  return p;
}
void cfmm_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

// Test hook (no CUDA call): the device layout finalize would build for m
// ProductTwoCoin pools.  info[6] = {m_padded, nb, bucketed, skewed, chunk, variant};
// order_out [cap] (device position -> pool index, -1 = padding), chunk_bucket_out
// [cap / chunk], swapped_out [m] are filled when cap >= m_padded (call with cap = 0 first).
int cfmm_debug_product_layout(int64_t n_tokens, int64_t m, const int64_t* Ai, int orient,
                              int variant, int64_t cap, int64_t* order_out,
                              int32_t* chunk_bucket_out, uint8_t* swapped_out, int64_t* info) {
  if (!Ai || !info || m < 0 || n_tokens < 2 || variant < -1 || variant > 0)
    return CFMM_ERR_INVALID;
  for (int64_t i = 0; i < 2 * m; ++i)
    if (Ai[i] < 1 || Ai[i] > n_tokens) return CFMM_ERR_INVALID;
  cfmm_ctx fake;
  fake.n_tokens = n_tokens;
  fake.tma_variant = variant;
  fake.orient_by_degree = orient;
  const cfmm::PoolLayout lay = layout_for(&fake, CFMM_POOL_PRODUCT, Ai, m, true);
  info[0] = lay.m_padded;
  info[1] = lay.nb;
  info[2] = lay.bucketed;
  info[3] = lay.skewed;
  info[4] = lay.bucketed ? cfmm::kTmaChunk : 0;
  info[5] = variant;
  if (cap >= lay.m_padded && order_out) {
    for (int64_t p = 0; p < lay.m_padded; ++p) order_out[p] = lay.order[(size_t)p];
    if (chunk_bucket_out)
      for (size_t t = 0; t < lay.tile_bucket.size(); ++t) chunk_bucket_out[t] = lay.tile_bucket[t];
    if (swapped_out)
      for (int64_t i = 0; i < m; ++i) swapped_out[i] = lay.swapped[(size_t)i];
  }
  return CFMM_OK;
}

// Measurement hook: the per-CTA phase timestamps (ns, %globaltimer) of the last TMA sweep
// recorded under option "trace": out[8 * grid] = per CTA {entry, slice ready, own range done,
// all chunks done, partials flushed, exit, grid barrier passed (fused exchange), SM id << 32 |
// chunks processed}.
int cfmm_debug_read_trace(cfmm_ctx* ctx, uint64_t* out, int64_t cap_ctas, int64_t* grid_out) {
  if (!ctx || !grid_out) return CFMM_ERR_INVALID;
  if (!ctx->d_trace.n) return fail(ctx, CFMM_ERR_STATE, "option \"trace\" is off");
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  *grid_out = ctx->trace_grid;
  if (out && cap_ctas >= ctx->trace_grid && ctx->trace_grid > 0) {
    CU_TRY(ctx, cudaDeviceSynchronize());
    CU_TRY(ctx, cudaMemcpy(out, ctx->d_trace.p, (size_t)ctx->trace_grid * 8 * sizeof(uint64_t),
                           cudaMemcpyDeviceToHost));
  }
  return CFMM_OK;
}

// Test hook: number of (a/b, sqrt a, sqrt b) results, over n host-provided
// operand pairs, where the guard-free in-range recurrences differ from the IEEE
// intrinsics.  Must be 0 for operands in [2^-100, 2^100].
int cfmm_selftest_inrange_math(cfmm_ctx* ctx, const double* a, const double* b, int64_t n,
                               int64_t* mismatches) {
  if (!ctx || !a || !b || !mismatches || n < 0) return CFMM_ERR_INVALID;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  DevBuf<double> da, db;
  DevBuf<unsigned long long> dm;
  const unsigned long long zero = 0;
  CU_TRY(ctx, da.upload(a, (size_t)n));
  CU_TRY(ctx, db.upload(b, (size_t)n));
  CU_TRY(ctx, dm.upload(&zero, 1));
  if (n > 0) {
    cfmm::inrange_math_selftest_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(
        da.p, db.p, n, dm.p);
    ctx->launches++;
  }
  unsigned long long out = 0;
  cudaError_t e = cudaMemcpyAsync(&out, dm.p, sizeof(out), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  da.release();
  db.release();
  dm.release();
  if (e != cudaSuccess) return fail(ctx, CFMM_ERR_CUDA, "selftest failed: %s", cudaGetErrorString(e));
  *mismatches = (int64_t)out;
  return CFMM_OK;
}

// ---- multi-GPU -----------------------------------------------------------------

int cfmm_comm_export(cfmm_ctx* ctx, void* handle_out) {
  if (!ctx || !handle_out) return CFMM_ERR_INVALID;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  static_assert(sizeof(cfmm::PeerHandle) <= CFMM_COMM_HANDLE_BYTES, "handle size");
  memset(handle_out, 0, CFMM_COMM_HANDLE_BYTES);
  if (!ctx->comm.export_handle(ctx->n_tokens + 1, (cfmm::PeerHandle*)handle_out))
    return fail(ctx, CFMM_ERR_COMM, "comm export failed: %s", ctx->comm.error().c_str());
  return CFMM_OK;
}

int cfmm_comm_attach(cfmm_ctx* ctx, int world, int rank, const void* handles) {
  if (!ctx || !handles) return CFMM_ERR_INVALID;
  if (world < 1 || world > cfmm::kMaxPeers || rank < 0 || rank >= world)
    return fail(ctx, CFMM_ERR_INVALID, "bad world/rank %d/%d", rank, world);
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  ctx->state_version++;
  if (!ctx->comm.attach(world, rank, (const unsigned char*)handles,
                        CFMM_COMM_HANDLE_BYTES, ctx->sm_count))
    return fail(ctx, CFMM_ERR_COMM, "comm attach failed: %s", ctx->comm.error().c_str());
  ctx->comm.force_mode(ctx->exchange_protocol);  // an option set before the attach holds
  return CFMM_OK;
}

// For callers of the asynchronous entry points (cfmm_sweep_device*): did any exchange enqueued so
// far give up on a peer?  Synchronises the context's last stream first.
int cfmm_comm_check(cfmm_ctx* ctx) {
  if (!ctx) return CFMM_ERR_INVALID;
  if (!ctx->comm.attached()) return CFMM_OK;
  CU_TRY(ctx, cudaSetDevice(ctx->device));
  CU_TRY(ctx, cudaStreamSynchronize(ctx->last_stream ? ctx->last_stream : ctx->stream));
  if (ctx->comm.timed_out())
    return fail(ctx, CFMM_ERR_COMM, "peer exchange timed out: a rank of the group did not deliver its packets");
  return CFMM_OK;
}

int cfmm_comm_detach(cfmm_ctx* ctx) {
  if (!ctx) return CFMM_ERR_INVALID;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  ctx->comm.detach();
  return CFMM_OK;
}

}  // extern "C"
