// peer_exchange.cuh -- sum-allreduce of [Ψ ; acc] (n_tokens+1 fp64) across the
// GPUs of one box, over NVLink peer memory (no NCCL on this path).
//
// The message is 8 KB .. 400 KB: purely latency-bound.  Protocol ("LL push",
// the idea NCCL's low-latency protocol uses): every rank WRITES its partial
// vector straight into a receive area in each peer's memory as
// self-validating packets -- each fp64 travels as two 8-byte words
// {hi32 | epoch32}, {lo32 | epoch32} (8-byte stores are single-copy atomic, so a
// word is either old or complete).  The receiver polls its own local memory
// until both words of a packet carry the current epoch, then adds the value.
// There is no flag and no fence on the exchange's critical path: one NVLink traversal
// per hop, and the reduction runs as packets land.  (The FUSED form, run in the tail of the
// sweep kernel, is preceded by one grid-wide barrier: the local partial sums must be
// complete before they are pushed.)  Every wait is bounded: a poll that sees no packet for
// kPollTimeoutNs raises the context's error word and gives up, so a dead peer turns into
// CFMM_ERR_COMM on the host instead of a hung GPU.  Ranks are summed
// in rank order, so every rank ends with the bitwise-identical vector (the
// replicated L-BFGS-B drivers stay in lock-step).
//
// The first version of this file (flag + pull over peer loads, system fences)
// was slower than ncclAllReduce; the push protocols below replaced it.
//
// Receive areas are double-buffered by epoch parity.  A rank pushes epoch e+2
// only after finishing exchange e+1, i.e. after receiving every peer's e+1
// packets, which a peer sends only after its own exchange e completed in stream
// order -- so nobody can still be reading the area that is being overwritten.
//
// Mapping: one process per GPU -> cudaIpc handles exchanged by the host side;
// several contexts in one process -> raw pointers + cudaDeviceEnablePeerAccess.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <unistd.h>

#include <cstring>
#include <string>

namespace cfmm {

constexpr int kMaxPeers = 16;
constexpr int kExchangeThreads = 256;
constexpr unsigned long long kPollTimeoutNs = 4000000000ull;  // 4 s: far beyond any healthy exchange

__device__ __forceinline__ unsigned long long exch_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

struct PeerHandle {
  cudaIpcMemHandle_t ipc;  // 64 B
  uint64_t raw_ptr;        // same-process shortcut
  int64_t len;             // doubles per vector
  int32_t pid;
  int32_t device;
  int32_t world_cap;       // receive areas allocated for this many ranks
  int32_t pad;
};

// Receive buffer of a rank: area(src, parity) = base + ((src*2 + parity) * len) ulonglong2
struct ExchangeView {
  ulonglong2* recv_local;             // this rank's receive buffer
  ulonglong2* recv_peer[kMaxPeers];   // peer-mapped receive buffers (own entry unused)
  int world, rank;
  int64_t slice;                      // two-shot: tokens owned per rank = ceil(len / world)
  int64_t gather_off;                 // two-shot: packet offset of the gathered-result area
  int64_t direct_off;                 // direct protocol: offset (in packets) of its 8-byte areas
  unsigned* error;                    // device word raised when a poll times out (host: CFMM_ERR_COMM)
};

__device__ __forceinline__ void st_packet(ulonglong2* p, unsigned long long a, unsigned long long b) {
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}
__device__ __forceinline__ ulonglong2 ld_packet(const ulonglong2* p) {
  ulonglong2 v;
  asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
  return v;
}

// poll one packet until both words carry `tag`; false (and the error word raised) on timeout
__device__ __forceinline__ bool packet_ready(const ulonglong2& v, unsigned long long tag) {
  return (v.x & 0xffffffffull) == tag && (v.y & 0xffffffffull) == tag;
}
__device__ __forceinline__ bool poll_packet(const ExchangeView& x, const ulonglong2* q, unsigned long long tag,
                                            ulonglong2* out) {
  ulonglong2 v = ld_packet(q);
  if (!packet_ready(v, tag)) {
    const unsigned long long t0 = exch_now_ns();
    unsigned spins = 0;
    do {
      v = ld_packet(q);
      if ((++spins & 1023u) == 0u) {
        if (*reinterpret_cast<volatile unsigned*>(x.error)) return false;  // somebody already gave up
        if (exch_now_ns() - t0 > kPollTimeoutNs) {
          atomicExch(x.error, 1u);
          return false;
        }
      }
    } while (!packet_ready(v, tag));
  }
  *out = v;
  return true;
}
__device__ __forceinline__ double packet_value(const ulonglong2& v) {
  return __longlong_as_double((long long)((v.x & 0xffffffff00000000ull) | (v.y >> 32)));
}

// The packets of every other rank for one element (area(p) + off), summed with `mine` in rank
// order.  First pass: every packet is loaded once, back to back (independent loads: one L2 round
// trip when all of them have landed, instead of world-1 dependent ones).  Only when one was late:
// second pass, polling them in turn.
__device__ __forceinline__ bool gather_sum(const ExchangeView& x, int64_t area_len, int64_t off, int par,
                                           unsigned long long tag, double mine, double* out) {
  double s = 0.0;
  bool all = true;
#pragma unroll
  for (int p = 0; p < kMaxPeers; ++p) {
    if (p >= x.world) continue;
    if (p == x.rank) {
      s += mine;
      continue;
    }
    const ulonglong2 v = ld_packet(x.recv_local + ((int64_t)(p * 2 + par) * area_len + off));
    all = all && packet_ready(v, tag);
    s += packet_value(v);
  }
  if (!all) {
    s = 0.0;
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) {
      if (p >= x.world) continue;
      if (p == x.rank) {
        s += mine;
        continue;
      }
      ulonglong2 v;
      if (!poll_packet(x, x.recv_local + ((int64_t)(p * 2 + par) * area_len + off), tag, &v)) return false;
      s += packet_value(v);
    }
  }
  *out = s;
  return true;
}

// one-shot body for elements first, first+stride, ... (callable from any kernel)
__device__ __forceinline__ void peer_allreduce_oneshot_body(const ExchangeView& x, const double* src,
                                                            double* dst, int64_t len, unsigned int epoch,
                                                            int64_t first, int64_t stride) {
  const int par = (int)(epoch & 1u);
  const unsigned long long tag = (unsigned long long)epoch;
  for (int64_t j = first; j < len; j += stride) {
    const double mine = __ldcg(src + j);
    const unsigned long long bits = (unsigned long long)__double_as_longlong(mine);
    const unsigned long long w0 = ((bits >> 32) << 32) | tag;         // {hi32 | epoch}
    const unsigned long long w1 = ((bits & 0xffffffffull) << 32) | tag;  // {lo32 | epoch}
    // push to every peer's area for source = me
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < x.world && p != x.rank)
        st_packet(x.recv_peer[p] + ((int64_t)(x.rank * 2 + par) * len + j), w0, w1);
    // gather: my own areas, summed in rank order
    double s;
    if (!gather_sum(x, len, j, par, tag, mine, &s)) return;
    dst[j] = s;
  }
}

__global__ void __launch_bounds__(kExchangeThreads)
    peer_allreduce_kernel(ExchangeView x, const double* src, double* dst, int64_t len,
                          unsigned int epoch) {
  peer_allreduce_oneshot_body(x, src, dst, len, epoch,
                              (int64_t)blockIdx.x * blockDim.x + threadIdx.x,
                              (int64_t)gridDim.x * blockDim.x);
}

// Two-shot variant for world > 2 (reduce-scatter + all-gather, both as LL
// pushes): element j is owned by rank j / slice.  A non-owner pushes its partial
// to the owner's contribution area and then polls its own gathered-result area;
// the owner polls the world-1 contributions, sums in rank order, writes the
// result and pushes it to every peer's gathered-result area.  Per rank
// 2·(W−1)/W·len packets cross NVLink instead of (W−1)·len, at the price of a
// second hop.  Every rank receives the owner's bits, so results are identical
// everywhere by construction.  No thread waits on another thread of its own
// rank, so the grid need not be co-resident.
__device__ __forceinline__ void peer_allreduce_twoshot_body(const ExchangeView& x, const double* src,
                                                            double* dst, int64_t len, unsigned int epoch,
                                                            int64_t first, int64_t stride) {
  const int par = (int)(epoch & 1u);
  const unsigned long long tag = (unsigned long long)epoch;
  for (int64_t j = first; j < len; j += stride) {
    const int owner = (int)(j / x.slice);
    const int64_t i = j - (int64_t)owner * x.slice;
    const double mine = __ldcg(src + j);
    if (owner != x.rank) {
      const unsigned long long bits = (unsigned long long)__double_as_longlong(mine);
      st_packet(x.recv_peer[owner] + ((int64_t)(x.rank * 2 + par) * x.slice + i),
                ((bits >> 32) << 32) | tag, ((bits & 0xffffffffull) << 32) | tag);
      const ulonglong2* q = x.recv_local + x.gather_off + (int64_t)par * len + j;
      ulonglong2 v;
      if (!poll_packet(x, q, tag, &v)) return;
      dst[j] = packet_value(v);
    } else {
      double s;
      if (!gather_sum(x, x.slice, i, par, tag, mine, &s)) return;
      dst[j] = s;
      const unsigned long long bits = (unsigned long long)__double_as_longlong(s);
      const unsigned long long w0 = ((bits >> 32) << 32) | tag, w1 = ((bits & 0xffffffffull) << 32) | tag;
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p)
        if (p < x.world && p != x.rank)
          st_packet(x.recv_peer[p] + x.gather_off + (int64_t)par * len + j, w0, w1);
    }
  }
}

__global__ void __launch_bounds__(kExchangeThreads)
    peer_allreduce_twoshot_kernel(ExchangeView x, const double* src, double* dst, int64_t len,
                                  unsigned int epoch) {
  peer_allreduce_twoshot_body(x, src, dst, len, epoch,
                              (int64_t)blockIdx.x * blockDim.x + threadIdx.x,
                              (int64_t)gridDim.x * blockDim.x);
}

// Direct protocol (default): ONE hop for any world size and 8 bytes per value.  A receive slot
// holds either the "empty" pattern (all ones: a NaN no arithmetic produces -- hardware NaNs are
// 0x7ff8000000000000 -- and a partial that carries exactly it is sent as the canonical NaN) or a
// value: the 8-byte store is atomic, so the value validates itself and needs no tag.  Every rank
// pushes its partial to all peers (area(src = me, parity)), polls its own world-1 slots with all
// loads of a pass issued back to back, sums the world values in rank order -- the same values in
// the same order everywhere: bitwise-identical results -- and resets the slots it consumed.  A
// slot is written again two exchanges later, which the writer cannot start before this rank
// has finished the next exchange (it needs this rank's contribution), i.e. after this kernel:
// the reset is never overtaken.  Per rank (W-1)·len·8 bytes leave over NVLink (2.8 MB at W = 8,
// n = 50k) against two dependent hops of the two-shot LL form.
constexpr unsigned long long kDirectEmpty = ~0ull;
__device__ __forceinline__ void st_u64_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_u64_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void peer_allreduce_direct_body(const ExchangeView& x, const double* src, double* dst,
                                                           int64_t len, unsigned int epoch, int64_t first,
                                                           int64_t stride) {
  const int par = (int)(epoch & 1u);
  unsigned long long* local = reinterpret_cast<unsigned long long*>(x.recv_local + x.direct_off);
  for (int64_t j = first; j < len; j += stride) {
    unsigned long long bits = (unsigned long long)__double_as_longlong(__ldcg(src + j));
    if (bits == kDirectEmpty) bits = 0x7ff8000000000000ull;
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < x.world && p != x.rank)
        st_u64_sys(reinterpret_cast<unsigned long long*>(x.recv_peer[p] + x.direct_off) +
                       ((int64_t)(x.rank * 2 + par) * len + j),
                   bits);
    double s;
    unsigned spins = 0;
    unsigned long long t0 = 0;
    for (;;) {
      bool all = true;
      s = 0.0;
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p) {
        if (p >= x.world) continue;
        unsigned long long v = bits;
        if (p != x.rank) {
          v = ld_u64_sys(local + ((int64_t)(p * 2 + par) * len + j));
          all = all && v != kDirectEmpty;
        }
        s += __longlong_as_double((long long)v);
      }
      if (all) break;
      if (spins == 0) t0 = exch_now_ns();
      if ((++spins & 1023u) == 0u) {
        if (*reinterpret_cast<volatile unsigned*>(x.error)) return;  // somebody already gave up
        if (exch_now_ns() - t0 > kPollTimeoutNs) {
          atomicExch(x.error, 1u);
          return;
        }
      }
    }
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p)
      if (p < x.world && p != x.rank) st_u64_sys(local + ((int64_t)(p * 2 + par) * len + j), kDirectEmpty);
    dst[j] = s;
  }
}

__global__ void __launch_bounds__(kExchangeThreads)
    peer_allreduce_direct_kernel(ExchangeView x, const double* src, double* dst, int64_t len,
                                 unsigned int epoch) {
  peer_allreduce_direct_body(x, src, dst, len, epoch, (int64_t)blockIdx.x * blockDim.x + threadIdx.x,
                             (int64_t)gridDim.x * blockDim.x);
}

// What a sweep kernel needs to run the exchange in its own tail.
struct FusedExchange {
  ExchangeView view;
  double* dst;                     // where the reduced [Ψ; acc] goes (may equal the accumulator)
  unsigned long long* grid_done;   // device counter: CTAs that finished accumulating, all sweeps
  unsigned long long target;       // value grid_done reaches when every CTA of THIS sweep is done
  unsigned int epoch;
  int mode;                        // 0 = off, 1 = LL one-shot, 2 = LL two-shot, 3 = direct
};

// The exchange in a sweep kernel's tail.
__device__ __forceinline__ void fused_exchange_tail(const FusedExchange& fx, const double* src, int64_t len,
                                                    int64_t first, int64_t stride) {
  if (fx.mode == 3)
    peer_allreduce_direct_body(fx.view, src, fx.dst, len, fx.epoch, first, stride);
  else if (fx.mode == 2)
    peer_allreduce_twoshot_body(fx.view, src, fx.dst, len, fx.epoch, first, stride);
  else
    peer_allreduce_oneshot_body(fx.view, src, fx.dst, len, fx.epoch, first, stride);
}

class PeerExchange {
 public:
  bool attached() const { return attached_ && world_ > 1; }
  const std::string& error() const { return err_; }
  int launches_per_reduce() const { return 1; }
  // protocol: 1 = LL one-shot, 2 = LL two-shot, 3 = direct; anything else = by world size: the
  // direct push up to 4 ranks, LL two-shot beyond: the one-hop push sends (W-1)x the bytes of the
  // two-shot form, and beyond 4 ranks those bytes cost more than the second hop on an NVSwitch
  // system.  The crossover has not been re-measured on H100; exchange_protocol overrides it.
  void force_mode(int mode) { mode_ = mode >= 1 && mode <= 3 ? mode : (world_ <= 4 ? 3 : 2); }
  int mode() const { return mode_; }
  // fused use: the sweep kernel itself runs the exchange body; returns the epoch to tag with
  unsigned int begin_fused(int* mode) {
    ++epoch_;
    if (epoch_ == 0) epoch_ = 2;
    *mode = mode_;
    return epoch_;
  }
  const ExchangeView& view() const { return view_; }
  // true when some poll of an earlier exchange timed out (checked by the host after a sync)
  bool timed_out() const {
    unsigned h = 0;
    if (!err_word_) return false;
    return cudaMemcpy(&h, err_word_, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess && h != 0;
  }

  bool export_handle(int64_t len, PeerHandle* out) {
    if (!base_) {
      len_ = len;
      // LL: kMaxPeers contribution areas x 2 parities, plus 2 gathered-result areas (two-shot);
      // direct: kMaxPeers x 2 areas of 8-byte slots behind them, all "empty"
      const size_t ll_bytes = (size_t)(kMaxPeers + 1) * 2 * (size_t)len * sizeof(ulonglong2);
      const size_t direct_bytes = (size_t)kMaxPeers * 2 * (size_t)len * sizeof(unsigned long long);
      bytes_ = ll_bytes + direct_bytes;
      if (!ok(cudaMalloc(&base_, bytes_), "cudaMalloc(exchange)")) return false;
      if (!ok(cudaMemset(base_, 0, ll_bytes), "cudaMemset(exchange)")) return false;
      if (!ok(cudaMemset((char*)base_ + ll_bytes, 0xff, direct_bytes), "cudaMemset(exchange)")) return false;
      if (!ok(cudaMalloc(&err_word_, sizeof(unsigned)), "cudaMalloc(exchange error word)")) return false;
      if (!ok(cudaMemset(err_word_, 0, sizeof(unsigned)), "cudaMemset(exchange error word)")) return false;
      // the receive areas must hold their initial pattern before any peer or local kernel looks at
      // them: memsets run on the legacy stream, which non-blocking streams do not wait for
      if (!ok(cudaStreamSynchronize(cudaStreamLegacy), "cudaStreamSynchronize(exchange init)")) return false;
    }
    memset(out, 0, sizeof(*out));
    if (!ok(cudaIpcGetMemHandle(&out->ipc, base_), "cudaIpcGetMemHandle")) return false;
    out->raw_ptr = (uint64_t)(uintptr_t)base_;
    out->len = len_;
    out->pid = (int32_t)getpid();
    int dev = 0;
    cudaGetDevice(&dev);
    out->device = dev;
    out->world_cap = kMaxPeers;
    return true;
  }

  bool attach(int world, int rank, const unsigned char* handles, size_t stride,
              int sm_count) {
    if (!base_) {
      err_ = "cfmm_comm_export must be called before cfmm_comm_attach";
      return false;
    }
    if (attached_) {  // epochs restart at 0 on attach; the receive areas must be fresh
      err_ = "already attached (cfmm_comm_detach, then export and attach again)";
      return false;
    }
    world_ = world;
    rank_ = rank;
    // every element is an independent push+poll: enough CTAs to cover the vector once
    int64_t want = (len_ + kExchangeThreads - 1) / kExchangeThreads;
    grid_ = (int)(want < 2 * sm_count ? want : 2 * sm_count);
    if (grid_ < 1) grid_ = 1;
    int my_dev = 0;
    cudaGetDevice(&my_dev);
    memset(&view_, 0, sizeof(view_));
    view_.world = world;
    view_.rank = rank;
    view_.recv_local = (ulonglong2*)base_;
    view_.slice = (len_ + world - 1) / world;
    view_.gather_off = (int64_t)kMaxPeers * 2 * len_;
    view_.direct_off = (int64_t)(kMaxPeers + 1) * 2 * len_;
    view_.error = err_word_;
    force_mode(0);
    for (int p = 0; p < world; ++p) {
      PeerHandle h;
      memcpy(&h, handles + (size_t)p * stride, sizeof(h));
      if (h.len != len_) {
        err_ = "rank " + std::to_string(p) + " exported a different vector length";
        return false;
      }
      void* pbase = nullptr;
      if (p == rank) {
        pbase = base_;
      } else if (h.pid == (int32_t)getpid()) {
        int can = 0;
        cudaDeviceCanAccessPeer(&can, my_dev, h.device);
        if (!can) {
          err_ = "no peer access between device " + std::to_string(my_dev) +
                 " and " + std::to_string(h.device);
          return false;
        }
        cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
          return ok(e, "cudaDeviceEnablePeerAccess");
        cudaGetLastError();
        pbase = (void*)(uintptr_t)h.raw_ptr;
      } else {
        if (!ok(cudaIpcOpenMemHandle(&pbase, h.ipc, cudaIpcMemLazyEnablePeerAccess),
                "cudaIpcOpenMemHandle"))
          return false;
        opened_[p] = pbase;
      }
      view_.recv_peer[p] = (ulonglong2*)pbase;
    }
    epoch_ = 0;
    attached_ = true;
    return true;
  }

  bool all_reduce(const double* src, double* dst, int64_t len, cudaStream_t st) {
    if (len != len_) {
      err_ = "all_reduce length mismatch";
      return false;
    }
    ++epoch_;
    if (epoch_ == 0) epoch_ = 2;  // 0 is the value of untouched memory; keep parity moving
    if (mode_ == 3)
      peer_allreduce_direct_kernel<<<grid_, kExchangeThreads, 0, st>>>(view_, src, dst, len, epoch_);
    else if (mode_ == 2)
      peer_allreduce_twoshot_kernel<<<grid_, kExchangeThreads, 0, st>>>(view_, src, dst, len, epoch_);
    else
      peer_allreduce_kernel<<<grid_, kExchangeThreads, 0, st>>>(view_, src, dst, len, epoch_);
    return ok(cudaGetLastError(), "peer_allreduce_kernel launch");
  }

  void detach() {
    for (int p = 0; p < kMaxPeers; ++p)
      if (opened_[p]) {
        cudaIpcCloseMemHandle(opened_[p]);
        opened_[p] = nullptr;
      }
    if (base_) cudaFree(base_);
    if (err_word_) cudaFree(err_word_);
    err_word_ = nullptr;
    base_ = nullptr;
    attached_ = false;
    world_ = 1;
  }

 private:
  bool ok(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    err_ = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
  }
  void* base_ = nullptr;
  unsigned* err_word_ = nullptr;
  void* opened_[kMaxPeers] = {};
  size_t bytes_ = 0;
  int64_t len_ = 0;
  int world_ = 1, rank_ = 0, grid_ = 64;
  unsigned int epoch_ = 0;
  bool attached_ = false;
  int mode_ = 3;
  ExchangeView view_;
  std::string err_;
};

}  // namespace cfmm
