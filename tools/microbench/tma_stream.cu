// Microbenchmark: the stream ceiling of the headline sweep's structure, per record size and CTA
// shape.  A persistent grid of SMs x CTAs/SM, a contiguous record range per CTA, a per-warp
// 2-stage cp.async.bulk ring with mbarriers, records handed out by a shared counter (the first
// two per warp static) -- exactly product_sweep_tma's chunk loop -- but the consumer does one
// dependent read of the stage per lane and record, so the loop costs next to nothing besides the
// copies, the waits, the counter and the re-arm.  201.7 MB per pass (the headline set's 20-byte
// stream); GB/s from CUDA events (median of the timed launches), with the GPU name, its power
// limit and the median SM clock sampled while the timed launches ran.  Then the headline set's
// record count (52,099 192-pool records) at 3872 B (201.7 MB, 20 B per pool) and at 3520 B
// (183.4 MB, 18 B per pool), 2 x 10 warps, interleaved over several rounds.
// Last, the L2 kept across passes (the H100's L2 holds 50 MB, a 3520-byte headline pass 183.4 MB): the
// same 3520-byte passes with an .L2::cache_hint policy on every bulk copy.  A fixed subset of the
// records is "kept" -- record r when r % k == 0, so every CTA keeps the same share of its range -- and
// the rest "streamed" as evict_first; the kept ones go as evict_normal or as evict_last.  Against that,
// one createpolicy.fractional policy (evict_last on a fraction 1/k of the lines, evict_first on the
// rest) on every copy.  Between configurations every line of the buffer goes back to evict_normal
// (applypriority), so no configuration inherits lines another one kept.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_stream tma_stream.cu -lnvidia-ml
//        (-L/usr/local/cuda/lib64/stubs where the driver's libnvidia-ml is not on the link path)
#include <cuda_runtime.h>
#include <nvml.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <thread>
#include <vector>

constexpr size_t kStreamBytes = 201700000;  // 104,167 records x 1936 B
constexpr int kHeadlineRecords = 52099;     // 192-pool records of the headline set
constexpr size_t kBufBytes = (size_t)kHeadlineRecords * 3872 > kStreamBytes ? (size_t)kHeadlineRecords * 3872 : kStreamBytes;
constexpr int kStages = 2;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\nbra WAIT_%=;\nDONE_%=:\n}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}

// L2 policy of the bulk copies (kernel parameter `hint`)
enum Hint {
  kNoHint = 0,      // plain cp.async.bulk
  kFirstNormal = 1, // record r % k == 0 evict_normal, the others evict_first
  kFirstLast = 2,   // record r % k == 0 evict_last, the others evict_first
  kFractional = 3,  // every copy: createpolicy.fractional evict_last on 1/k of the lines, evict_first on the rest
  kAllFirst = 4,    // every copy evict_first
};

template <int REC, int WARPS, int CTAS>
__global__ void __launch_bounds__(WARPS * 32, CTAS) stream(const unsigned char* __restrict__ src, int n_rec,
                                                             unsigned* __restrict__ out, int hint = kNoHint, int k = 0) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t full[WARPS][kStages];
  __shared__ int s_next;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, G = gridDim.x;
  const int c0 = (int)((long long)n_rec * blockIdx.x / G), c1 = (int)((long long)n_rec * (blockIdx.x + 1) / G);
  unsigned char* my = smem + (size_t)warp * kStages * REC;
  // the two policies, created once per thread: pol_keep for the kept records, pol_stream for the others
  uint64_t pol_keep = 0, pol_stream = 0;
  if (hint == kFractional) {
    const float frac = 1.0f / (float)k;
    asm volatile("createpolicy.fractional.L2::evict_last.L2::evict_first.b64 %0, %1;" : "=l"(pol_keep) : "f"(frac));
    pol_stream = pol_keep;
  } else if (hint != kNoHint) {
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_stream));
    if (hint == kFirstLast) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_keep));
    else if (hint == kFirstNormal) asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol_keep));
    else pol_keep = pol_stream;
  }
  auto issue = [&](int r, int st) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&full[warp][st])), "r"(REC) : "memory");
    if (hint == kNoHint) {
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       smem_u32(my + st * REC)), "l"(src + (size_t)r * REC), "r"(REC), "r"(smem_u32(&full[warp][st]))
                   : "memory");
    } else {
      const uint64_t pol = k > 0 && r % k == 0 ? pol_keep : pol_stream;
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                       smem_u32(my + st * REC)), "l"(src + (size_t)r * REC), "r"(REC), "r"(smem_u32(&full[warp][st])), "l"(pol)
                   : "memory");
    }
  };
  if (lane == 0) {
    for (int s = 0; s < kStages; ++s)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&full[warp][s])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  int cid0 = c0 + warp, cid1 = cid0 + WARPS;
  if (cid0 >= c1) cid0 = -1;
  if (cid1 >= c1) cid1 = -1;
  if (threadIdx.x == 0) s_next = c0 + 2 * WARPS;
  __syncthreads();
  if (lane == 0 && cid0 >= 0) issue(cid0, 0);
  if (lane == 0 && cid1 >= 0) issue(cid1, 1);
  unsigned acc = 0, par = 0;
  int st = 0;
  while (true) {
    const int c = st ? cid1 : cid0;
    if (c < 0) break;
    mbar_wait(&full[warp][st], (par >> st) & 1u);
    par ^= 1u << st;
    acc += reinterpret_cast<const unsigned*>(my + st * REC)[(acc & 1u) + lane * 4];  // one dependent read
    __syncwarp();
    int k = -1;
    if (lane == 0) {
      k = atomicAdd(&s_next, 1);
      if (k < c1) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(k, st);
      } else {
        k = -1;
      }
    }
    k = __shfl_sync(0xffffffffu, k, 0);
    if (st) cid1 = k; else cid0 = k;
    st ^= 1;
  }
  if (acc == 0x12345678u) out[0] = acc;
}

// every 128-byte line of [p, p + bytes) back to evict_normal in the L2
__global__ void reset_priority(const unsigned char* p, size_t bytes) {
  for (size_t off = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 128; off < bytes; off += (size_t)gridDim.x * blockDim.x * 128)
    asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(p + off) : "memory");
}

static nvmlDevice_t g_nvml;
static bool g_have_nvml = false;

// returns the median launch time in µs (0 when the shape does not fit); n_rec <= 0: kStreamBytes / REC
template <int REC, int WARPS, int CTAS>
double run(const unsigned char* d_src, unsigned* d_out, int sms, std::vector<unsigned>& clocks, int n_rec = 0,
           int hint = kNoHint, int keep_k = 0) {
  constexpr int smem = WARPS * kStages * REC;
  auto k = stream<REC, WARPS, CTAS>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k, WARPS * 32, smem);
  if (n_rec <= 0) n_rec = (int)(kStreamBytes / REC);
  const int grid = sms * CTAS;
  if (occ < CTAS) {
    printf("%5d B  %d x %2d warps: does not fit (%d CTAs/SM)\n", REC, CTAS, WARPS, occ);
    return 0.0;
  }
  constexpr int kLaunches = 200;
  std::vector<cudaEvent_t> ev(kLaunches + 1);
  for (auto& e : ev) cudaEventCreate(&e);
  for (int i = 0; i < 20; ++i) k<<<grid, WARPS * 32, smem>>>(d_src, n_rec, d_out, hint, keep_k);
  cudaDeviceSynchronize();
  cudaEventRecord(ev[0]);
  for (int i = 0; i < kLaunches; ++i) {
    k<<<grid, WARPS * 32, smem>>>(d_src, n_rec, d_out, hint, keep_k);
    cudaEventRecord(ev[i + 1]);
  }
  // sample the SM clock while the timed launches run
  while (g_have_nvml && cudaEventQuery(ev[kLaunches]) == cudaErrorNotReady) {
    unsigned mhz = 0;
    if (nvmlDeviceGetClockInfo(g_nvml, NVML_CLOCK_SM, &mhz) == NVML_SUCCESS) clocks.push_back(mhz);
    std::this_thread::sleep_for(std::chrono::milliseconds(1));
  }
  cudaEventSynchronize(ev[kLaunches]);
  std::vector<float> t(kLaunches);
  for (int i = 0; i < kLaunches; ++i) cudaEventElapsedTime(&t[i], ev[i], ev[i + 1]);
  std::sort(t.begin(), t.end());
  const double med_us = t[kLaunches / 2] * 1e3, min_us = t[0] * 1e3;
  const double bytes = (double)n_rec * REC;
  if (hint == kNoHint)
    printf("%5d B  %d x %2d warps  %7d records  %2d KB ring/SM  median %7.2f us  min %7.2f us  %7.1f GB/s (median)\n", REC,
           CTAS, WARPS, n_rec, CTAS * smem / 1024, med_us, min_us, bytes / (med_us * 1e3));
  for (auto& e : ev) cudaEventDestroy(e);
  return med_us;
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  unsigned power_mw = 0;
  if (nvmlInit() == NVML_SUCCESS && nvmlDeviceGetHandleByIndex(0, &g_nvml) == NVML_SUCCESS) {
    g_have_nvml = true;
    nvmlDeviceGetPowerManagementLimit(g_nvml, &power_mw);
  }
  printf("GPU %s, %d SMs, power limit %.0f W\n", prop.name, sms, power_mw / 1000.0);
  unsigned char* d_src;
  unsigned* d_out;
  cudaMalloc(&d_src, kBufBytes + 4096);
  cudaMalloc(&d_out, 4);
  cudaMemset(d_src, 1, kBufBytes + 4096);
  std::vector<unsigned> clocks;
  run<1936, 14, 2>(d_src, d_out, sms, clocks);
  run<1936, 10, 2>(d_src, d_out, sms, clocks);
  run<1936, 24, 1>(d_src, d_out, sms, clocks);
  run<3856, 14, 2>(d_src, d_out, sms, clocks);
  run<3856, 10, 2>(d_src, d_out, sms, clocks);
  run<3856, 24, 1>(d_src, d_out, sms, clocks);
  run<3872, 14, 2>(d_src, d_out, sms, clocks);
  run<3872, 10, 2>(d_src, d_out, sms, clocks);
  run<3872, 24, 1>(d_src, d_out, sms, clocks);
  run<1936, 14, 2>(d_src, d_out, sms, clocks);  // the first shape again: drift check
  // the headline record count at both 192-pool record sizes, alternated
  constexpr int kRounds = 7;
  double t20[kRounds], t18[kRounds];
  for (int r = 0; r < kRounds; ++r) {
    t20[r] = run<3872, 10, 2>(d_src, d_out, sms, clocks, kHeadlineRecords);
    t18[r] = run<3520, 10, 2>(d_src, d_out, sms, clocks, kHeadlineRecords);
  }
  std::sort(t20, t20 + kRounds);
  std::sort(t18, t18 + kRounds);
  printf("headline records, %d rounds of medians: 3872 B %.2f..%.2f us (median %.2f), 3520 B %.2f..%.2f us (median %.2f), "
         "%.1f %% less time\n",
         kRounds, t20[0], t20[kRounds - 1], t20[kRounds / 2], t18[0], t18[kRounds - 1], t18[kRounds / 2],
         100.0 * (1.0 - t18[kRounds / 2] / t20[kRounds / 2]));
  // the L2 kept across passes: per (policy, k) the medians of the rounds, all configurations interleaved
  {
    struct Cfg {
      int hint, k;
      const char* name;
    };
    const Cfg cfgs[] = {{kNoHint, 0, "no hint"},          {kAllFirst, 0, "all evict_first"},
                        {kFirstNormal, 11, "normal/first"}, {kFirstNormal, 8, "normal/first"},
                        {kFirstNormal, 6, "normal/first"},  {kFirstNormal, 5, "normal/first"},
                        {kFirstLast, 11, "last/first"},     {kFirstLast, 8, "last/first"},
                        {kFirstLast, 6, "last/first"},      {kFirstLast, 5, "last/first"},
                        {kFractional, 11, "fractional"},    {kFractional, 8, "fractional"},
                        {kFractional, 6, "fractional"},     {kFractional, 5, "fractional"}};
    constexpr int kCfgs = sizeof(cfgs) / sizeof(cfgs[0]);
    const size_t pass_bytes = (size_t)kHeadlineRecords * 3520;
    std::vector<std::vector<double>> t(kCfgs);
    for (int r = 0; r < kRounds; ++r)
      for (int c = 0; c < kCfgs; ++c) {
        reset_priority<<<sms * 8, 256>>>(d_src, pass_bytes);
        t[c].push_back(run<3520, 10, 2>(d_src, d_out, sms, clocks, kHeadlineRecords, cfgs[c].hint, cfgs[c].k));
      }
    reset_priority<<<sms * 8, 256>>>(d_src, pass_bytes);
    cudaDeviceSynchronize();
    printf("L2 kept across 3520-byte headline passes (%.1f MB per pass), %d rounds of medians of 200 back-to-back passes:\n",
           pass_bytes / 1e6, kRounds);
    for (int c = 0; c < kCfgs; ++c) {
      std::sort(t[c].begin(), t[c].end());
      const int kept = cfgs[c].k > 0 ? (kHeadlineRecords + cfgs[c].k - 1) / cfgs[c].k : 0;
      printf("  %-16s k = %2d  kept %5.1f MB  %7.2f..%7.2f us  median %7.2f us  %+6.1f %% against no hint\n", cfgs[c].name,
             cfgs[c].k, kept * 3520 / 1e6, t[c].front(), t[c].back(), t[c][kRounds / 2],
             100.0 * (t[c][kRounds / 2] / t[0][kRounds / 2] - 1.0));
    }
  }
  if (!clocks.empty()) {
    std::sort(clocks.begin(), clocks.end());
    printf("SM clock during the timed launches: median %u MHz (min %u, max %u, %zu samples)\n", clocks[clocks.size() / 2],
           clocks.front(), clocks.back(), clocks.size());
  } else {
    printf("SM clock: not read (NVML unavailable)\n");
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    printf("CUDA error: %s\n", cudaGetErrorString(e));
    return 1;
  }
  return 0;
}
