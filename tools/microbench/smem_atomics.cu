// Microbenchmark: cost of accumulating one value per "pool" into a 1600-slot shared slice
// with random slots, for the candidate primitives of the Ψ[b] accumulation.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o smem_atomics smem_atomics.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>

constexpr int NB = 1600;
constexpr int THREADS = 448;

__device__ __forceinline__ uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s; }

template <int MODE>
__global__ void __launch_bounds__(THREADS, 2) bench(int iters, double* out, double* gpsi, int n_tokens) {
  __shared__ double s_nu[NB];
  __shared__ unsigned long long s64[NB];
  __shared__ unsigned int s32[3 * NB];
  for (int i = threadIdx.x; i < NB; i += THREADS) { s_nu[i] = 1.0 + i; s64[i] = 0; s32[i] = 0; s32[NB + i] = 0; s32[2 * NB + i] = 0; }
  __syncthreads();
  uint32_t seed = blockIdx.x * THREADS + threadIdx.x + 12345u;
  const int lane = threadIdx.x & 31;
  double acc = 0.0;
  for (int it = 0; it < iters; ++it) {
    uint32_t r = lcg(seed) >> 8;
    int slot = (int)(r % NB);
    if (MODE == 5 || MODE == 7) slot = (slot & ~15) | (lane & 15);  // conflict-free by construction
    const double nu = s_nu[slot];
    const double val = nu * 1e-3 + (double)(r & 255);
    acc += nu;
    if (MODE == 0) {
      // nothing: LDS only
    } else if (MODE == 1 || MODE == 5) {
      atomicAdd(reinterpret_cast<double*>(&s64[slot]), val);  // LDS.64 + ATOMS.CAST.SPIN.64 loop
    } else if (MODE == 2) {
      // three 32-bit REDs (16/16/32 limbs of a 64-bit fixed-point value)
      const long long q = __double2ll_rn(val * 1048576.0);
      atomicAdd(&s32[slot], (unsigned)(q & 0xffff));
      atomicAdd(&s32[NB + slot], (unsigned)((q >> 16) & 0xffff));
      atomicAdd(&s32[2 * NB + slot], (unsigned)(q >> 32));
    } else if (MODE == 3 || MODE == 7) {
      // lo with return (carry), hi RED
      const long long q = __double2ll_rn(val * 1048576.0);
      const unsigned lo = (unsigned)q;
      const unsigned old = atomicAdd(&s32[2 * slot], lo);
      const unsigned carry = (old + lo) < old ? 1u : 0u;
      atomicAdd(&s32[2 * slot + 1], (unsigned)(q >> 32) + carry);
    } else if (MODE == 4) {
      const long long q = __double2ll_rn(val * 1048576.0);
      atomicAdd(&s32[slot], (unsigned)q);
      atomicAdd(&s32[NB + slot], (unsigned)(q >> 32));
    } else if (MODE == 6) {
      // global fp64 RED, spread over n_tokens
      const int t = (int)(r % (unsigned)n_tokens);
      asm volatile("red.global.add.f64 [%0], %1;" ::"l"(gpsi + t), "d"(val) : "memory");
    } else if (MODE == 8) {
      // float hi/lo pair of native fp32 shared REDs (precision reference only)
      const float hi = (float)val;
      const float lo = (float)(val - (double)hi);
      atomicAdd(reinterpret_cast<float*>(&s32[slot]), hi);
      atomicAdd(reinterpret_cast<float*>(&s32[NB + slot]), lo);
    } else if (MODE == 9) {
      // single native 32-bit RED
      atomicAdd(&s32[slot], (unsigned)(r & 255));
    }
  }
  __syncthreads();
  double t = acc;
  for (int i = threadIdx.x; i < NB; i += THREADS) t += (double)s64[i] + s32[i] + s32[NB + i] + s32[2 * NB + i];
  if (t == 123.456) out[0] = t;
}

static int g_grid = 0;  // two CTAs per SM, as the sweep kernel runs

template <int MODE>
float run(int iters, double* out, double* gpsi, int n_tokens) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  bench<MODE><<<g_grid, THREADS>>>(iters / 10, out, gpsi, n_tokens);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  bench<MODE><<<g_grid, THREADS>>>(iters, out, gpsi, n_tokens);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  return ms;
}

int main() {
  double *out, *gpsi; const int n_tokens = 50000;
  cudaMalloc(&out, 8); cudaMalloc(&gpsi, 8 * n_tokens); cudaMemset(gpsi, 0, 8 * n_tokens);
  int sms = 0, khz = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);  // maximum SM clock
  g_grid = 2 * sms;
  const int iters = 2000;
  const double ops = (double)g_grid * THREADS * iters;
  const char* names[] = {"0 LDS only", "1 fp64 atomicAdd (CAS loop) random", "2 3x RED.32 limbs", "3 ATOMS.ADD.32 ret + RED.32 carry",
                         "4 2x RED.32", "5 fp64 CAS conflict-free lanes", "6 global RED.F64 spread 50k", "7 carry scheme conflict-free",
                         "8 2x RED.F32", "9 1x RED.32"};
  float ms[10];
  ms[0] = run<0>(iters, out, gpsi, n_tokens); ms[1] = run<1>(iters, out, gpsi, n_tokens);
  ms[2] = run<2>(iters, out, gpsi, n_tokens); ms[3] = run<3>(iters, out, gpsi, n_tokens);
  ms[4] = run<4>(iters, out, gpsi, n_tokens); ms[5] = run<5>(iters, out, gpsi, n_tokens);
  ms[6] = run<6>(iters, out, gpsi, n_tokens); ms[7] = run<7>(iters, out, gpsi, n_tokens);
  ms[8] = run<8>(iters, out, gpsi, n_tokens); ms[9] = run<9>(iters, out, gpsi, n_tokens);
  for (int m = 0; m < 10; ++m) {
    // cycles per warp-op per SM at the maximum SM clock: (ms*1e-3*clock) / (ops/32/SMs)
    const double cyc = ms[m] * 1e-3 * (khz * 1e3) / (ops / 32.0 / sms);
    printf("%-40s %8.3f ms  %7.2f cyc/warp-op/SM  (%.1f us per 10M ops)\n", names[m], ms[m], cyc, ms[m] * 1e3 * 1e7 / ops);
  }
  return 0;
}
