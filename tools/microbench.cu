// tools/microbench.cu -- measured denominators for the integer-pipe roofline:
// sustained POPC / LOP3 / IADD3 issue rates per SM. One CTA of 1024 threads per
// SM; rates are lane-results per SM clock from in-kernel clock64() deltas, so
// they do not depend on the DVFS state. Also times a plain HBM copy.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench tools/microbench.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int ITERS = 4096;
constexpr int ILP = 8;

template <int MODE>
__global__ void __launch_bounds__(1024) pipe_kernel(unsigned* out, long long* cycles, unsigned seed) {
  unsigned x[ILP], acc[ILP];
#pragma unroll
  for (int i = 0; i < ILP; ++i) { x[i] = seed * (threadIdx.x + 1) + i * 0x9e3779b9u; acc[i] = i; }
  unsigned y = seed ^ threadIdx.x;
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; ++i) {
      if (MODE == 0) {            // POPC only (dependent chain per i keeps it from folding)
        x[i] = __popc(x[i]) + 0x10001u * i;  // 1 POPC + 1 IADD
      } else if (MODE == 1) {     // LOP3 only
        x[i] = (x[i] ^ y) & (x[(i + 1) % ILP] | 0x55555555u);
      } else if (MODE == 2) {     // IADD3 only
        x[i] = x[i] + y + x[(i + 1) % ILP];
      } else if (MODE == 3) {     // the kernel's pattern: XOR + POPC + accumulate
        acc[i] += __popc(x[i] ^ y);
        x[i] += 0x9e3779b9u;      // keep inputs changing (extra IADD)
      } else if (MODE == 4) {     // carry-save: 3 words -> 2 POPC
        unsigned a = x[i] ^ y, b = x[(i + 1) % ILP] ^ y, c = x[(i + 2) % ILP] ^ (y >> 1);
        unsigned s = a ^ b ^ c, cy = (a & b) | (c & (a ^ b));
        acc[i] += __popc(s) + 2 * __popc(cy);
        x[i] += 0x9e3779b9u;
      }
    }
    y += 0x7f4a7c15u;
  }
  long long t1 = clock64();
  unsigned r = 0;
#pragma unroll
  for (int i = 0; i < ILP; ++i) r ^= x[i] ^ acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = r;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char* name, double results_per_iter_lane, int sms) {
  unsigned* out; long long* cyc;
  CK(cudaMalloc(&out, sms * 1024 * 4)); CK(cudaMalloc(&cyc, sms * 8));
  pipe_kernel<MODE><<<sms, 1024>>>(out, cyc, 12345u);
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  pipe_kernel<MODE><<<sms, 1024>>>(out, cyc, 777u);
  cudaEventRecord(e1);
  CK(cudaDeviceSynchronize());
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  std::vector<long long> h(sms);
  CK(cudaMemcpy(h.data(), cyc, sms * 8, cudaMemcpyDeviceToHost));
  std::sort(h.begin(), h.end());
  const double lane_results = 1024.0 * ITERS * ILP * results_per_iter_lane;
  const double per_clk = lane_results / (double)h[sms / 2];
  const double total_per_s = lane_results * sms / (ms * 1e-3);
  printf("{\"bench\": \"%s\", \"results_per_clk_per_sm\": %.2f, \"median_cycles\": %lld, "
         "\"chip_results_per_s\": %.4e, \"ms\": %.4f, \"implied_mhz\": %.0f}\n",
         name, per_clk, h[sms / 2], total_per_s, ms, h[sms / 2] / (ms * 1e-3) / 1e6);
  cudaFree(out); cudaFree(cyc);
}

__global__ void copy_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = in[i];
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  int sms = prop.multiProcessorCount;
  printf("{\"device\": \"%s\", \"sms\": %d, \"cc\": \"%d.%d\", \"smem_optin\": %zu}\n", prop.name, sms,
         prop.major, prop.minor, (size_t)prop.sharedMemPerBlockOptin);
  run<0>("popc (+1 iadd)", 1.0, sms);
  run<1>("lop3 x2", 2.0, sms);
  run<2>("iadd3", 1.0, sms);
  run<3>("xor+popc+acc word-ops", 1.0, sms);
  run<4>("csa3 word-ops (3 words, 2 popc)", 3.0, sms);
  // HBM copy
  size_t bytes = (size_t)2 << 30;
  uint4 *a, *b; CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes));
  CK(cudaMemset(a, 1, bytes));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9;
  for (int r = 0; r < 6; ++r) {
    cudaEventRecord(e0);
    copy_kernel<<<sms * 16, 512>>>(a, b, bytes / 16);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    best = std::min(best, ms);
  }
  printf("{\"bench\": \"hbm copy 2GiB (read+write)\", \"GBps\": %.1f, \"ms\": %.3f}\n",
         2.0 * bytes / (best * 1e-3) / 1e9, best);
  return 0;
}
