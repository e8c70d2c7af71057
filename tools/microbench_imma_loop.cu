// tools/microbench_imma_loop.cu -- what throttles the IMMA inner loop of bconv_imma_kernel?
// 3 CTAs x 128 threads per SM (the kernel's residency), 16 accumulator tiles per warp.
//   mode 0: IMMA only (operands fixed in registers)
//   mode 1: + B fragments from shared memory (one LDS.64 per two IMMAs, as in the kernel)
//   mode 2: + A words from shared memory and the bits->bytes expansion (the full inner step)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench_imma_loop tools/microbench_imma_loop.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include <algorithm>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int KSTEPS = 16;     // k-steps (words) staged in shared memory
constexpr int ITERS = 256;

__device__ __forceinline__ void mma(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void expand01(uint32_t w, uint32_t sel, uint32_t& lo, uint32_t& hi) {
  const uint32_t byte = __byte_perm(w, 0u, sel);
  lo = ((byte & 0x0Fu) * 0x00204081u) & 0x01010101u;
  hi = ((byte >> 4) * 0x00204081u) & 0x01010101u;
}

template <int MODE>
__global__ void __launch_bounds__(128, 3) k(unsigned* out, long long* cycles, unsigned seed) {
  __shared__ uint2 B_s[KSTEPS * 8 * 32];
  __shared__ uint4 A_s[(KSTEPS / 4) * 128];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, gid = lane >> 2, tig = lane & 3;
  for (int i = tid; i < KSTEPS * 8 * 32; i += 128) B_s[i] = make_uint2(seed * (i + 1), seed ^ (i * 77u));
  for (int i = tid; i < (KSTEPS / 4) * 128; i += 128) A_s[i] = make_uint4(seed + i, seed * 3u + i, i * 5u, seed ^ i);
  __syncthreads();
  int acc[2][8][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[m][n][0] = acc[m][n][1] = acc[m][n][2] = acc[m][n][3] = n;
  uint32_t afix[2][4];
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int i = 0; i < 4; ++i) afix[m][i] = (seed * (tid + 7) + i) & 0x01010101u;
  uint32_t bfix0 = seed ^ tid, bfix1 = seed * 31u + tid;
  const uint32_t sel = 0x4440u | tig;
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll 1
    for (int kv = 0; kv < KSTEPS / 4; ++kv) {
      uint32_t a[4][2][4];
      if (MODE == 2) {
#pragma unroll
        for (int m = 0; m < 2; ++m) {
          const uint4 r0 = A_s[kv * 128 + warp * 32 + m * 16 + gid];
          const uint4 r1 = A_s[kv * 128 + warp * 32 + m * 16 + 8 + gid];
          const uint32_t w0[4] = {r0.x, r0.y, r0.z, r0.w}, w1[4] = {r1.x, r1.y, r1.z, r1.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            expand01(w0[q], sel, a[q][m][0], a[q][m][2]);
            expand01(w1[q], sel, a[q][m][1], a[q][m][3]);
          }
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int n = 0; n < 8; ++n) {
          uint2 b = make_uint2(bfix0, bfix1);
          if (MODE >= 1) b = B_s[((kv * 4 + q) * 8 + n) * 32 + lane];
          if (MODE == 2) { mma(acc[0][n], a[q][0], b.x, b.y); mma(acc[1][n], a[q][1], b.x, b.y); }
          else { mma(acc[0][n], afix[0], b.x, b.y); mma(acc[1][n], afix[1], b.x, b.y); }
        }
    }
  }
  long long t1 = clock64();
  unsigned r = 0;
#pragma unroll
  for (int m = 0; m < 2; ++m)
#pragma unroll
    for (int n = 0; n < 8; ++n) r ^= acc[m][n][0] ^ acc[m][n][1] ^ acc[m][n][2] ^ acc[m][n][3];
  out[blockIdx.x * 128 + tid] = r;
  if (tid == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char* name, int sms) {
  const int ctas = sms * 3;
  unsigned* out; long long* cyc;
  CK(cudaMalloc(&out, ctas * 128 * 4)); CK(cudaMalloc(&cyc, ctas * 8));
  k<MODE><<<ctas, 128>>>(out, cyc, 12345u);
  CK(cudaDeviceSynchronize());
  k<MODE><<<ctas, 128>>>(out, cyc, 777u);
  CK(cudaDeviceSynchronize());
  std::vector<long long> h(ctas);
  CK(cudaMemcpy(h.data(), cyc, ctas * 8, cudaMemcpyDeviceToHost));
  std::sort(h.begin(), h.end());
  // per SM: 3 CTAs x 4 warps x ITERS x KSTEPS x 16 IMMAs x 4096 MACs
  const double macs = 3.0 * 4 * ITERS * KSTEPS * 16 * 4096;
  printf("{\"bench\": \"%s\", \"int8_MACs_per_clk_per_sm\": %.1f, \"median_cycles\": %lld}\n", name,
         macs / (double)h[ctas / 2], h[ctas / 2]);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  run<0>("IMMA only, 12 warps/SM, 16 accumulator tiles per warp", sms);
  run<1>("+ B fragments by LDS.64 (1 per 2 IMMAs)", sms);
  run<2>("+ A words by LDS.128 and bits->bytes expansion (kernel's inner step)", sms);
  return 0;
}
