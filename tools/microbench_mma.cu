// tools/microbench_mma.cu -- does the GPU have a faster home for the binary inner product than
// the ALU/XU pipes? Measures, per SM clock (in-kernel clock64, 1024 threads per SM):
//   (a) legacy mma.sync.m16n8k32 s8 (IMMA)            -> int8 MACs / clk / SM
//   (b) mma.sync.m16n8k256 b1 and.popc (on sm_90a a native BMMA.168256.AND.POPC)
//                                                     -> binary MACs / clk / SM
//   (c) the kernel's carry-save XOR/POPC tree           -> binary MACs / clk / SM
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench_mma tools/microbench_mma.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <cstdint>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int ITERS = 2048;
constexpr int ILP = 4;

template <int MODE>
__global__ void __launch_bounds__(1024) k(unsigned* out, long long* cycles, unsigned seed) {
  unsigned a[4], b[2];
  int c[ILP][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = seed * (threadIdx.x + 3) + i * 0x9e3779b9u;
  b[0] = seed ^ (threadIdx.x * 0x85ebca6bu); b[1] = b[0] * 3u + 1u;
#pragma unroll
  for (int i = 0; i < ILP; ++i) { c[i][0] = c[i][1] = c[i][2] = c[i][3] = i; }
  __syncthreads();
  long long t0 = clock64();
#pragma unroll 1
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; ++i) {
      if (MODE == 0) {
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c[i][0]), "+r"(c[i][1]), "+r"(c[i][2]), "+r"(c[i][3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
      } else if (MODE == 1) {
        asm volatile("mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(c[i][0]), "+r"(c[i][1]), "+r"(c[i][2]), "+r"(c[i][3])
                     : "r"(a[0] + i), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
      } else {
        // 8 words x 4 outputs per (it, i): the kernel's xor_popc8_acc, weights = a[], activations vary
        unsigned w[8] = {a[0], a[1], a[2], a[3], b[0], b[1], a[0] ^ b[1], a[1] ^ b[0]};
#pragma unroll
        for (int o = 0; o < 4; ++o) {
          unsigned x[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) x[q] = w[q] ^ (unsigned)(c[i][o] + q * 0x01010101u + it);
          unsigned s1, c1, s2, c2, s3, c3, s4, c4;
          asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(s1) : "r"(x[0]), "r"(x[1]), "r"(x[2]));
          asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(c1) : "r"(x[0]), "r"(x[1]), "r"(x[2]));
          asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(s2) : "r"(x[3]), "r"(x[4]), "r"(x[5]));
          asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(c2) : "r"(x[3]), "r"(x[4]), "r"(x[5]));
          asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(s3) : "r"(s1), "r"(s2), "r"(x[6]));
          asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(c3) : "r"(s1), "r"(s2), "r"(x[6]));
          asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(s4) : "r"(c1), "r"(c2), "r"(c3));
          asm("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(c4) : "r"(c1), "r"(c2), "r"(c3));
          c[i][o] += __popc(s3) + __popc(x[7]) + 2 * __popc(s4) + 4 * __popc(c4);
        }
      }
    }
    a[0] += 0x7f4a7c15u;
  }
  long long t1 = clock64();
  unsigned r = 0;
#pragma unroll
  for (int i = 0; i < ILP; ++i) r ^= c[i][0] ^ c[i][1] ^ c[i][2] ^ c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = r;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int MODE>
void run(const char* name, double macs_per_warp_op, double lane_ops, int sms) {
  unsigned* out; long long* cyc;
  CK(cudaMalloc(&out, sms * 1024 * 4)); CK(cudaMalloc(&cyc, sms * 8));
  k<MODE><<<sms, 1024>>>(out, cyc, 12345u);
  CK(cudaDeviceSynchronize());
  k<MODE><<<sms, 1024>>>(out, cyc, 777u);
  CK(cudaDeviceSynchronize());
  std::vector<long long> h(sms);
  CK(cudaMemcpy(h.data(), cyc, sms * 8, cudaMemcpyDeviceToHost));
  std::sort(h.begin(), h.end());
  // MODE 0/1: one warp-wide op per (it, i) per warp; MODE 2: lane_ops word-ops per lane
  const double macs = MODE < 2 ? 32.0 * ITERS * ILP * macs_per_warp_op          // 32 warps per CTA
                               : 1024.0 * ITERS * ILP * lane_ops * 32.0;          // word-op = 32 MACs
  printf("{\"bench\": \"%s\", \"binary_or_int8_MACs_per_clk_per_sm\": %.1f, \"median_cycles\": %lld}\n",
         name, macs / (double)h[sms / 2], h[sms / 2]);
  cudaFree(out); cudaFree(cyc);
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  int sms = prop.multiProcessorCount;
  printf("{\"device\": \"%s\", \"sms\": %d}\n", prop.name, sms);
  run<0>("mma.sync m16n8k32 s8 (legacy IMMA), int8 MACs", 16.0 * 8 * 32, 0, sms);
  run<1>("mma.sync m16n8k256 b1 and.popc (native BMMA on sm_90a), binary MACs", 16.0 * 8 * 256, 0, sms);
  run<2>("carry-save XOR/POPC tree (this kernel), binary MACs", 0, 8.0 * 4, sms);
  return 0;
}
