// lce_b200_builtins.cu -- fp32 TFLite builtins as CUDA kernels (include/
// lce_b200_builtins.h). These are the callers either side of the binary path in the
// QuickNet / Bi-RealNet graphs, kept on the device so activations never leave HBM.
// Semantics follow TFLite's reference kernels (tensorflow/lite/kernels/internal/
// reference/conv.h:27, depthwiseconv_float.h:25, pooling.h:28,196, add.h,
// fully_connected.h:29, softmax.h:31, reduce.h); fp32 accumulate with FMA.
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cstdint>
#include <cstdlib>

#include "lce_b200.h"
#include "lce_b200_builtins.h"
#include "lce_b200_chain.cuh"

namespace lce_b200_internal {
int fail(const char* fmt, ...);       // lce_b200.cu
int launch_check(const char* what);   // lce_b200.cu
// wgmma tf32 pointwise convolution (lce_b200_pw.cuh): 0 launched, -1 not eligible
int pw_tf32_conv(const float* in, const float* filter, const float* bias, float* out, int32_t* packed, long long M, int N,
                 int K, int act, int pairs_ok, void* stream);
// wgmma tf32 7x7 / stride 2 / 3 -> 64 convolution (Bi-RealNet's stem): 0 launched, -1 not eligible
int stem7_tf32_conv(const float* in, const float* filter, const float* bias, float* out, int B, int H, int W, int OH, int OW,
                    int ph, int pw, int act, void* stream);
}  // namespace lce_b200_internal
using lce_b200_internal::fail;
using lce_b200_internal::launch_check;

namespace {

__device__ __forceinline__ float apply_act(float x, int act) {
  switch (act) {
    case LCE_ACT_RELU: return fmaxf(x, 0.0f);
    case LCE_ACT_RELU_N1_TO_1: return fminf(fmaxf(x, -1.0f), 1.0f);
    case LCE_ACT_RELU6: return fminf(fmaxf(x, 0.0f), 6.0f);
    default: return x;
  }
}

int out_size(int padding, int image, int filter, int stride, int dil) {
  const int eff = (filter - 1) * dil + 1;
  if (stride == 0) return 0;
  if (padding == LCE_PADDING_SAME) return (image + stride - 1) / stride;
  if (padding == LCE_PADDING_VALID) return (image + stride - eff) / stride;
  return 0;
}
int pad_before(int stride, int dil, int in, int filter, int out) {
  const int eff = (filter - 1) * dil + 1;
  int total = (out - 1) * stride + eff - in;
  if (total < 0) total = 0;
  return total / 2;
}
inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }
int grid_for(long long n, int per_block, int max_blocks = 132 * 32) {
  long long b = (n + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return static_cast<int>(b);
}

struct ConvGeom {
  int B, H, W, Cin, KH, KW, Cout, sh, sw, dh, dw, ph, pw, OH, OW, act;
};

// ---- small-K direct convolution (stem 3x3x3->16, 16->64 pointwise: K <= 32) --------
// One thread = one output pixel x 16 consecutive output channels; consecutive lanes
// take consecutive 16-channel groups of the same pixel, so a warp writes one
// contiguous span (coalesced 128-bit stores) and reads each input value once
// (broadcast). All weights sit in shared memory as [K][group][16 (+4 pad)].
constexpr int kDirectMaxK = 32;
constexpr int kDirectMaxCout = 128;
constexpr int kDirectGroupStride = 20;   // 16 + 4 floats: conflict-free LDS.128 across groups
// KH/KW/CIN > 0: compile-time shape (stem 3x3x3, pointwise 1x1x16) => fully unrolled K loop.
// Each thread computes kPX pixels x 16 channels so every 128-bit weight read from shared
// memory feeds 4*kPX FMAs (with one pixel per thread the kernel was LDS-bound: ncu showed
// short-scoreboard / MIO-throttle stalls dominating).
template <int KH_, int KW_, int CIN_, int kPX, bool kTileLoop = false>
__global__ void __launch_bounds__(128) conv_direct16_kernel(const float* __restrict__ in,
                                                            const float* __restrict__ filter,
                                                            const float* __restrict__ bias,
                                                            float* __restrict__ out, ConvGeom g,
                                                            long long M, int G, int tiles_per_block,
                                                            int32_t* __restrict__ packed) {
  extern __shared__ __align__(16) float w_s[];   // [K][G][20] then bias [G][16]
  const int KH = KH_ ? KH_ : g.KH, KW = KW_ ? KW_ : g.KW, CIN = CIN_ ? CIN_ : g.Cin;
  const int K = KH * KW * CIN;
  float* b_s = w_s + K * G * kDirectGroupStride;
  for (int i = threadIdx.x; i < K * G * 16; i += blockDim.x) {
    const int c = i & 15, gi = (i >> 4) % G, k = (i >> 4) / G;
    const int co = gi * 16 + c;
    w_s[(k * G + gi) * kDirectGroupStride + c] =
        co < g.Cout ? filter[static_cast<size_t>(co) * K + k] : 0.0f;
  }
  for (int i = threadIdx.x; i < G * 16; i += blockDim.x)
    b_s[i] = (bias && i < g.Cout) ? bias[i] : 0.0f;
  __syncthreads();
  // thread -> (pixel quad, channel group); consecutive lanes = consecutive groups, then pixels.
  // Pixel p of a thread is m0 + p * pstride with pstride = blockDim.x / G pixels, so that for
  // every p a warp still writes one contiguous span. 32-bit index math (host checks the range).
  const unsigned px_per_blk = blockDim.x / static_cast<unsigned>(G);
  const unsigned lpx = threadIdx.x / static_cast<unsigned>(G);
  const int gi = static_cast<int>(threadIdx.x - lpx * G);
  if (lpx >= px_per_blk) return;
  const unsigned ohw = g.OH * g.OW;
  // the weights staged above serve `tiles_per_block` consecutive pixel tiles
  const int n_tile = kTileLoop ? tiles_per_block : 1;
  for (int tile = 0; tile < n_tile; ++tile) {
  const unsigned blk_m0 = (blockIdx.x * n_tile + tile) * px_per_blk * kPX;
  if (blk_m0 >= static_cast<unsigned>(M)) break;
  long long ibase[kPX];
  int iy0[kPX], ix0[kPX];
  bool ok[kPX];
#pragma unroll
  for (int p = 0; p < kPX; ++p) {
    const unsigned mu = blk_m0 + p * px_per_blk + lpx;
    ok[p] = mu < static_cast<unsigned>(M);
    const unsigned mm = ok[p] ? mu : 0u;
    const unsigned bu = mm / ohw;
    const unsigned r = mm - bu * ohw;
    const unsigned oy = r / static_cast<unsigned>(g.OW), ox = r - oy * g.OW;
    iy0[p] = static_cast<int>(oy) * g.sh - g.ph;
    ix0[p] = static_cast<int>(ox) * g.sw - g.pw;
    ibase[p] = static_cast<long long>(bu) * g.H * g.W;
  }
  float acc[kPX][16];
#pragma unroll
  for (int p = 0; p < kPX; ++p)
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[p][c] = 0.0f;
  const float* wp = w_s + gi * kDirectGroupStride;
  auto fma16 = [&](const float (&x)[kPX], int k) {
    const float4* w4 = reinterpret_cast<const float4*>(wp + k * G * kDirectGroupStride);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 w = w4[q];
#pragma unroll
      for (int p = 0; p < kPX; ++p) {
        acc[p][4 * q] = fmaf(x[p], w.x, acc[p][4 * q]);
        acc[p][4 * q + 1] = fmaf(x[p], w.y, acc[p][4 * q + 1]);
        acc[p][4 * q + 2] = fmaf(x[p], w.z, acc[p][4 * q + 2]);
        acc[p][4 * q + 3] = fmaf(x[p], w.w, acc[p][4 * q + 3]);
      }
    }
  };
  auto tap = [&](int fy, int fx, int k0, int cin) {
    const float* src[kPX];
    bool inside[kPX];
#pragma unroll
    for (int p = 0; p < kPX; ++p) {
      const int iy = iy0[p] + fy * g.dh, ix = ix0[p] + fx * g.dw;
      inside[p] = ok[p] && static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
                  static_cast<unsigned>(ix) < static_cast<unsigned>(g.W);
      src[p] = in + (ibase[p] + static_cast<long long>(iy) * g.W + ix) * cin;
    }
    if (CIN_ > 0 && CIN_ % 4 == 0) {
#pragma unroll
      for (int c4 = 0; c4 < (CIN_ > 0 ? CIN_ / 4 : 1); ++c4) {
        float4 v[kPX];
#pragma unroll
        for (int p = 0; p < kPX; ++p)
          v[p] = inside[p] ? __ldg(reinterpret_cast<const float4*>(src[p]) + c4)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
        float x[kPX];
#pragma unroll
        for (int p = 0; p < kPX; ++p) x[p] = v[p].x;
        fma16(x, k0 + c4 * 4);
#pragma unroll
        for (int p = 0; p < kPX; ++p) x[p] = v[p].y;
        fma16(x, k0 + c4 * 4 + 1);
#pragma unroll
        for (int p = 0; p < kPX; ++p) x[p] = v[p].z;
        fma16(x, k0 + c4 * 4 + 2);
#pragma unroll
        for (int p = 0; p < kPX; ++p) x[p] = v[p].w;
        fma16(x, k0 + c4 * 4 + 3);
      }
    } else {
      for (int ci = 0; ci < cin; ++ci) {
        float x[kPX];
#pragma unroll
        for (int p = 0; p < kPX; ++p) x[p] = inside[p] ? __ldg(src[p] + ci) : 0.0f;
        fma16(x, k0 + ci);
      }
    }
  };
  if (KH_ > 0) {
#pragma unroll
    for (int fy = 0; fy < (KH_ > 0 ? KH_ : 1); ++fy)
#pragma unroll
      for (int fx = 0; fx < (KW_ > 0 ? KW_ : 1); ++fx) tap(fy, fx, (fy * KW_ + fx) * CIN_, CIN_);
  } else {
    for (int fy = 0; fy < KH; ++fy)
      for (int fx = 0; fx < KW; ++fx) tap(fy, fx, (fy * KW + fx) * CIN, CIN);
  }
  const int c0 = gi * 16;
  const float* bb = b_s + c0;
#pragma unroll
  for (int p = 0; p < kPX; ++p) {
    const long long m = static_cast<long long>(blk_m0) + p * px_per_blk + lpx;
    uint32_t bits = 0;
    if (ok[p]) {
      float* o = out + m * g.Cout + c0;
      if (c0 + 16 <= g.Cout && (g.Cout & 3) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 v = make_float4(apply_act(acc[p][4 * q] + bb[4 * q], g.act),
                                       apply_act(acc[p][4 * q + 1] + bb[4 * q + 1], g.act),
                                       apply_act(acc[p][4 * q + 2] + bb[4 * q + 2], g.act),
                                       apply_act(acc[p][4 * q + 3] + bb[4 * q + 3], g.act));
          reinterpret_cast<float4*>(o)[q] = v;
          bits |= ((v.x < 0.0f ? 1u : 0u) | (v.y < 0.0f ? 2u : 0u) | (v.z < 0.0f ? 4u : 0u) |
                   (v.w < 0.0f ? 8u : 0u)) << (4 * q);
        }
      } else {
        for (int c = 0; c < 16 && c0 + c < g.Cout; ++c) o[c] = apply_act(acc[p][c] + bb[c], g.act);
      }
    }
    if (packed != nullptr) {
      // fused LceQuantize (host guarantees Cout % 32 == 0 and an even group count): lanes gi and
      // gi ^ 1 are neighbours and hold the two halves of one word; every lane runs the shuffle
      uint32_t v = bits << ((gi & 1) * 16);
      v |= __shfl_xor_sync(0xffffffffu, v, 1);
      if (ok[p] && (gi & 1) == 0) packed[m * (g.Cout >> 5) + (gi >> 1)] = static_cast<int32_t>(v);
    }
  }
  }  // tile
}

// ---- plain-GEMM convolution (1x1, stride 1: A = [M, K] row-major): 128x128x16 tiles, 8x8
// outputs per thread, 128-bit global loads along K, register-prefetch double buffering ----
constexpr int kPM = 128, kPN = 128, kPK = 16;
__global__ void __launch_bounds__(256, 2) conv_gemm128_kernel(const float* __restrict__ A,
                                                           const float* __restrict__ Wt,
                                                           const float* __restrict__ bias,
                                                           float* __restrict__ out, long long M,
                                                           int N, int K, int act,
                                                           int32_t* __restrict__ packed) {
  __shared__ __align__(16) float A_s[2][kPK][kPM + 4];
  __shared__ __align__(16) float B_s[2][kPK][kPN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long m0 = static_cast<long long>(blockIdx.x) * kPM;
  const int n0 = blockIdx.y * kPN;
  // loader mapping: 2 float4 of A and 2 of B per thread per K-chunk
  const int lrow = tid >> 2;          // 0..63 (+64)
  const int lk = (tid & 3) * 4;       // 0,4,8,12
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  float4 ra[2], rb[2];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long m = m0 + lrow + 64 * h;
      const int n = n0 + lrow + 64 * h;
      const int k = k0 + lk;
      ra[h] = (m < M && k < K) ? __ldg(reinterpret_cast<const float4*>(A + m * K + k))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
      rb[h] = (n < N && k < K) ? __ldg(reinterpret_cast<const float4*>(Wt + static_cast<size_t>(n) * K + k))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + 64 * h;
      A_s[buf][lk][r] = ra[h].x; A_s[buf][lk + 1][r] = ra[h].y;
      A_s[buf][lk + 2][r] = ra[h].z; A_s[buf][lk + 3][r] = ra[h].w;
      B_s[buf][lk][r] = rb[h].x; B_s[buf][lk + 1][r] = rb[h].y;
      B_s[buf][lk + 2][r] = rb[h].z; B_s[buf][lk + 3][r] = rb[h].w;
    }
  };
  fetch(0);
  stash(0);
  __syncthreads();
  const int nk = (K + kPK - 1) / kPK;
  for (int it = 0; it < nk; ++it) {
    const int buf = it & 1;
    if (it + 1 < nk) fetch((it + 1) * kPK);
#pragma unroll
    for (int kk = 0; kk < kPK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&A_s[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&A_s[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&B_s[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&B_s[buf][kk][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) {
      stash(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    const bool row_ok = m < M;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        v[q] = apply_act(acc[i][jh * 4 + q] + ((bias && n + q < N) ? bias[n + q] : 0.0f), act);
      if (row_ok) {
        float* o = out + m * N + n;
        if (n + 3 < N && (N & 3) == 0) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        else
          for (int q = 0; q < 4 && n + q < N; ++q) o[q] = v[q];
      }
      if (packed != nullptr) {
        // fused LceQuantize (host guarantees N % 32 == 0): the 8 lanes tx & 7 = 0..7 hold one word
        uint32_t w = ((v[0] < 0.0f ? 1u : 0u) | (v[1] < 0.0f ? 2u : 0u) | (v[2] < 0.0f ? 4u : 0u) |
                      (v[3] < 0.0f ? 8u : 0u)) << ((tx & 7) * 4);
        w |= __shfl_xor_sync(0xffffffffu, w, 1);
        w |= __shfl_xor_sync(0xffffffffu, w, 2);
        w |= __shfl_xor_sync(0xffffffffu, w, 4);
        if (row_ok && (tx & 7) == 0 && n < N)
          packed[m * (N >> 5) + ((n0 + jh * 64) >> 5) + (tx >> 3)] = static_cast<int32_t>(w);
      }
    }
  }
}

// ---- plain GEMM for few output rows (FULLY_CONNECTED at batch 256: a 128 x 128 tiling would
// give 16 CTAs to 132 SMs): 32 x 64 tiles, 2 x 4 outputs per thread, K chunks of 32 ----
constexpr int kSM_ = 32, kSN_ = 64, kSK_ = 32;
__global__ void __launch_bounds__(256) gemm_small_m_kernel(const float* __restrict__ A,
                                                           const float* __restrict__ Wt,
                                                           const float* __restrict__ bias,
                                                           float* __restrict__ out, long long M,
                                                           int N, int K, int act) {
  __shared__ __align__(16) float A_s[kSK_][kSM_ + 2];
  __shared__ __align__(16) float B_s[kSK_][kSN_ + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long m0 = static_cast<long long>(blockIdx.x) * kSM_;
  const int n0 = blockIdx.y * kSN_;
  const int arow = tid >> 3, akq = (tid & 7) * 4;      // A: 32 rows x 8 float4
  const int bcol = tid >> 2, bkq = (tid & 3) * 8;      // B: 64 cols x 4 x 2 float4
  float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  for (int k0 = 0; k0 < K; k0 += kSK_) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 a = (m0 + arow < M && k0 + akq < K)
                         ? __ldg(reinterpret_cast<const float4*>(A + (m0 + arow) * K + k0 + akq)) : z;
    float4 b[2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
      b[h] = (n0 + bcol < N && k0 + bkq + 4 * h < K)
                 ? __ldg(reinterpret_cast<const float4*>(Wt + static_cast<size_t>(n0 + bcol) * K +
                                                         k0 + bkq + 4 * h)) : z;
    A_s[akq][arow] = a.x; A_s[akq + 1][arow] = a.y; A_s[akq + 2][arow] = a.z; A_s[akq + 3][arow] = a.w;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      B_s[bkq + 4 * h][bcol] = b[h].x; B_s[bkq + 4 * h + 1][bcol] = b[h].y;
      B_s[bkq + 4 * h + 2][bcol] = b[h].z; B_s[bkq + 4 * h + 3][bcol] = b[h].w;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kSK_; ++kk) {
      const float2 av = *reinterpret_cast<const float2*>(&A_s[kk][ty * 2]);
      const float4 bv = *reinterpret_cast<const float4*>(&B_s[kk][tx * 4]);
      acc[0][0] = fmaf(av.x, bv.x, acc[0][0]); acc[0][1] = fmaf(av.x, bv.y, acc[0][1]);
      acc[0][2] = fmaf(av.x, bv.z, acc[0][2]); acc[0][3] = fmaf(av.x, bv.w, acc[0][3]);
      acc[1][0] = fmaf(av.y, bv.x, acc[1][0]); acc[1][1] = fmaf(av.y, bv.y, acc[1][1]);
      acc[1][2] = fmaf(av.y, bv.z, acc[1][2]); acc[1][3] = fmaf(av.y, bv.w, acc[1][3]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const long long m = m0 + ty * 2 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < N) out[m * N + n] = apply_act(acc[i][j] + (bias ? bias[n] : 0.0f), act);
    }
  }
}

// ---- implicit-GEMM convolution, any filter / stride / dilation: 128 pixels x 64 channels x 16
// tiles, 8 x 4 outputs per thread, register-prefetch double buffering. The k -> (tap, channel)
// decomposition is tabulated once per CTA in shared memory (offset inside the image and the
// (dy, dx) displacement for the bounds test), so the gather costs ~8 instructions per element
// instead of three divisions. Bi-RealNet's 7x7x3 stem (K = 147) runs here.
constexpr int kIM = 128, kIN = 64, kIK = 16, kIKMax = 4096;
__global__ void __launch_bounds__(256, 2) conv_igemm_kernel(const float* __restrict__ in,
                                                            const float* __restrict__ filter,
                                                            const float* __restrict__ bias,
                                                            float* __restrict__ out, ConvGeom g,
                                                            long long M) {
  __shared__ __align__(16) float A_s[2][kIK][kIM + 4];
  __shared__ __align__(16) float B_s[2][kIK][kIN + 4];
  extern __shared__ int ktab[];  // [Kpad] element offset, [Kpad] (dy << 16) | dx
  const int K = g.KH * g.KW * g.Cin;
  const int Kpad = (K + kIK - 1) / kIK * kIK;
  int* koff = ktab;
  int* kdydx = ktab + Kpad;
  const int tid = threadIdx.x;
  for (int k = tid; k < Kpad; k += 256) {
    if (k < K) {
      const int tap = k / g.Cin, ci = k - tap * g.Cin;
      const int fy = tap / g.KW, fx = tap - fy * g.KW;
      koff[k] = (fy * g.dh * g.W + fx * g.dw) * g.Cin + ci;
      kdydx[k] = ((fy * g.dh) << 16) | (fx * g.dw);
    } else {
      koff[k] = 0;
      kdydx[k] = 0x7fff7fff;  // fails every bounds test
    }
  }
  const long long m0 = static_cast<long long>(blockIdx.x) * kIM;
  const int n0 = blockIdx.y * kIN;
  // loader roles: A -- row (tid & 127), 8 consecutive k; B -- channel (tid >> 2), 4 consecutive k
  const int lrow = tid & (kIM - 1);
  const int lkh = (tid >> 7) * 8;
  const int bn = tid >> 2, bkq = (tid & 3) * 4;
  int iy0 = 0, ix0 = 0;
  const float* base = in;
  bool row_ok = m0 + lrow < M;
  if (row_ok) {
    const long long m = m0 + lrow;
    const int ohw = g.OH * g.OW;
    const long long b = m / ohw;
    const int r = static_cast<int>(m - b * ohw);
    const int oy = r / g.OW, ox = r - oy * g.OW;
    iy0 = oy * g.sh - g.ph;
    ix0 = ox * g.sw - g.pw;
    base = in + ((b * g.H + iy0) * g.W + ix0) * g.Cin;  // dereferenced only where in bounds
  }
  const bool bn_ok = n0 + bn < g.Cout;
  const float* wrow = filter + static_cast<size_t>(bn_ok ? n0 + bn : 0) * K;
  __syncthreads();

  float ra[8], rb[4];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + lkh + e;
      const int d = kdydx[k];
      const int iy = iy0 + (d >> 16), ix = ix0 + (d & 0xffff);
      const bool ok = row_ok && static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
                      static_cast<unsigned>(ix) < static_cast<unsigned>(g.W);
      ra[e] = ok ? __ldg(base + koff[k]) : 0.0f;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = k0 + bkq + e;
      rb[e] = (bn_ok && k < K) ? __ldg(wrow + k) : 0.0f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < 8; ++e) A_s[buf][lkh + e][lrow] = ra[e];
#pragma unroll
    for (int e = 0; e < 4; ++e) B_s[buf][bkq + e][bn] = rb[e];
  };
  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  fetch(0);
  stash(0);
  __syncthreads();
  const int nk = Kpad / kIK;
  for (int it = 0; it < nk; ++it) {
    const int buf = it & 1;
    if (it + 1 < nk) fetch((it + 1) * kIK);
#pragma unroll
    for (int kk = 0; kk < kIK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&A_s[buf][kk][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&A_s[buf][kk][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&B_s[buf][kk][tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) {
      stash(buf ^ 1);
      __syncthreads();
    }
  }
  const int n = n0 + tx * 4;
  float bb[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) bb[q] = (bias && n + q < g.Cout) ? bias[n + q] : 0.0f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + ty * 8 + i;
    if (m >= M) continue;
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = apply_act(acc[i][q] + bb[q], g.act);
    float* o = out + m * g.Cout + n;
    if (n + 3 < g.Cout && (g.Cout & 3) == 0 && !(reinterpret_cast<uintptr_t>(out) & 15))
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
    else
      for (int q = 0; q < 4 && n + q < g.Cout; ++q) o[q] = v[q];
  }
}

// Same tiling with 128 threads and 8 x 8 outputs per thread (rows {ty*4.., 64+ty*4..}, channels
// {tx*4.., 32+tx*4..}): half the shared-memory reads per FMA of the 8 x 4 variant, whose ncu
// profile on Bi-RealNet's stem showed the LSU / shared-memory pipe at 61-75 % next to 53 % FMA.
__global__ void __launch_bounds__(128, 4) conv_igemm8x8_kernel(const float* __restrict__ in,
                                                               const float* __restrict__ filter,
                                                               const float* __restrict__ bias,
                                                               float* __restrict__ out, ConvGeom g,
                                                               long long M) {
  __shared__ __align__(16) float A_s[2][kIK][kIM + 4];
  __shared__ __align__(16) float B_s[2][kIK][kIN + 4];
  extern __shared__ int ktab[];
  const int K = g.KH * g.KW * g.Cin;
  const int Kpad = (K + kIK - 1) / kIK * kIK;
  int* koff = ktab;
  int* kdydx = ktab + Kpad;
  const int tid = threadIdx.x;
  for (int k = tid; k < Kpad; k += 128) {
    if (k < K) {
      const int tap = k / g.Cin, ci = k - tap * g.Cin;
      const int fy = tap / g.KW, fx = tap - fy * g.KW;
      koff[k] = (fy * g.dh * g.W + fx * g.dw) * g.Cin + ci;
      kdydx[k] = ((fy * g.dh) << 16) | (fx * g.dw);
    } else {
      koff[k] = 0;
      kdydx[k] = 0x7fff7fff;
    }
  }
  const long long m0 = static_cast<long long>(blockIdx.x) * kIM;
  const int n0 = blockIdx.y * kIN;
  // loader roles: A -- row tid, all 16 k of the chunk; B -- channel tid >> 1, 8 consecutive k
  const int lrow = tid;
  const int bn = tid >> 1, bkq = (tid & 1) * 8;
  int iy0 = 0, ix0 = 0;
  const float* base = in;
  const bool row_ok = m0 + lrow < M;
  if (row_ok) {
    const long long m = m0 + lrow;
    const int ohw = g.OH * g.OW;
    const long long b = m / ohw;
    const int r = static_cast<int>(m - b * ohw);
    const int oy = r / g.OW, ox = r - oy * g.OW;
    iy0 = oy * g.sh - g.ph;
    ix0 = ox * g.sw - g.pw;
    base = in + ((b * g.H + iy0) * g.W + ix0) * g.Cin;
  }
  const bool bn_ok = n0 + bn < g.Cout;
  const float* wrow = filter + static_cast<size_t>(bn_ok ? n0 + bn : 0) * K;
  __syncthreads();

  float ra[16], rb[8];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      const int k = k0 + e;
      const int d = kdydx[k];
      const int iy = iy0 + (d >> 16), ix = ix0 + (d & 0xffff);
      const bool ok = row_ok && static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
                      static_cast<unsigned>(ix) < static_cast<unsigned>(g.W);
      ra[e] = ok ? __ldg(base + koff[k]) : 0.0f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = k0 + bkq + e;
      rb[e] = (bn_ok && k < K) ? __ldg(wrow + k) : 0.0f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int e = 0; e < 16; ++e) A_s[buf][e][lrow] = ra[e];
#pragma unroll
    for (int e = 0; e < 8; ++e) B_s[buf][bkq + e][bn] = rb[e];
  };
  const int tx = tid & 7, ty = tid >> 3;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  fetch(0);
  stash(0);
  __syncthreads();
  const int nk = Kpad / kIK;
  for (int it = 0; it < nk; ++it) {
    const int buf = it & 1;
    if (it + 1 < nk) fetch((it + 1) * kIK);
#pragma unroll
    for (int kk = 0; kk < kIK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&A_s[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&A_s[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&B_s[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&B_s[buf][kk][32 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) {
      stash(buf ^ 1);
      __syncthreads();
    }
  }
  const bool vec = (g.Cout & 3) == 0 && !(reinterpret_cast<uintptr_t>(out) & 15);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 32 + tx * 4;
      float v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        v[q] = apply_act(acc[i][jh * 4 + q] + ((bias && n + q < g.Cout) ? bias[n + q] : 0.0f), g.act);
      float* o = out + m * g.Cout + n;
      if (vec && n + 3 < g.Cout) *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
      else
        for (int q = 0; q < 4 && n + q < g.Cout; ++q) o[q] = v[q];
    }
  }
}

// ---- general implicit-GEMM convolution: 64x64x16 tiles, 4x4 per thread (fallback for K > 4096) ----------
constexpr int kGM = 64, kGN = 64, kGK = 16;
__global__ void __launch_bounds__(256) conv_gemm_kernel(const float* __restrict__ in,
                                                        const float* __restrict__ filter,
                                                        const float* __restrict__ bias,
                                                        float* __restrict__ out, ConvGeom g,
                                                        long long M) {
  __shared__ __align__(16) float A_s[kGK][kGM + 4];
  __shared__ __align__(16) float B_s[kGK][kGN + 4];
  __shared__ long long pix_base[kGM];  // offset of (b, iy0, ix0) or -1 for rows past M
  __shared__ int pix_iy0[kGM], pix_ix0[kGM];
  const int K = g.KH * g.KW * g.Cin;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = static_cast<long long>(blockIdx.x) * kGM;
  const int n0 = blockIdx.y * kGN;
  if (tid < kGM) {
    const long long m = m0 + tid;
    if (m < M) {
      const int ohw = g.OH * g.OW;
      const long long b = m / ohw;
      const int r = static_cast<int>(m - b * ohw);
      const int oy = r / g.OW, ox = r - oy * g.OW;
      pix_iy0[tid] = oy * g.sh - g.ph;
      pix_ix0[tid] = ox * g.sw - g.pw;
      pix_base[tid] = b * g.H * g.W;
    } else {
      pix_base[tid] = -1;
      pix_iy0[tid] = pix_ix0[tid] = 0;
    }
  }
  __syncthreads();
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  const int lk = tid & 15;   // k within the chunk handled by this thread when loading
  const int lr = tid >> 4;   // row group: rows lr, lr+16, lr+32, lr+48
  for (int k0 = 0; k0 < K; k0 += kGK) {
    const int k = k0 + lk;
    int fy = 0, fx = 0, ci = 0;
    const bool k_ok = k < K;
    if (k_ok) {
      const int tap = k / g.Cin;
      ci = k - tap * g.Cin;
      fy = tap / g.KW;
      fx = tap - fy * g.KW;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int row = lr + 16 * q;
      float v = 0.0f;
      if (k_ok && pix_base[row] >= 0) {
        const int iy = pix_iy0[row] + fy * g.dh, ix = pix_ix0[row] + fx * g.dw;
        if (static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
            static_cast<unsigned>(ix) < static_cast<unsigned>(g.W))
          v = __ldg(in + (pix_base[row] + static_cast<long long>(iy) * g.W + ix) * g.Cin + ci);
      }
      A_s[lk][row] = v;
      const int n = n0 + row;
      B_s[lk][row] = (k_ok && n < g.Cout) ? __ldg(filter + static_cast<size_t>(n) * K + k) : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&A_s[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&B_s[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < g.Cout) out[m * g.Cout + n] = apply_act(acc[i][j] + (bias ? bias[n] : 0.0f), g.act);
    }
  }
}

__global__ void __launch_bounds__(256) depthwise_kernel(const float* __restrict__ in,
                                                        const float* __restrict__ filter,
                                                        const float* __restrict__ bias,
                                                        float* __restrict__ out, ConvGeom g,
                                                        long long n) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += stride) {
    const int c = static_cast<int>(i % g.Cout);
    long long r = i / g.Cout;
    const int ox = static_cast<int>(r % g.OW);
    r /= g.OW;
    const int oy = static_cast<int>(r % g.OH);
    const long long b = r / g.OH;
    float acc = 0.0f;
    for (int fy = 0; fy < g.KH; ++fy) {
      const int iy = oy * g.sh - g.ph + fy * g.dh;
      if (static_cast<unsigned>(iy) >= static_cast<unsigned>(g.H)) continue;
      for (int fx = 0; fx < g.KW; ++fx) {
        const int ix = ox * g.sw - g.pw + fx * g.dw;
        if (static_cast<unsigned>(ix) >= static_cast<unsigned>(g.W)) continue;
        acc = fmaf(__ldg(in + ((b * g.H + iy) * g.W + ix) * g.Cin + c),
                   __ldg(filter + (fy * g.KW + fx) * g.Cout + c), acc);
      }
    }
    out[i] = apply_act(acc + (bias ? bias[c] : 0.0f), g.act);
  }
}

// 4 channels per thread (C % 4 == 0): 128-bit loads of inputs, weights and outputs. 3-D grid
// (x: (ox, c4), y: oy, z: batch) -- the flat-index version spent most of its instructions on
// integer div/mod (ncu: issue-bound at ~30 % of DRAM bandwidth).
template <int KHW>   // KHW = 3: 3x3 window fully unrolled (all loads in flight); 0: runtime
__global__ void __launch_bounds__(256) depthwise_v4_kernel(const float4* __restrict__ in,
                                                           const float4* __restrict__ filter,
                                                           const float4* __restrict__ bias,
                                                           float4* __restrict__ out, ConvGeom g) {
  const int C4 = g.Cout >> 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.OW * C4) return;
  const int ox = i / C4, c = i - ox * C4;
  const int oy = blockIdx.y;
  const long long b = blockIdx.z;
  const int KH = KHW ? KHW : g.KH, KW = KHW ? KHW : g.KW;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4* img = in + b * g.H * g.W * C4 + c;
#pragma unroll
  for (int fy = 0; fy < KH; ++fy) {
    const int iy = oy * g.sh - g.ph + fy * g.dh;
    if (static_cast<unsigned>(iy) >= static_cast<unsigned>(g.H)) continue;
#pragma unroll
    for (int fx = 0; fx < KW; ++fx) {
      const int ix = ox * g.sw - g.pw + fx * g.dw;
      if (static_cast<unsigned>(ix) >= static_cast<unsigned>(g.W)) continue;
      const float4 x = __ldg(img + (static_cast<long long>(iy) * g.W + ix) * C4);
      const float4 w = __ldg(filter + (fy * KW + fx) * C4 + c);
      acc.x = fmaf(x.x, w.x, acc.x); acc.y = fmaf(x.y, w.y, acc.y);
      acc.z = fmaf(x.z, w.z, acc.z); acc.w = fmaf(x.w, w.w, acc.w);
    }
  }
  float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias) bb = __ldg(bias + c);
  out[((b * g.OH + oy) * g.OW + ox) * C4 + c] =
      make_float4(apply_act(acc.x + bb.x, g.act), apply_act(acc.y + bb.y, g.act),
                  apply_act(acc.z + bb.z, g.act), apply_act(acc.w + bb.w, g.act));
}

template <bool MAX, int FHW>   // FHW = 2 / 3: window fully unrolled; 0: runtime
__global__ void __launch_bounds__(256) pool_v4_kernel(const float4* __restrict__ in,
                                                      float4* __restrict__ out, int H, int W,
                                                      int C4, int OH, int OW, int fh_, int fw_,
                                                      int sh, int sw, int ph, int pw, int act) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= OW * C4) return;
  const int ox = i / C4, c = i - ox * C4;
  const int oy = blockIdx.y;
  const long long b = blockIdx.z;
  const int fh = FHW ? FHW : fh_, fw = FHW ? FHW : fw_;
  const int y0 = oy * sh - ph, x0 = ox * sw - pw;
  const float4* img = in + b * H * W * C4 + c;
  float4 v = MAX ? make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX)
                 : make_float4(0.f, 0.f, 0.f, 0.f);
  int cnt = 0;
#pragma unroll
  for (int fy = 0; fy < fh; ++fy) {
    const int y = y0 + fy;
    if (static_cast<unsigned>(y) >= static_cast<unsigned>(H)) continue;
#pragma unroll
    for (int fx = 0; fx < fw; ++fx) {
      const int x = x0 + fx;
      if (static_cast<unsigned>(x) >= static_cast<unsigned>(W)) continue;
      const float4 e = __ldg(img + (static_cast<long long>(y) * W + x) * C4);
      ++cnt;
      if (MAX) { v.x = fmaxf(v.x, e.x); v.y = fmaxf(v.y, e.y); v.z = fmaxf(v.z, e.z); v.w = fmaxf(v.w, e.w); }
      else { v.x += e.x; v.y += e.y; v.z += e.z; v.w += e.w; }
    }
  }
  if (!MAX) {
    const float d = static_cast<float>(max(1, cnt));
    v.x = v.x / d; v.y = v.y / d; v.z = v.z / d; v.w = v.w / d;
  }
  out[((b * OH + oy) * OW + ox) * C4 + c] =
      make_float4(apply_act(v.x, act), apply_act(v.y, act), apply_act(v.z, act),
                  apply_act(v.w, act));
}

// max-pool 2x2 / stride 1 / VALID fused into the depthwise 3x3 that consumes it: one thread =
// one output pixel x 4 channels; the 4x4 input window is loaded once (16 x LDG.128), the nine
// pooled values are formed in registers and multiplied in the same (fy, fx) order as
// depthwise_v4_kernel, so the result is bit-identical to the two-kernel sequence.
// On an H100 80GB HBM3 at a 700 W power limit, QuickNet batch 256 (per-node CUDA events, 200
// steps): 111.8 / 60.8 / 34.3 us for 56x56x64 / 28x28x128 / 14x14x256, 2.30 / 2.11 / 1.87 TB/s
// of operands read once and results written once. A tiled kernel that stages each tile's input
// window (4 output rows x 8 columns x 32 channels) in shared memory by cp.async, forms every
// pooled value once and blurs from there measured slower on the same card: 143.6 / 82.7 / 43.0 us
// one tile per CTA, 180.5 / 98.8 / 49.4 us persistent with a two-deep window buffer. So the
// one-thread-per-output kernel stays, and the reuse stays with L1.
#ifndef LCE_POOL_MINBLOCKS
#define LCE_POOL_MINBLOCKS 4
#endif
__global__ void __launch_bounds__(256, LCE_POOL_MINBLOCKS) pool2_dw3_v4_kernel(const float4* __restrict__ in,
                                                              const float4* __restrict__ filter,
                                                              const float4* __restrict__ bias,
                                                              float4* __restrict__ out, int H, int W,
                                                              int C4, int PH, int PW, int OH, int OW,
                                                              int sh, int sw, int ph, int pw, int act) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= OW * C4) return;
  const int ox = i / C4, c = i - ox * C4;
  const int oy = blockIdx.y;
  const long long b = blockIdx.z;
  const int y0 = oy * sh - ph, x0 = ox * sw - pw;   // top-left pooled coordinate of the window
  const float4* img = in + b * H * W * C4 + c;
  const float4 lowest = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
  auto vmax = [](const float4& a, const float4& q) {
    return make_float4(fmaxf(a.x, q.x), fmaxf(a.y, q.y), fmaxf(a.z, q.z), fmaxf(a.w, q.w));
  };
  // Interior windows (all 4 x 4 inputs and 3 x 3 pooled values exist; the whole warp agrees): the
  // same arithmetic in the same order with one base pointer and two constant strides. The general
  // path below spends 250 of its 600 instructions on per-load index arithmetic and predicates, and
  // the kernel is issue-bound (ncu: 68 % issue utilisation at half the HBM rate).
  if (__all_sync(__activemask(), y0 >= 0 && x0 >= 0 && y0 + 3 < H && x0 + 3 < W && y0 + 2 < PH && x0 + 2 < PW)) {
    const size_t cs = static_cast<size_t>(C4), rs = static_cast<size_t>(W) * cs;
    const float4* p0 = img + (static_cast<size_t>(y0) * W + x0) * cs;
    const float4* wp = filter + c;
    float4 hp[3];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) {
      const float4* row = p0 + dy * rs;
      const float4 v0 = __ldg(row), v1 = __ldg(row + cs), v2 = __ldg(row + 2 * cs), v3 = __ldg(row + 3 * cs);
      float4 h[3] = {vmax(v0, v1), vmax(v1, v2), vmax(v2, v3)};
      if (dy > 0) {
#pragma unroll
        for (int fx = 0; fx < 3; ++fx) {
          const float4 m = vmax(lowest, vmax(hp[fx], h[fx]));
          const float4 w = __ldg(wp + ((dy - 1) * 3 + fx) * cs);
          acc.x = fmaf(m.x, w.x, acc.x); acc.y = fmaf(m.y, w.y, acc.y);
          acc.z = fmaf(m.z, w.z, acc.z); acc.w = fmaf(m.w, w.w, acc.w);
        }
      }
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) hp[dx] = h[dx];
    }
    float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
    if (bias) bb = __ldg(bias + c);
    out[((b * OH + oy) * OW + ox) * C4 + c] =
        make_float4(apply_act(acc.x + bb.x, act), apply_act(acc.y + bb.y, act),
                    apply_act(acc.z + bb.z, act), apply_act(acc.w + bb.w, act));
    return;
  }
  // Row by row (one input row of 4 pixels live at a time: half the registers of holding the
  // 4 x 4 window, so twice the resident warps): h[x] = max(v[x], v[x+1]) per input row, a pooled
  // row is max(h of two consecutive input rows). max is exact in any order; the final
  // max(lowest, .) reproduces pool_v4_kernel's result for an all-NaN window too.
  bool xin[4];
#pragma unroll
  for (int dx = 0; dx < 4; ++dx) xin[dx] = static_cast<unsigned>(x0 + dx) < static_cast<unsigned>(W);
  float4 hp[3];   // h of the previous input row
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int dy = 0; dy < 4; ++dy) {
    const int y = y0 + dy;
    const bool yin = static_cast<unsigned>(y) < static_cast<unsigned>(H);
    const float4* row = img + (static_cast<long long>(y) * W + x0) * C4;
    float4 v[4];
#pragma unroll
    for (int dx = 0; dx < 4; ++dx) v[dx] = (yin && xin[dx]) ? __ldg(row + dx * C4) : lowest;
    float4 h[3];
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) h[dx] = vmax(v[dx], v[dx + 1]);
    if (dy > 0) {
      const int fy = dy - 1;
      const int py = y0 + fy;
      if (static_cast<unsigned>(py) < static_cast<unsigned>(PH)) {
#pragma unroll
        for (int fx = 0; fx < 3; ++fx) {
          const int px = x0 + fx;
          if (static_cast<unsigned>(px) >= static_cast<unsigned>(PW)) continue;
          const float4 m = vmax(lowest, vmax(hp[fx], h[fx]));
          const float4 w = __ldg(filter + (fy * 3 + fx) * C4 + c);
          acc.x = fmaf(m.x, w.x, acc.x); acc.y = fmaf(m.y, w.y, acc.y);
          acc.z = fmaf(m.z, w.z, acc.z); acc.w = fmaf(m.w, w.w, acc.w);
        }
      }
    }
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) hp[dx] = h[dx];
  }
  float4 bb = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias) bb = __ldg(bias + c);
  out[((b * OH + oy) * OW + ox) * C4 + c] =
      make_float4(apply_act(acc.x + bb.x, act), apply_act(acc.y + bb.y, act),
                  apply_act(acc.z + bb.z, act), apply_act(acc.w + bb.w, act));
}

template <bool MAX>
__global__ void __launch_bounds__(256) pool_kernel(const float* __restrict__ in,
                                                   float* __restrict__ out, int B, int H, int W,
                                                   int C, int OH, int OW, int fh, int fw, int sh,
                                                   int sw, int ph, int pw, int act) {
  const long long n = static_cast<long long>(B) * OH * OW * C;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += stride) {
    const int c = static_cast<int>(i % C);
    long long r = i / C;
    const int ox = static_cast<int>(r % OW);
    r /= OW;
    const int oy = static_cast<int>(r % OH);
    const long long b = r / OH;
    const int y0 = oy * sh - ph, x0 = ox * sw - pw;
    const int ys = max(0, y0), ye = min(H, y0 + fh), xs = max(0, x0), xe = min(W, x0 + fw);
    float v = MAX ? -FLT_MAX : 0.0f;
    for (int y = ys; y < ye; ++y)
      for (int x = xs; x < xe; ++x) {
        const float e = __ldg(in + ((b * H + y) * W + x) * C + c);
        v = MAX ? fmaxf(v, e) : v + e;
      }
    if (!MAX) v = v / static_cast<float>(max(1, (ye - ys) * (xe - xs)));  // pooling.h:60-78
    out[i] = apply_act(v, act);
  }
}

// TFLite's MAXIMUM and MINIMUM (reference/maximum_minimum.h): a comparison and a select, so a NaN in
// `a` gives b, and max(-0, +0) is the second operand
__device__ __forceinline__ float tfl_maximum(float a, float b) { return a > b ? a : b; }
__device__ __forceinline__ float tfl_minimum(float a, float b) { return a < b ? a : b; }

// OP 0 add, 1 mul, 2 activation only, 3 MAXIMUM, 4 MINIMUM, 5 DIV (IEEE division), 6 ROUND (halves
// to even, reference/round.h; b unused, no activation)
template <int OP>
__device__ __forceinline__ float eltwise_op(float x, float y) {
  if (OP == 0) return x + y;
  if (OP == 1) return x * y;
  if (OP == 3) return tfl_maximum(x, y);
  if (OP == 4) return tfl_minimum(x, y);
  if (OP == 5) return __fdiv_rn(x, y);
  if (OP == 6) return rintf(x);
  return x;
}

template <int OP>
__global__ void __launch_bounds__(256) eltwise_kernel(const float* __restrict__ a,
                                                      const float* __restrict__ b,
                                                      float* __restrict__ out, long long n,
                                                      long long b_len, int act, int vec_ok) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long t0 = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (vec_ok) {   // same shape, 16-byte aligned, n % 4 == 0: 128-bit path
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    float4* o4 = reinterpret_cast<float4*>(out);
    for (long long i = t0; i < (n >> 2); i += stride) {
      float4 x = a4[i];
      if (OP != 2) {
        const float4 y = OP == 6 ? x : b4[i];
        x = make_float4(eltwise_op<OP>(x.x, y.x), eltwise_op<OP>(x.y, y.y), eltwise_op<OP>(x.z, y.z),
                        eltwise_op<OP>(x.w, y.w));
      }
      o4[i] = make_float4(apply_act(x.x, act), apply_act(x.y, act), apply_act(x.z, act),
                          apply_act(x.w, act));
    }
    return;
  }
  if (OP != 2 && OP != 6 && b_len == 1) {   // a single-element b: one read, no index arithmetic
    const float y = __ldg(b);
    for (long long i = t0; i < n; i += stride) out[i] = apply_act(eltwise_op<OP>(a[i], y), act);
    return;
  }
  for (long long i = t0; i < n; i += stride) {
    const float x = a[i];
    out[i] = apply_act(OP == 2 || OP == 6 ? eltwise_op<OP>(x, x) : eltwise_op<OP>(x, b[i % b_len]), act);
  }
}

// lce_b200_f32_chain_sign: one pass of the per-channel chain (lce_b200_chain.cuh). PACK: one thread
// per (row, channel slot of a sign word), so each warp owns one packed word and ballots it (slots
// past `channels` give 0 bits); else one thread per element. x and out may be the same buffer.
template <bool PACK, typename I>
__global__ void __launch_bounds__(256) chain_sign_kernel(const float* x, const lce_chain_desc ch,
                                                         I rows, int channels, int cw, float* out,
                                                         int32_t* __restrict__ packed) {
  const bool has_si = ch.shift_in != nullptr, has_a = ch.alpha != nullptr;
  const bool has_so = ch.shift_out != nullptr, has_ss = ch.sign_shift != nullptr;
  const I span = PACK ? static_cast<I>(cw) * 32 : static_cast<I>(channels);
  const I n = rows * span;
  const I stride = static_cast<I>(gridDim.x) * blockDim.x;   // a multiple of 32: warps stay whole
  for (I i = static_cast<I>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const I row = i / span;
    const int c = static_cast<int>(i - row * span);
    bool bit = false;
    if (!PACK || c < channels) {
      const I e = row * channels + c;
      const float o = lce::chain_rprelu(x[e], has_si, has_si ? __ldg(ch.shift_in + c) : 0.0f, has_a,
                                        has_a ? __ldg(ch.alpha + c) : 0.0f, has_so,
                                        has_so ? __ldg(ch.shift_out + c) : 0.0f);
      if (out) out[e] = o;
      if (PACK) bit = lce::chain_sign(o, has_ss, has_ss ? __ldg(ch.sign_shift + c) : 0.0f);
    }
    if (PACK) {
      const unsigned word = __ballot_sync(0xffffffffu, bit);
      if ((threadIdx.x & 31) == 0) packed[i >> 5] = static_cast<int32_t>(word);
    }
  }
}

// lce_b200_f32_gate_sign: one pass of the gated tail (lce_b200_chain.cuh) over [batch][pixels][C],
// threads laid out as in chain_sign_kernel. x and out may be the same buffer. SPATIAL
// (lce_b200_f32_scale_sign): the gate row is the position row % pixels, not the image.
template <bool PACK, typename I, bool SPATIAL = false>
__global__ void __launch_bounds__(256) gate_sign_kernel(const float* x, const lce_gate_desc gd,
                                                        const float* __restrict__ residual, int act,
                                                        I rows, I pixels, int channels, int cw,
                                                        float* out, int32_t* __restrict__ packed) {
  const bool has_a = gd.alpha != nullptr;
  const bool has_sc = gd.sign_scale != nullptr, has_sh = gd.sign_shift != nullptr;
  const I span = PACK ? static_cast<I>(cw) * 32 : static_cast<I>(channels);
  const I n = rows * span;
  const I stride = static_cast<I>(gridDim.x) * blockDim.x;   // a multiple of 32: warps stay whole
  for (I i = static_cast<I>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const I row = i / span;
    const int c = static_cast<int>(i - row * span);
    bool bit = false;
    if (!PACK || c < channels) {
      const I e = row * channels + c;
      const I b = row / pixels;
      const I gi = SPATIAL ? row - b * pixels : b;
      float o = lce::gate_prelu(x[e], __ldg(gd.gate + gi * channels + c), has_a,
                                has_a ? __ldg(gd.alpha + c) : 0.0f);
      if (residual) o = __fadd_rn(o, residual[e]);
      o = apply_act(o, act);
      if (out) out[e] = o;
      if (PACK)
        bit = lce::affine_sign(o, has_sc, has_sc ? __ldg(gd.sign_scale + c) : 0.0f, has_sh,
                               has_sh ? __ldg(gd.sign_shift + c) : 0.0f);
    }
    if (PACK) {
      const unsigned word = __ballot_sync(0xffffffffu, bit);
      if ((threadIdx.x & 31) == 0) packed[i >> 5] = static_cast<int32_t>(word);
    }
  }
}

// lce_b200_f32_affine_sign: the signs of x * scale + shift over a strided [rows][channels] map,
// threads laid out as in chain_sign_kernel with the packed output; copy (optional) receives x.
template <typename I>
__global__ void __launch_bounds__(256) affine_sign_kernel(const float* __restrict__ x, I x_stride,
                                                          I rows, int channels, int cw,
                                                          const float* __restrict__ scale,
                                                          const float* __restrict__ shift,
                                                          int32_t* __restrict__ packed,
                                                          float* __restrict__ copy, I copy_stride) {
  const bool has_sc = scale != nullptr, has_sh = shift != nullptr;
  const I span = static_cast<I>(cw) * 32;
  const I n = rows * span;
  const I stride = static_cast<I>(gridDim.x) * blockDim.x;   // a multiple of 32: warps stay whole
  for (I i = static_cast<I>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const I row = i / span;
    const int c = static_cast<int>(i - row * span);
    bool bit = false;
    if (c < channels) {
      const float v = x[row * x_stride + c];
      if (copy) copy[row * copy_stride + c] = v;
      bit = lce::affine_sign(v, has_sc, has_sc ? __ldg(scale + c) : 0.0f, has_sh,
                             has_sh ? __ldg(shift + c) : 0.0f);
    }
    const unsigned word = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) packed[i >> 5] = static_cast<int32_t>(word);
  }
}

// lce_b200_f32_maxpool_affine_sign: MAX_POOL_2D -> MUL -> ADD -> LceQuantize in one pass. One warp
// per (output pixel, 32-channel word): lane l owns channel 32 * word + l, so every tap is one
// coalesced 128-byte read, and the ballot of the lanes' signs is the packed word (lanes past C vote
// 0). The window is visited in pool_kernel's order (rows, then columns, in-bounds taps only) from
// -FLT_MAX with fmaxf, then the pool's activation; FHW > 0 fixes a square window so the taps unroll.
// The max of channel `img[0]`'s in-bounds taps of the fh x fw window at (y0, x0) of an H x W x C map,
// visited in pool_kernel's order from -FLT_MAX with fmaxf.
template <typename I>
__device__ __forceinline__ float window_max(const float* __restrict__ img, int y0, int x0, int fh, int fw,
                                            int H, int W, int C) {
  float v = -FLT_MAX;
#pragma unroll
  for (int fy = 0; fy < fh; ++fy) {
    const int y = y0 + fy;
    if (static_cast<unsigned>(y) >= static_cast<unsigned>(H)) continue;
#pragma unroll
    for (int fx = 0; fx < fw; ++fx) {
      const int xx = x0 + fx;
      if (static_cast<unsigned>(xx) >= static_cast<unsigned>(W)) continue;
      v = fmaxf(v, __ldg(img + (static_cast<I>(y) * W + xx) * C));
    }
  }
  return v;
}

template <int FHW, typename I>
__global__ void __launch_bounds__(256) maxpool_affine_sign_kernel(
    const float* __restrict__ x, int H, int W, int C, int OH, int OW, int cw, int fh_, int fw_, int sh,
    int sw, int ph, int pw, int act, const float* __restrict__ scale, const float* __restrict__ shift,
    int32_t* __restrict__ packed, I words) {
  const bool has_sc = scale != nullptr, has_sh = shift != nullptr;
  const int fh = FHW ? FHW : fh_, fw = FHW ? FHW : fw_;
  const int lane = threadIdx.x & 31;
  const I warps = static_cast<I>(gridDim.x) * (blockDim.x >> 5);
  for (I wi = static_cast<I>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); wi < words; wi += warps) {
    const I pix = wi / cw;
    const int c = static_cast<int>(wi - pix * cw) * 32 + lane;
    const int ox = static_cast<int>(pix % OW);
    const I r = pix / OW;
    const int oy = static_cast<int>(r % OH);
    const I b = r / OH;
    bool bit = false;
    if (c < C) {
      const int y0 = oy * sh - ph, x0 = ox * sw - pw;
      const float v = window_max<I>(x + b * H * W * C + c, y0, x0, fh, fw, H, W, C);
      bit = lce::affine_sign(apply_act(v, act), has_sc, has_sc ? __ldg(scale + c) : 0.0f, has_sh,
                             has_sh ? __ldg(shift + c) : 0.0f);
    }
    const unsigned word = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) packed[wi] = static_cast<int32_t>(word);
  }
}

// lce_b200_f32_quant2_planes: [MAX_POOL_2D ->] the 2-bit DoReFa quantiser in one pass, threads laid
// out as in maxpool_affine_sign_kernel (C % 32 == 0, so every lane owns a channel). The level
// q = rint(min(max(v, 0), 1) * 3) in {0, 1, 2, 3} is computed with the float operations of the MAXIMUM
// -> MINIMUM -> MUL -> ROUND builtins; the ballots of its two bits are the word of plane 0 and of
// plane 1, and a pixel's 3 * cw output words are [plane 0 | plane 1 | plane 1], so a binary
// convolution over 3 * C channels with each tap's filter words repeated three times accumulates
// plane 0 + 2 * plane 1. FHW == 1 is the quantiser alone (no window, no pool activation).
template <int FHW, typename I>
__global__ void __launch_bounds__(256) quant2_planes_kernel(
    const float* __restrict__ x, int H, int W, int C, int OH, int OW, int cw, int fh_, int fw_, int sh,
    int sw, int ph, int pw, int act, int32_t* __restrict__ planes, I words) {
  const int fh = FHW ? FHW : fh_, fw = FHW ? FHW : fw_;
  const int lane = threadIdx.x & 31;
  const I warps = static_cast<I>(gridDim.x) * (blockDim.x >> 5);
  for (I wi = static_cast<I>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); wi < words; wi += warps) {
    const I pix = wi / cw;
    const int word = static_cast<int>(wi - pix * cw);
    float v;
    if (FHW == 1) {
      v = __ldg(x + pix * C + word * 32 + lane);
    } else {
      const int ox = static_cast<int>(pix % OW);
      const I r = pix / OW;
      const int oy = static_cast<int>(r % OH);
      const I b = r / OH;
      v = apply_act(window_max<I>(x + b * H * W * C + word * 32 + lane, oy * sh - ph, ox * sw - pw, fh, fw,
                                  H, W, C), act);
    }
    const int q = static_cast<int>(rintf(__fmul_rn(tfl_minimum(tfl_maximum(v, 0.0f), 1.0f), 3.0f)));
    const unsigned p0 = __ballot_sync(0xffffffffu, q & 1);
    const unsigned p1 = __ballot_sync(0xffffffffu, q & 2);
    if (lane < 3) planes[pix * (3 * cw) + lane * cw + word] = static_cast<int32_t>(lane == 0 ? p0 : p1);
  }
}

// lce_b200_f32_shift_sign_planes: ABC-Net's N shifted signs of one float map, N x (ADD(x, shift_k) ->
// LceQuantize), in one pass; one warp per pixel and 32-channel word, as quant2_planes_kernel.
struct ShiftPlanes {
  float shift[8];
  int32_t* planes[8];
};
template <typename I>
__global__ void __launch_bounds__(256) shift_sign_planes_kernel(const float* __restrict__ x, int C, int cw, int n,
                                                                const __grid_constant__ ShiftPlanes sp, I words) {
  const int lane = threadIdx.x & 31;
  const I warps = static_cast<I>(gridDim.x) * (blockDim.x >> 5);
  for (I wi = static_cast<I>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); wi < words; wi += warps) {
    const I pix = wi / cw;
    const int word = static_cast<int>(wi - pix * cw);
    const float v = __ldg(x + pix * C + word * 32 + lane);
    for (int k = 0; k < n; ++k) {
      const unsigned b = __ballot_sync(0xffffffffu, __fadd_rn(v, sp.shift[k]) < 0.0f);
      if (lane == 0) sp.planes[k][wi] = static_cast<int32_t>(b);
    }
  }
}

// RESIZE_NEAREST_NEIGHBOR / RESIZE_BILINEAR (reference/resize_nearest_neighbor.h, resize_bilinear.h).
// One axis of the resize: the host computes `scale` as the reference does, in float; every step here
// is one explicitly rounded operation so that nvcc contracts nothing into an FMA.
struct ResizeAxis {
  int in, out;
  float scale;
};
struct ResizeGeom {
  ResizeAxis y, x;
  int batch, C;
  int align_corners, half_pixel_centers;
};
// GetNearestNeighbor: the source index of output index o
__device__ __forceinline__ int nearest_src(int o, const ResizeAxis& a, int align, int half) {
  const float v = __fmul_rn(__fadd_rn(static_cast<float>(o), half ? 0.5f : 0.0f), a.scale);
  int s = min(align ? static_cast<int>(roundf(v)) : static_cast<int>(floorf(v)), a.in - 1);
  if (half) s = max(s, 0);
  return s;
}
// ComputeInterpolationValues: the source coordinate v and its clamped neighbours lo, hi
__device__ __forceinline__ float bilinear_src(int o, const ResizeAxis& a, int half, int* lo, int* hi) {
  const float of = static_cast<float>(o);
  const float v = half ? __fsub_rn(__fmul_rn(__fadd_rn(of, 0.5f), a.scale), 0.5f) : __fmul_rn(of, a.scale);
  *lo = max(static_cast<int>(floorf(v)), 0);
  *hi = min(static_cast<int>(ceilf(v)), a.in - 1);
  return v;
}

// The resize kernels walk the output by rows: blockIdx.y strides over the B * OH output rows, so each
// row's source rows (and for the bilinear one its vertical weight) are found once per thread and row,
// and blockIdx.x / threadIdx.x stride over the row's OW * C floats, taken VEC = 4 at a time when the
// row is a whole number of 16-byte float4s (a float4 may span two pixels when C % 4 != 0, as at the
// 21 classes of a segmentation head), else one at a time. Element offsets are 64-bit; a row's own
// index is 32-bit (the host refuses rows within 2^22 floats of 2^31).
template <int VEC>
__global__ void __launch_bounds__(256) resize_nearest_kernel(const float* __restrict__ in,
                                                             float* __restrict__ out, ResizeGeom g) {
  const int row_len = g.x.out * g.C;
  for (long long row = blockIdx.y; row < static_cast<long long>(g.y.out) * g.batch; row += gridDim.y) {
    const long long b = row / g.y.out;
    const int sy = nearest_src(static_cast<int>(row - b * g.y.out), g.y, g.align_corners, g.half_pixel_centers);
    const float* src = in + (b * g.y.in + sy) * g.x.in * g.C;
    float* dst = out + row * row_len;
    for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * VEC; j < row_len; j += gridDim.x * blockDim.x * VEC) {
      int ox = j / g.C, c = j - ox * g.C;
      float v[VEC];
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        v[k] = __ldg(src + nearest_src(ox, g.x, g.align_corners, g.half_pixel_centers) * g.C + c);
        if (++c == g.C) { c = 0; ++ox; }
      }
      if (VEC == 4) reinterpret_cast<float4*>(dst)[j >> 2] = make_float4(v[0], v[1], v[2], v[3]);
      else dst[j] = v[0];
    }
  }
}

__device__ __forceinline__ float bilinear_mix(float x00, float x10, float x01, float x11, float dy, float dx) {
  // x00*(1-dy)*(1-dx) + x10*dy*(1-dx) + x01*(1-dy)*dx + x11*dy*dx, left to right, every step rounded
  const float ey = __fsub_rn(1.0f, dy), ex = __fsub_rn(1.0f, dx);
  float s = __fmul_rn(__fmul_rn(x00, ey), ex);
  s = __fadd_rn(s, __fmul_rn(__fmul_rn(x10, dy), ex));
  s = __fadd_rn(s, __fmul_rn(__fmul_rn(x01, ey), dx));
  return __fadd_rn(s, __fmul_rn(__fmul_rn(x11, dy), dx));
}

template <int VEC>
__global__ void __launch_bounds__(256) resize_bilinear_kernel(const float* __restrict__ in,
                                                              float* __restrict__ out, ResizeGeom g) {
  const int row_len = g.x.out * g.C;
  for (long long row = blockIdx.y; row < static_cast<long long>(g.y.out) * g.batch; row += gridDim.y) {
    const long long b = row / g.y.out;
    int y0, y1;
    const float vy = bilinear_src(static_cast<int>(row - b * g.y.out), g.y, g.half_pixel_centers, &y0, &y1);
    // the weights come from the clamped lower neighbours, as in the reference
    const float dy = __fsub_rn(vy, static_cast<float>(y0));
    const float* src0 = in + (b * g.y.in + y0) * g.x.in * g.C;
    const float* src1 = in + (b * g.y.in + y1) * g.x.in * g.C;
    float* dst = out + row * row_len;
    for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * VEC; j < row_len; j += gridDim.x * blockDim.x * VEC) {
      int ox = j / g.C, c = j - ox * g.C;
      float v[VEC];
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        int x0, x1;
        const float vx = bilinear_src(ox, g.x, g.half_pixel_centers, &x0, &x1);
        const float dx = __fsub_rn(vx, static_cast<float>(x0));
        v[k] = bilinear_mix(__ldg(src0 + x0 * g.C + c), __ldg(src1 + x0 * g.C + c), __ldg(src0 + x1 * g.C + c),
                            __ldg(src1 + x1 * g.C + c), dy, dx);
        if (++c == g.C) { c = 0; ++ox; }
      }
      if (VEC == 4) reinterpret_cast<float4*>(dst)[j >> 2] = make_float4(v[0], v[1], v[2], v[3]);
      else dst[j] = v[0];
    }
  }
}

// lce_b200_f32_upsample_add_sign: a decoder merge RESIZE_NEAREST_NEIGHBOR(u) -> ADD(skip) [->
// LceQuantize] in one pass, by output rows as the resize kernels. One warp per output pixel and
// 32-channel word, as shift_sign_planes_kernel: lane l reads channel 32 * word + l of u at the nearest
// source pixel and of skip, adds them as the ADD builtin does (one rounding, then its activation),
// stores the sum when `out` is set and ballots the signs into the packed word when `packed` is set
// (lanes past C vote 0).
__global__ void __launch_bounds__(256) upsample_add_sign_kernel(const float* __restrict__ u,
                                                                const float* __restrict__ skip, ResizeGeom g,
                                                                int cw, int act, float* __restrict__ out,
                                                                int32_t* __restrict__ packed) {
  const int lane = threadIdx.x & 31;
  const int row_words = g.x.out * cw;
  for (long long row = blockIdx.y; row < static_cast<long long>(g.y.out) * g.batch; row += gridDim.y) {
    const long long b = row / g.y.out;
    const int sy = nearest_src(static_cast<int>(row - b * g.y.out), g.y, g.align_corners, g.half_pixel_centers);
    const float* src = u + (b * g.y.in + sy) * g.x.in * g.C;
    for (int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < row_words; w += gridDim.x * (blockDim.x >> 5)) {
      const int ox = w / cw;
      const int c = (w - ox * cw) * 32 + lane;
      bool bit = false;
      if (c < g.C) {
        const long long at = (row * g.x.out + ox) * g.C + c;
        const int sx = nearest_src(ox, g.x, g.align_corners, g.half_pixel_centers);
        const float s = apply_act(__fadd_rn(__ldg(src + sx * g.C + c), __ldg(skip + at)), act);
        if (out) out[at] = s;
        bit = lce::chain_sign(s, false, 0.0f);
      }
      const unsigned word = __ballot_sync(0xffffffffu, bit);
      if (packed && lane == 0) packed[row * row_words + w] = static_cast<int32_t>(word);
    }
  }
}

// ARG_MAX (reference/arg_min_max.h, ArgMinMax with std::greater) over x [outer, n, inner]: for each
// (outer, inner) position v = x[0], idx = 0, then x[i] is taken only when x[i] > v. So ties go to the
// lowest index (-0.0 == +0.0), a NaN at index 0 gives 0 and a NaN elsewhere is never taken. Split
// across lanes, the same result is 0 when x[0] is NaN and otherwise the max of the non-NaN values by
// (value, lowest index): an associative and commutative merge.
struct ArgBest {
  float v;
  int i;   // -1: no non-NaN value seen yet
};
// x[i], with i increasing from one call to the next
__device__ __forceinline__ void argbest_take(ArgBest& a, float v, int i) {
  if (!isnan(v) && (a.i < 0 || v > a.v)) {
    a.v = v;
    a.i = i;
  }
}
__device__ __forceinline__ ArgBest argbest_merge(ArgBest a, ArgBest b) {
  if (b.i < 0) return a;
  return a.i < 0 || b.v > a.v || (b.v == a.v && b.i < a.i) ? b : a;
}

// One thread per (outer, inner) position, walking the axis as the reference does: adjacent threads
// read adjacent inner positions, so the loads coalesce when inner > 1; at inner == 1 (short rows)
// each thread reads its own row.
template <typename OutT>
__global__ void __launch_bounds__(256) argmax_kernel(const float* __restrict__ in, long long outer, int n,
                                                     long long inner, OutT* __restrict__ out) {
  const long long total = outer * inner;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long o = p / inner;
    const float* x = in + o * n * inner + (p - o * inner);
    float v = __ldg(x);
    int idx = 0;
    for (int i = 1; i < n; ++i) {
      const float xi = __ldg(x + i * inner);
      if (xi > v) {
        v = xi;
        idx = i;
      }
    }
    out[p] = static_cast<OutT>(idx);
  }
}

// One warp per row at inner == 1 (long rows): lane l takes elements l, l + 32, ... in order, then the
// lanes merge their (value, index) pairs.
template <typename OutT>
__global__ void __launch_bounds__(256) argmax_warp_kernel(const float* __restrict__ in, long long rows, int n,
                                                          OutT* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long r = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
       r += warps) {
    const float* x = in + r * n;
    ArgBest b{0.0f, -1};
    for (int i = lane; i < n; i += 32) argbest_take(b, __ldg(x + i), i);
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      const ArgBest o{__shfl_xor_sync(0xffffffffu, b.v, off), __shfl_xor_sync(0xffffffffu, b.i, off)};
      b = argbest_merge(b, o);
    }
    if (lane == 0) out[r] = static_cast<OutT>(isnan(__ldg(x)) ? 0 : b.i);
  }
}

// REDUCE_MAX (lce_b200_f32_reduce_max). One thread per (outer, inner) position, walking the axis as the
// reference does (cur = -FLT_MAX, then cur = x > cur ? x : cur): adjacent threads read adjacent inner
// positions, so the loads coalesce when inner > 1; at inner == 1 (short rows) each thread reads its own row.
__global__ void __launch_bounds__(256) reduce_max_kernel(const float* __restrict__ in, long long outer, long long n,
                                                         long long inner, float* __restrict__ out) {
  const long long total = outer * inner;
  for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < total;
       p += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long o = p / inner;
    const float* x = in + o * n * inner + (p - o * inner);
    float cur = -FLT_MAX;
    for (long long i = 0; i < n; ++i) {
      const float xi = __ldg(x + i * inner);
      cur = xi > cur ? xi : cur;
    }
    out[p] = cur;
  }
}

// One warp per row at inner == 1 (long rows): lane l walks elements l, l + 32, ... by the same rule and
// keeps the index of its value (-1 for the initial one); the lanes then merge, the larger value or of
// equal ones the lower index winning, which is what the sequential walk keeps.
__global__ void __launch_bounds__(256) reduce_max_warp_kernel(const float* __restrict__ in, long long rows,
                                                              long long n, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warps = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
  for (long long r = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5); r < rows;
       r += warps) {
    const float* x = in + r * n;
    float v = -FLT_MAX;
    long long idx = LLONG_MAX;
    for (long long i = lane; i < n; i += 32) {
      const float xi = __ldg(x + i);
      if (xi > v) {
        v = xi;
        idx = i;
      }
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, off);
      const long long oi = __shfl_xor_sync(0xffffffffu, idx, off);
      if (ov > v || (ov == v && oi < idx)) {
        v = ov;
        idx = oi;
      }
    }
    if (lane == 0) out[r] = v;
  }
}

// RESIZE_BILINEAR -> ARG_MAX over the channel axis in one pass, by output rows as
// resize_bilinear_kernel: blockIdx.y strides over the B * OH output rows. The CTA stages the row's two
// source rows y0 and y1 (in_w * C floats each, as float4s when both are 16-byte aligned) in shared
// memory; then each thread takes one output pixel, computes its C values with bilinear_src and
// bilinear_mix exactly as the resize kernel does and keeps ARG_MAX's running index over them. Only the
// label is stored; the resized map is never written.
template <typename OutT>
__global__ void __launch_bounds__(256) bilinear_argmax_kernel(const float* __restrict__ in, ResizeGeom g,
                                                              OutT* __restrict__ out) {
  extern __shared__ float4 stage4[];
  const int src_len = g.x.in * g.C;
  float* s0 = reinterpret_cast<float*>(stage4);
  float* s1 = s0 + src_len;
  for (long long row = blockIdx.y; row < static_cast<long long>(g.y.out) * g.batch; row += gridDim.y) {
    const long long b = row / g.y.out;
    int y0, y1;
    const float vy = bilinear_src(static_cast<int>(row - b * g.y.out), g.y, g.half_pixel_centers, &y0, &y1);
    const float dy = __fsub_rn(vy, static_cast<float>(y0));
    const float* src0 = in + (b * g.y.in + y0) * src_len;
    const float* src1 = in + (b * g.y.in + y1) * src_len;
    __syncthreads();   // every thread is done with the previous row's stage
    if (src_len % 4 == 0 && !((reinterpret_cast<uintptr_t>(src0) | reinterpret_cast<uintptr_t>(src1)) & 15)) {
      for (int j = threadIdx.x; j < src_len / 4; j += blockDim.x) {
        reinterpret_cast<float4*>(s0)[j] = __ldg(reinterpret_cast<const float4*>(src0) + j);
        reinterpret_cast<float4*>(s1)[j] = __ldg(reinterpret_cast<const float4*>(src1) + j);
      }
    } else {
      for (int j = threadIdx.x; j < src_len; j += blockDim.x) {
        s0[j] = __ldg(src0 + j);
        s1[j] = __ldg(src1 + j);
      }
    }
    __syncthreads();
    for (int ox = threadIdx.x; ox < g.x.out; ox += blockDim.x) {
      int x0, x1;
      const float vx = bilinear_src(ox, g.x, g.half_pixel_centers, &x0, &x1);
      const float dx = __fsub_rn(vx, static_cast<float>(x0));
      const float* p00 = s0 + x0 * g.C;
      const float* p10 = s1 + x0 * g.C;
      const float* p01 = s0 + x1 * g.C;
      const float* p11 = s1 + x1 * g.C;
      float v = bilinear_mix(p00[0], p10[0], p01[0], p11[0], dy, dx);
      int idx = 0;
      for (int c = 1; c < g.C; ++c) {
        const float vc = bilinear_mix(p00[c], p10[c], p01[c], p11[c], dy, dx);
        if (vc > v) {
          v = vc;
          idx = c;
        }
      }
      out[row * g.x.out + ox] = static_cast<OutT>(idx);
    }
  }
}

// DEPTH_TO_SPACE (reference/depth_to_space.h): out[b, y*r + i, x*r + j, c] = in[b, y, x, (i*r + j)*C' + c]
// with C' = C / r^2. By output rows as the resize kernels: blockIdx.y strides over the B * H * r output
// rows, and an output row (b, Y) is W runs of r * C' contiguous floats, run x read from LR pixel
// (b, Y / r, x) at channel (Y % r) * r * C'. Consecutive threads store consecutive floats (VEC = 4 at a
// time when a run is a whole number of float4s). Element offsets are 64-bit; an index within a row is
// 32-bit (the host refuses rows within 2^22 floats of 2^31).
template <int VEC>
__global__ void __launch_bounds__(256) depth_to_space_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                             int H, int W, int C, int r, long long rows) {
  const int run = C / r;   // r * C'
  const int row_len = W * run;
  for (long long row = blockIdx.y; row < rows; row += gridDim.y) {
    const long long by = row / r;   // b * H + y
    const int i = static_cast<int>(row - by * r);
    const float* src = in + by * W * C + i * run;
    float* dst = out + row * row_len;
    for (int j = (blockIdx.x * blockDim.x + threadIdx.x) * VEC; j < row_len; j += gridDim.x * blockDim.x * VEC) {
      const int x = j / run, t = j - x * run;
      const float* s = src + static_cast<long long>(x) * C + t;
      if (VEC == 4) reinterpret_cast<float4*>(dst)[j >> 2] = __ldg(reinterpret_cast<const float4*>(s));
      else dst[j] = __ldg(s);
    }
  }
}

// TRANSPOSE_CONV (reference/transpose_conv.h) as a gather: output pixel (oy, ox) of phase
// ((oy + pad_h) mod s_h, (ox + pad_w) mod s_w) is a stride-1 convolution over the input with only the
// taps fy = oy + pad_h - iy * s_h, fx = ox + pad_w - ix * s_w that land in the filter. Each thread
// computes one output pixel x 4 consecutive channels; consecutive threads take consecutive channel
// groups of one pixel, so the input row is a broadcast and the stores are coalesced. Every output is
// one fmaf chain from 0.0f over the taps in the reference's scatter order (input rows, then columns,
// ascending) and, within a tap, the input channels ascending; then one __fadd_rn of the bias and the
// activation, as the reference zeroes, accumulates, adds the bias and clamps. No atomics: the result
// does not depend on scheduling. VEC4: in_c % 4 == 0 and 16-byte aligned input and filter.
struct TConvGeom {
  int B, H, W, Cin, KH, KW, Cout, OH, OW, sh, sw, ph, pw, act;
};
template <bool VEC4>
__global__ void __launch_bounds__(256) transpose_conv_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                             const float* __restrict__ bias, float* __restrict__ out,
                                                             const TConvGeom g, long long total) {
  const int groups = (g.Cout + 3) >> 2;
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total; t += step) {
    const long long pix = t / groups;
    const int co = static_cast<int>(t - pix * groups) * 4;
    const long long by = pix / g.OW;
    const int ox = static_cast<int>(pix - by * g.OW);
    const long long b = by / g.OH;
    const int oy = static_cast<int>(by - b * g.OH);
    const int nq = min(4, g.Cout - co);
    const int vy = oy + g.ph, vx = ox + g.pw;
    // the input rows / columns whose tap lands in the filter: 0 <= v - i * s < K
    const int ly = vy - g.KH + 1, lx = vx - g.KW + 1;
    const int iy0 = ly <= 0 ? 0 : (ly + g.sh - 1) / g.sh, iy1 = min(vy / g.sh, g.H - 1);
    const int ix0 = lx <= 0 ? 0 : (lx + g.sw - 1) / g.sw, ix1 = min(vx / g.sw, g.W - 1);
    // filter rows of the thread's channels; a channel past Cout reads the last one and is not stored
    const float* wr[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) wr[q] = w + static_cast<long long>(co + min(q, nq - 1)) * g.KH * g.KW * g.Cin;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int iy = iy0; iy <= iy1; ++iy) {
      const int fy = vy - iy * g.sh;
      for (int ix = ix0; ix <= ix1; ++ix) {
        const int fx = vx - ix * g.sw;
        const float* xr = in + ((b * g.H + iy) * g.W + ix) * g.Cin;
        const long long wo = (static_cast<long long>(fy) * g.KW + fx) * g.Cin;
        if (VEC4) {
          for (int ci = 0; ci < g.Cin; ci += 4) {
            const float4 x = __ldg(reinterpret_cast<const float4*>(xr + ci));
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float4 f = __ldg(reinterpret_cast<const float4*>(wr[q] + wo + ci));
              acc[q] = fmaf(x.x, f.x, acc[q]);
              acc[q] = fmaf(x.y, f.y, acc[q]);
              acc[q] = fmaf(x.z, f.z, acc[q]);
              acc[q] = fmaf(x.w, f.w, acc[q]);
            }
          }
        } else {
          for (int ci = 0; ci < g.Cin; ++ci) {
            const float x = __ldg(xr + ci);
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(x, __ldg(wr[q] + wo + ci), acc[q]);
          }
        }
      }
    }
    float* o = out + pix * g.Cout + co;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (q < nq) o[q] = apply_act(bias ? __fadd_rn(acc[q], __ldg(bias + co + q)) : acc[q], g.act);
  }
}

// The sub-pixel tail of a super-resolution network,
//   CONV_2D(x, KHxKW, stride 1, SAME) -> DEPTH_TO_SPACE(r) [-> ADD(RESIZE_BILINEAR(img))],
// in one pass (Graph::FuseSubpixelConvs). A CTA computes BM low-resolution pixels x BN >= Cout conv
// channels as conv_igemm8x8_kernel does: the input patches and filter rows staged KC k at a time, each
// thread 8 pixels x TN channels, and every output the igemm kernels' own chain: acc = 0, fmaf in
// k = (fy * KW + fx) * Cin + ci order with a padded tap as fmaf(0, w, acc), then zero terms up to a
// multiple of kIK, then apply_act(acc + bias). The CTA's tile goes to shared memory, from where the
// pixels' channels n = (i * r + j) * C' + c are stored at their high-resolution addresses
// (b, y * r + i, x * r + j, c): each of the r passes writes runs of r * C' floats, consecutive threads
// consecutive floats. With img, each value is first added to img's bilinear value at that pixel (the
// resize kernel's bilinear_src / bilinear_mix, then the ADD builtin's add and activation). The conv
// output, the shuffled map and the resized image are never written.
struct SubpixelGeom {
  int B, H, W, Cin, KH, KW, ph, pw, Cout, r, Cp;   // Cout = Cp * r * r
  int act, add_act;
  ResizeGeom img;   // img [B, ih, iw, Cp] to (H * r, W * r), when the residual is present
};
constexpr int kSpKC = 8;   // k per staged chunk; kIK (16) is a multiple, so the K padding is igemm's
template <int NCOL, int TN>
struct SubpixelTile {
  static constexpr int kRowThreads = 128 / NCOL, BM = kRowThreads * 8, BN = NCOL * TN;
  static constexpr int kStageFloats = 2 * kSpKC * (BM + 4) + 2 * kSpKC * (BN + 4);
  static constexpr int kOutFloats = BM * (BN + 1);
  static constexpr int kFloats = kStageFloats > kOutFloats ? kStageFloats : kOutFloats;
};
template <int NCOL, int TN>
__global__ void __launch_bounds__(128) subpixel_conv_kernel(const float* __restrict__ in,
                                                            const float* __restrict__ filter,
                                                            const float* __restrict__ bias,
                                                            const float* __restrict__ img,
                                                            float* __restrict__ out, SubpixelGeom g,
                                                            unsigned M) {
  using Tile = SubpixelTile<NCOL, TN>;
  constexpr int BM = Tile::BM, BN = Tile::BN, RPT = BM / 128, TQ = TN / 4;
  extern __shared__ __align__(16) float sp_smem[];
  float (*A_s)[kSpKC][BM + 4] = reinterpret_cast<float (*)[kSpKC][BM + 4]>(sp_smem);
  float (*B_s)[kSpKC][BN + 4] = reinterpret_cast<float (*)[kSpKC][BN + 4]>(sp_smem + 2 * kSpKC * (BM + 4));
  float* out_s = sp_smem;   // [BM][BN + 1], after the K loop
  const int K = g.KH * g.KW * g.Cin;
  const int Kpad = (K + kIK - 1) / kIK * kIK;
  int* koff = reinterpret_cast<int*>(sp_smem + Tile::kFloats);
  int* kdydx = koff + Kpad;
  const int tid = threadIdx.x;
  for (int k = tid; k < Kpad; k += 128) {
    if (k < K) {
      const int tap = k / g.Cin, ci = k - tap * g.Cin;
      const int fy = tap / g.KW, fx = tap - fy * g.KW;
      koff[k] = (fy * g.W + fx) * g.Cin + ci;
      kdydx[k] = (fy << 16) | fx;
    } else {
      koff[k] = 0;
      kdydx[k] = 0x7fff7fff;   // fails every bounds test
    }
  }
  const unsigned m0 = blockIdx.x * static_cast<unsigned>(BM);
  const unsigned hw = static_cast<unsigned>(g.H) * g.W;
  int iy0[RPT], ix0[RPT];
  bool row_ok[RPT];
  const float* base[RPT];
#pragma unroll
  for (int q = 0; q < RPT; ++q) {
    const unsigned m = m0 + tid + 128 * q;
    row_ok[q] = m < M;
    const unsigned mm = row_ok[q] ? m : 0u;
    const unsigned b = mm / hw, rem = mm - b * hw;
    const int y = static_cast<int>(rem / g.W), x = static_cast<int>(rem - (rem / g.W) * g.W);
    iy0[q] = y - g.ph;
    ix0[q] = x - g.pw;
    base[q] = in + ((static_cast<long long>(b) * g.H + iy0[q]) * g.W + ix0[q]) * g.Cin;   // read only in bounds
  }
  __syncthreads();

  float ra[RPT][kSpKC], rb[BN * kSpKC / 128];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int e = 0; e < kSpKC; ++e) {
      const int d = kdydx[k0 + e], o = koff[k0 + e];
#pragma unroll
      for (int q = 0; q < RPT; ++q) {
        const int iy = iy0[q] + (d >> 16), ix = ix0[q] + (d & 0xffff);
        const bool ok = row_ok[q] && static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
                        static_cast<unsigned>(ix) < static_cast<unsigned>(g.W);
        ra[q][e] = ok ? __ldg(base[q] + o) : 0.0f;
      }
    }
#pragma unroll
    for (int e = 0; e < BN * kSpKC / 128; ++e) {
      const int idx = tid + 128 * e, n = idx / kSpKC, k = k0 + idx % kSpKC;
      rb[e] = (n < g.Cout && k < K) ? __ldg(filter + static_cast<size_t>(n) * K + k) : 0.0f;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int q = 0; q < RPT; ++q)
#pragma unroll
      for (int e = 0; e < kSpKC; ++e) A_s[buf][e][tid + 128 * q] = ra[q][e];
#pragma unroll
    for (int e = 0; e < BN * kSpKC / 128; ++e) {
      const int idx = tid + 128 * e;
      B_s[buf][idx % kSpKC][idx / kSpKC] = rb[e];
    }
  };
  const int tx = tid % NCOL, ty = tid / NCOL;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;
  fetch(0);
  stash(0);
  __syncthreads();
  const int nk = Kpad / kSpKC;
  for (int it = 0; it < nk; ++it) {
    const int buf = it & 1;
    if (it + 1 < nk) fetch((it + 1) * kSpKC);
#pragma unroll
    for (int kk = 0; kk < kSpKC; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&A_s[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&A_s[buf][kk][BM / 2 + ty * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[TN];
#pragma unroll
      for (int q = 0; q < TQ; ++q) {
        const float4 b = *reinterpret_cast<const float4*>(&B_s[buf][kk][q * (BN / TQ) + tx * 4]);
        bv[4 * q] = b.x;
        bv[4 * q + 1] = b.y;
        bv[4 * q + 2] = b.z;
        bv[4 * q + 3] = b.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) {
      stash(buf ^ 1);
      __syncthreads();
    }
  }
  __syncthreads();   // out_s reuses the staging memory
  constexpr int SP = BN + 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = i < 4 ? ty * 4 + i : BM / 2 + ty * 4 + (i - 4);
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = (j / 4) * (BN / TQ) + tx * 4 + (j & 3);
      if (n < g.Cout) out_s[row * SP + n] = apply_act(acc[i][j] + (bias ? bias[n] : 0.0f), g.act);
    }
  }
  __syncthreads();
  const int rows = static_cast<int>(min(static_cast<unsigned>(BM), M - m0));
  const int run = g.r * g.Cp;   // floats of one LR pixel in one HR row
  const long long hr_row = static_cast<long long>(g.W) * run;
  for (int i = 0; i < g.r; ++i) {
    for (int e = tid; e < rows * run; e += 128) {
      const int p = e / run, t = e - p * run;
      const unsigned m = m0 + p;
      const unsigned b = m / hw, rem = m - b * hw;
      const int y = static_cast<int>(rem / g.W), x = static_cast<int>(rem - (rem / g.W) * g.W);
      const int Y = y * g.r + i;
      float v = out_s[p * SP + i * run + t];
      if (img) {
        const int jx = t / g.Cp, c = t - jx * g.Cp;
        int y0, y1, x0, x1;
        const float vy = bilinear_src(Y, g.img.y, g.img.half_pixel_centers, &y0, &y1);
        const float vx = bilinear_src(x * g.r + jx, g.img.x, g.img.half_pixel_centers, &x0, &x1);
        const float* src0 = img + (static_cast<long long>(b) * g.img.y.in + y0) * g.img.x.in * g.Cp + c;
        const float* src1 = img + (static_cast<long long>(b) * g.img.y.in + y1) * g.img.x.in * g.Cp + c;
        const float rv = bilinear_mix(__ldg(src0 + x0 * g.Cp), __ldg(src1 + x0 * g.Cp), __ldg(src0 + x1 * g.Cp),
                                      __ldg(src1 + x1 * g.Cp), __fsub_rn(vy, static_cast<float>(y0)),
                                      __fsub_rn(vx, static_cast<float>(x0)));
        v = apply_act(v + rv, g.add_act);
      }
      out[(static_cast<long long>(b) * g.H * g.r + Y) * hr_row + static_cast<long long>(x) * run + t] = v;
    }
  }
}

// LOGISTIC, TFLite's float reference (reference/logistic.h) with CUDA's expf
__global__ void __launch_bounds__(256) logistic_kernel(const float* __restrict__ in,
                                                       float* __restrict__ out, long long n) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const float x = in[i];
    float r;
    if (x > 16.619047164916992188f) r = 1.0f;
    else if (x < -9.0f) r = expf(x);
    else r = 1.0f / (1.0f + expf(-x));
    out[i] = r;
  }
}

// mean over H*W: one thread per (b, c), c fastest => coalesced rows.
__global__ void __launch_bounds__(256) mean_hw_kernel(const float* __restrict__ in,
                                                      float* __restrict__ out, int B, int HW,
                                                      int C, int pre_act) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  const float* p = in + static_cast<size_t>(b) * HW * C + c;
  float s = 0.0f;
  for (int k = 0; k < HW; ++k) s += apply_act(p[static_cast<size_t>(k) * C], pre_act);
  out[i] = s / static_cast<float>(HW);
}

// softmax: one CTA of 128 threads per row (a warp per row left 256 rows on 32 CTAs); the row
// lives in registers between the three passes (<= 8 elements per thread, else re-read).
__global__ void __launch_bounds__(128) softmax_kernel(const float* __restrict__ in,
                                                      float* __restrict__ out, int cols, float beta) {
  __shared__ float red[4];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* x = in + static_cast<long long>(blockIdx.x) * cols;
  float* y = out + static_cast<long long>(blockIdx.x) * cols;
  constexpr int kR = 8;
  const bool in_regs = cols <= kR * 128;
  float v[kR];
  float mx = -FLT_MAX;
  if (in_regs) {
#pragma unroll
    for (int j = 0; j < kR; ++j) {
      const int c = tid + j * 128;
      v[j] = c < cols ? x[c] : -FLT_MAX;
      mx = fmaxf(mx, v[j]);
    }
  } else {
    for (int c = tid; c < cols; c += 128) mx = fmaxf(mx, x[c]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.0f;
  if (in_regs) {
#pragma unroll
    for (int j = 0; j < kR; ++j) {
      const int c = tid + j * 128;
      v[j] = c < cols ? expf((v[j] - mx) * beta) : 0.0f;
      sum += v[j];
    }
  } else {
    for (int c = tid; c < cols; c += 128) sum += expf((x[c] - mx) * beta);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = (red[0] + red[1]) + (red[2] + red[3]);
  if (in_regs) {
#pragma unroll
    for (int j = 0; j < kR; ++j) {
      const int c = tid + j * 128;
      if (c < cols) y[c] = v[j] / sum;
    }
  } else {
    for (int c = tid; c < cols; c += 128) y[c] = expf((x[c] - mx) * beta) / sum;
  }
}

// constant pad of a 4-D tensor of 32-bit elements (float32, or bitpacked int32 words).
struct Pad4 { int in[4], out[4], before[4]; };
__global__ void __launch_bounds__(256) pad4d32_kernel(const uint32_t* __restrict__ in,
                                                      uint32_t* __restrict__ out, Pad4 p,
                                                      uint32_t fill, long long total) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  long long r = i;
  const int d3 = static_cast<int>(r % p.out[3]); r /= p.out[3];
  const int d2 = static_cast<int>(r % p.out[2]); r /= p.out[2];
  const int d1 = static_cast<int>(r % p.out[1]); r /= p.out[1];
  const int d0 = static_cast<int>(r);
  const int s0 = d0 - p.before[0], s1 = d1 - p.before[1], s2 = d2 - p.before[2],
            s3 = d3 - p.before[3];
  uint32_t v = fill;
  if (static_cast<unsigned>(s0) < static_cast<unsigned>(p.in[0]) &&
      static_cast<unsigned>(s1) < static_cast<unsigned>(p.in[1]) &&
      static_cast<unsigned>(s2) < static_cast<unsigned>(p.in[2]) &&
      static_cast<unsigned>(s3) < static_cast<unsigned>(p.in[3]))
    v = in[((static_cast<long long>(s0) * p.in[1] + s1) * p.in[2] + s2) * p.in[3] + s3];
  out[i] = v;
}

// ---- fused stem: [DEQUANTIZE ->] CONV_2D(3x3, stride 2, 3 -> C1) -> DEPTHWISE_CONV_2D(3x3,
// stride 2) in one pass, C1 = 16 (QuickNet, QuickNetLarge) or 8 (QuickNetSmall). Unfused, the
// dequantised image (154 MB at batch 256) and the first conv's map (205 MB at C1 = 16, 103 MB at 8)
// each make a round trip through HBM; fused, a step reads the int8 image and writes the depthwise
// map. The text below counts C1 = 16; at C1 = 8 each first-conv pixel is two 16-byte cells.
//   Persistent CTAs (one per SM, 512 threads). A tile = 4 output rows x <= 56 output columns of
// one image. Its 19 x 227 x 3 input patch is fetched as raw bytes (cp.async, double-buffered: the
// next tile's patch arrives while this one computes), padded in the QUANTISED domain (zero point;
// 0.0f for a float image); the 9 x 113 x 16 first-conv strip stays in shared memory. For byte
// images the CTA is two independent groups of 256 threads, each with its own tiles, patch buffers,
// strip and named barrier, so that one group's latency-bound phases (patch wait, depthwise stage,
// barriers) are covered by the other's FMA stage (142 -> 124 us at batch 256).
//   Stage 1: thread = 2 adjacent first-conv pixels x 16 channels. Per patch row it reads 15 input
// values (int8: 4 x LDS.32, then a 256-entry table of float(scale * (q - zero_point)) -- exactly
// DEQUANTIZE's values -- replicated per bank, so a lookup never conflicts) and issues 3 x 3 x 16
// FMAs: two channels per step, the input value broadcast, the weight pair a constant-bank
// operand (the filters travel by value in the parameter bank); operands staged in shared memory
// would be bound by the LDS pipe instead.
//   Stage 2: thread = (output column, 4 channels, row pair); out-of-range taps are skipped.
// Every output is accumulated in the order of conv_direct16_kernel / depthwise_v4_kernel with the
// same IEEE fma, so the result is bit-identical to the separate kernels.
// two IEEE fmas, one per channel of the pair
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
constexpr int kS2R = 4, kS2TW = 56;
constexpr int kS2R1 = 2 * kS2R + 1;            // 9 first-conv rows per tile
constexpr int kS2C1 = 2 * kS2TW + 1;           // 113 first-conv columns
constexpr int kS2R0 = 2 * kS2R1 + 1;           // 19 input rows
constexpr int kS2C0 = 2 * kS2C1 + 1;           // 227 input columns
constexpr int kS2RawCols = 240;                // fetched per row: 15 x 16 columns
constexpr int kS2Threads = 512;
struct Stem2Geom {
  int B, H, W, OH1, OW1, ph1, pw1, OH2, OW2, ph2, pw2, act1, act2;
  int n_rt, n_ct;        // row / column tiles per image
  int aligned;           // rows can be fetched with 16-byte cp.async
  int in_zero_point;
  double in_scale;
};
template <int C1>
struct StemWeights {
  float w1[27][C1];   // [tap * 3 + ci][co]
  float b1[C1];
  float w2[9][C1];    // [tap][c]
  float b2[C1];
};
template <typename TIn, int C1>
struct Stem2Layout {
  static constexpr int kRawPitch = kS2RawCols * 3 * static_cast<int>(sizeof(TIn));          // 720 / 2880 B
  static constexpr int kLutBytes = sizeof(TIn) == 1 ? 256 * 32 * 4 : 0;
  // byte images: the CTA runs TWO independent groups of 256 threads, each on its own tile with its own
  // patch buffers and strip and its own named barrier -- while one group sits in the latency-bound
  // phases (patch wait, depthwise stage, barriers) the other keeps the FMA pipe busy. Float images
  // need 4x the patch memory: one group of 512 threads.
  static constexpr int kGroups = sizeof(TIn) == 1 ? 2 : 1;
  static constexpr int kC1Bufs = 1;
  static constexpr size_t kGroupRawBytes = 2 * static_cast<size_t>(kS2R0) * kRawPitch + 64;
  static constexpr size_t kSmemBytes = kGroups * (kGroupRawBytes + kC1Bufs * kS2R1 * kS2C1 * C1 * 4) + (9 * C1 + C1) * 4 + kLutBytes;
};

template <typename TIn, bool kUnsigned, int C1>
__global__ void __launch_bounds__(kS2Threads, 1)
stem_conv_dw_kernel(const TIn* __restrict__ in, float* __restrict__ out, const __grid_constant__ StemWeights<C1> Wt,
                    const Stem2Geom s) {
  static_assert(C1 == 8 || C1 == 16, "the fused stem takes 8 or 16 first-conv channels");
  extern __shared__ __align__(16) unsigned char sm_raw[];
  using Lay = Stem2Layout<TIn, C1>;
  constexpr int kRawPitch = Lay::kRawPitch;
  constexpr bool kQuant = sizeof(TIn) == 1;
  constexpr int kGroups = Lay::kGroups, kG = kS2Threads / kGroups;                // threads per group
  constexpr int kC1Bufs = Lay::kC1Bufs;
  constexpr int kC1Floats = kS2R1 * kS2C1 * C1;
  constexpr int kQ = C1 / 4;                                                      // 16-byte cells per pixel
  const int gid = threadIdx.x / kG, tid = threadIdx.x - gid * kG, lane = threadIdx.x & 31;   // tid: inside the group
  unsigned char* raw0 = sm_raw + gid * Lay::kGroupRawBytes;                       // [2][19][kRawPitch] (+ slack)
  float* c1_all = reinterpret_cast<float*>(sm_raw + kGroups * Lay::kGroupRawBytes);
  float* c1_0 = c1_all + gid * kC1Bufs * kC1Floats;                               // [kC1Bufs][9][113][C1], swizzled
  float* w2s = c1_all + kGroups * kC1Bufs * kC1Floats;                            // [9][C1]
  float* b2s = w2s + 9 * C1;
  float* lut = b2s + C1;                                                          // [256][32]
  auto group_barrier = [&]() {
    if (kGroups == 1) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"r"(1 + gid), "r"(kG) : "memory");
  };

  for (int i = threadIdx.x; i < 9 * C1; i += kS2Threads) w2s[i] = Wt.w2[i / C1][i % C1];
  if (threadIdx.x < C1) b2s[threadIdx.x] = Wt.b2[threadIdx.x];
  if (kQuant) {
    for (int i = threadIdx.x; i < 256 * 32; i += kS2Threads) {
      const int byte = i >> 5;
      const int q = kUnsigned ? byte : (byte < 128 ? byte : byte - 256);
      lut[i] = static_cast<float>(s.in_scale * static_cast<double>(q - s.in_zero_point));
    }
  }
  const TIn pad_value = kQuant ? static_cast<TIn>(s.in_zero_point) : static_cast<TIn>(0);

  const int tiles = s.B * s.n_rt * s.n_ct;
  struct Tile { int b, rt, ct, oy2_0, ox2_0, tw, y1_0, x1_0, y0_0, x0_0; };
  auto place = [&](Tile& T) {
    T.oy2_0 = T.rt * kS2R;
    T.ox2_0 = T.ct * kS2TW;
    T.tw = min(kS2TW, s.OW2 - T.ox2_0);
    T.y1_0 = T.oy2_0 * 2 - s.ph2; T.x1_0 = T.ox2_0 * 2 - s.pw2;
    T.y0_0 = T.y1_0 * 2 - s.ph1;  T.x0_0 = T.x1_0 * 2 - s.pw1;
  };
  // tile index -> (image, row tile, column tile) once; then a step of (groups in the grid) tiles by carries
  const int tile_step = static_cast<int>(gridDim.x) * kGroups;
  const int step_ct = tile_step % s.n_ct, step_r = tile_step / s.n_ct;
  const int step_rt = step_r % s.n_rt, step_b = step_r / s.n_rt;
  auto advance = [&](Tile& T) {
    T.ct += step_ct;
    if (T.ct >= s.n_ct) { T.ct -= s.n_ct; T.rt += 1; }
    T.rt += step_rt;
    if (T.rt >= s.n_rt) { T.rt -= s.n_rt; T.b += 1; }
    T.b += step_b;
    place(T);
  };
  // raw[r][j * 3 + ci] = input(y0_0 + r, x0_0 + j, ci) for j < 227, the pad value outside the image
  auto load_tile = [&](const Tile& T, unsigned char* raw) {
    const TIn* img = in + static_cast<long long>(T.b) * s.H * s.W * 3;
    if (s.aligned && T.x0_0 >= 0 && (T.x0_0 & 15) == 0) {
      const int xr1 = min(s.W, T.x0_0 + kS2RawCols);
      const int row_elems = (xr1 - T.x0_0) * 3;
      const int n16 = (row_elems * static_cast<int>(sizeof(TIn))) >> 4;      // whole chunks: see `aligned`
      for (int i = tid; i < kS2R0 * n16; i += kG) {
        const int r = i / n16, c = i - r * n16;
        const int y = T.y0_0 + r;
        if (static_cast<unsigned>(y) >= static_cast<unsigned>(s.H)) continue;
        const unsigned char* src = reinterpret_cast<const unsigned char*>(img + (static_cast<long long>(y) * s.W + T.x0_0) * 3) + c * 16;
        const uint32_t dst = static_cast<uint32_t>(__cvta_generic_to_shared(raw + r * kRawPitch + c * 16));
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
      }
      // rows above / below the image, and the columns right of it (bytes no chunk writes)
      const int tail = kS2C0 * 3 - row_elems;
      for (int r = 0; r < kS2R0; ++r) {
        TIn* rr = reinterpret_cast<TIn*>(raw + r * kRawPitch);
        if (static_cast<unsigned>(T.y0_0 + r) >= static_cast<unsigned>(s.H)) {
          for (int e = tid; e < kS2C0 * 3; e += kG) rr[e] = pad_value;
        } else if (tid < tail) {
          rr[row_elems + tid] = pad_value;
        }
      }
    } else {
      for (int i = tid; i < kS2R0 * kS2C0; i += kG) {
        const int r = i / kS2C0, j = i - r * kS2C0;
        const int y = T.y0_0 + r, x = T.x0_0 + j;
        TIn* dst = reinterpret_cast<TIn*>(raw + r * kRawPitch) + j * 3;
        if (static_cast<unsigned>(y) < static_cast<unsigned>(s.H) && static_cast<unsigned>(x) < static_cast<unsigned>(s.W)) {
          const TIn* src = img + (static_cast<long long>(y) * s.W + x) * 3;
          dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
        } else {
          dst[0] = pad_value; dst[1] = pad_value; dst[2] = pad_value;
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  // ---- stage 1: first conv on the strip rows / columns that lie inside its map
  auto stage1 = [&](const Tile& T, const unsigned char* raw, float* c1) {
    const int l1_lo = max(0, -T.y1_0), l1_hi = min(kS2R1, s.OH1 - T.y1_0);
    const int cl_lo = max(0, -T.x1_0) & ~1, cl_hi = min(2 * T.tw + 1, s.OW1 - T.x1_0);
    if (l1_hi <= l1_lo || cl_hi <= cl_lo) return;
    const int tpr = (cl_hi - cl_lo + 1) >> 1;
    const int tasks = (l1_hi - l1_lo) * tpr;
    for (int task = tid; task < tasks; task += kG) {
      const int rr = task / tpr, tt = task - rr * tpr;
      const int l1 = l1_lo + rr, cg = cl_lo + 2 * tt;
      float2 acc[2][C1 / 2];
#pragma unroll
      for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int c = 0; c < C1 / 2; ++c) acc[p][c] = make_float2(0.0f, 0.0f);
      const unsigned char* row0 = raw + (2 * l1) * kRawPitch + 6 * cg * static_cast<int>(sizeof(TIn));
      // byte images: all 12 words of the three patch rows are requested before the first lookup
      uint32_t rw[3][4];
      if (kQuant) {
#pragma unroll
        for (int fy = 0; fy < 3; ++fy)
#pragma unroll
          for (int k = 0; k < 4; ++k) rw[fy][k] = reinterpret_cast<const uint32_t*>(row0 + fy * kRawPitch)[k];
      }
#pragma unroll
      for (int fy = 0; fy < 3; ++fy) {
        float xv[16];
        if (kQuant) {
          // 15 bytes from a 4-byte aligned start (cg is even), then table[byte][lane]
          const float* lt = lut + lane;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint32_t w = rw[fy][k];
            xv[4 * k] = lt[__byte_perm(w, 0, 0x4440) << 5];
            xv[4 * k + 1] = lt[__byte_perm(w, 0, 0x4441) << 5];
            xv[4 * k + 2] = lt[__byte_perm(w, 0, 0x4442) << 5];
            if (k < 3) xv[4 * k + 3] = lt[__byte_perm(w, 0, 0x4443) << 5];
          }
        } else {
          const float4* xr = reinterpret_cast<const float4*>(row0 + fy * kRawPitch);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float4 f = xr[k];
            xv[4 * k] = f.x; xv[4 * k + 1] = f.y; xv[4 * k + 2] = f.z; xv[4 * k + 3] = f.w;
          }
        }
#pragma unroll
        for (int fx = 0; fx < 3; ++fx)
#pragma unroll
          for (int ci = 0; ci < 3; ++ci) {
            const int kk = (fy * 3 + fx) * 3 + ci;
#pragma unroll
            for (int c = 0; c < C1 / 2; ++c) {
              const float2 w = make_float2(Wt.w1[kk][2 * c], Wt.w1[kk][2 * c + 1]);
#pragma unroll
              for (int p = 0; p < 2; ++p) {
                const float x = xv[(2 * p + fx) * 3 + ci];
                acc[p][c] = fma2_rn(make_float2(x, x), w, acc[p][c]);
              }
            }
          }
      }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int cl = cg + p;
        if (cl >= cl_hi) continue;
        float* dst = c1 + (l1 * kS2C1 + cl) * C1;
        const int sw = (cl >> 1) & (kQ - 1);   // 16-byte cell swizzle: neighbouring tasks hit different banks
#pragma unroll
        for (int q = 0; q < kQ; ++q)
          *reinterpret_cast<float4*>(dst + ((q ^ sw) << 2)) =
              make_float4(apply_act(acc[p][2 * q].x + Wt.b1[4 * q], s.act1), apply_act(acc[p][2 * q].y + Wt.b1[4 * q + 1], s.act1),
                          apply_act(acc[p][2 * q + 1].x + Wt.b1[4 * q + 2], s.act1),
                          apply_act(acc[p][2 * q + 1].y + Wt.b1[4 * q + 3], s.act1));
      }
    }
  };
  // ---- stage 2: depthwise 3x3 stride 2. Thread = (output column, 4 channels, row pair): the
  // column offsets, their validity and the 9 weight vectors are per-thread constants;
  // out-of-range taps are skipped like depthwise_v4_kernel skips them.
  auto stage2 = [&](const Tile& T, const float* c1) {
    const int n2 = T.tw * kQ;
    for (int task = tid; task < 2 * n2; task += kG) {
    const int half = task >= n2 ? 1 : 0;
    const int r2 = task - half * n2;
    const int lx = r2 / kQ, q = r2 % kQ;
    int off[3];
    bool cok[3];
#pragma unroll
    for (int fx = 0; fx < 3; ++fx) {
      const int cl = 2 * lx + fx;
      cok[fx] = static_cast<unsigned>(T.x1_0 + cl) < static_cast<unsigned>(s.OW1);
      off[fx] = cl * C1 + ((q ^ ((cl >> 1) & (kQ - 1))) << 2);
    }
    float4 wv[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wv[k] = *reinterpret_cast<const float4*>(w2s + k * C1 + q * 4);
    const float4 bb = *reinterpret_cast<const float4*>(b2s + q * 4);
    float4* o = reinterpret_cast<float4*>(out) +
                ((static_cast<long long>(T.b) * s.OH2 + T.oy2_0) * s.OW2 + T.ox2_0 + lx) * kQ + q;
    for (int ly = 2 * half; ly < 2 * half + 2 && T.oy2_0 + ly < s.OH2; ++ly) {
      float2 a0 = make_float2(0.f, 0.f), a1 = make_float2(0.f, 0.f);
#pragma unroll
      for (int fy = 0; fy < 3; ++fy) {
        const int l1 = 2 * ly + fy;
        if (static_cast<unsigned>(T.y1_0 + l1) >= static_cast<unsigned>(s.OH1)) continue;
        const float* rowp = c1 + l1 * (kS2C1 * C1);
#pragma unroll
        for (int fx = 0; fx < 3; ++fx) {
          if (!cok[fx]) continue;
          const float4 x = *reinterpret_cast<const float4*>(rowp + off[fx]);
          const float4 w = wv[fy * 3 + fx];
          a0 = fma2_rn(make_float2(x.x, x.y), make_float2(w.x, w.y), a0);
          a1 = fma2_rn(make_float2(x.z, x.w), make_float2(w.z, w.w), a1);
        }
      }
      o[static_cast<long long>(ly) * s.OW2 * kQ] =
          make_float4(apply_act(a0.x + bb.x, s.act2), apply_act(a0.y + bb.y, s.act2),
                      apply_act(a1.x + bb.z, s.act2), apply_act(a1.y + bb.w, s.act2));
    }
    }
  };

  // Pipeline over this group's tiles (one strip):
  //   iteration i:  [barrier: patch i landed, strip free] fetch patch i+1 (async) | stage 1 of tile i |
  //                 [barrier] | stage 2 of tile i
  __syncthreads();                       // the table, depthwise weights (written by all 512 threads)
  int t = blockIdx.x * kGroups + gid;
  if (t >= tiles) return;
  Tile cur;
  cur.ct = t % s.n_ct;
  cur.rt = (t / s.n_ct) % s.n_rt;
  cur.b = t / (s.n_ct * s.n_rt);
  place(cur);
  load_tile(cur, raw0);
  for (int i = 0; t < tiles; t += tile_step, ++i) {
    unsigned char* raw = raw0 + (i & 1) * (kS2R0 * kRawPitch);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    group_barrier();   // patch i complete for every thread; stage 2 of tile i-1 is done with the strip
    Tile nxt = cur;
    advance(nxt);
    if (t + tile_step < tiles) load_tile(nxt, raw0 + ((i + 1) & 1) * (kS2R0 * kRawPitch));
    stage1(cur, raw, c1_0);
    group_barrier();   // strip complete
    stage2(cur, c1_0);
    cur = nxt;
  }
}

template <typename TIn, bool kUnsigned, int C1>
int launch_stem2(const void* in, const StemWeights<C1>& wt, float* out, const Stem2Geom& s, void* stream) {
  static bool attr_dev[64] = {};   // the attribute is per device
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  constexpr size_t smem = Stem2Layout<TIn, C1>::kSmemBytes;
  if (!(dev >= 0 && dev < 64 && attr_dev[dev])) {
    if (cudaFuncSetAttribute(stem_conv_dw_kernel<TIn, kUnsigned, C1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem)) != cudaSuccess)
      return fail("stem_conv_dw: cannot raise the shared-memory limit");
    if (dev >= 0 && dev < 64) attr_dev[dev] = true;
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long tiles = static_cast<long long>(s.B) * s.n_rt * s.n_ct;
  if (tiles > (1LL << 29)) return fail("stem_conv_dw: too many tiles");
  constexpr int groups = Stem2Layout<TIn, C1>::kGroups;
  const unsigned grid = static_cast<unsigned>(std::min<long long>((tiles + groups - 1) / groups, sms));
  stem_conv_dw_kernel<TIn, kUnsigned, C1><<<grid, kS2Threads, smem, as_stream(stream)>>>(static_cast<const TIn*>(in), out, wt, s);
  return launch_check("stem_conv_dw_kernel");
}

// The filters in the kernel's order, then the launch for the image's element type.
template <int C1>
int stem2_run(int in_type, const void* in, const float* w1, const float* b1, const float* w2, const float* b2,
              float* out, const Stem2Geom& s, void* stream) {
  StemWeights<C1> wt;
  for (int k = 0; k < 27; ++k)
    for (int c = 0; c < C1; ++c) wt.w1[k][c] = w1[c * 27 + k];   // OHWI [C1][3][3][3] -> [k][co]
  for (int i = 0; i < 9 * C1; ++i) wt.w2[i / C1][i % C1] = w2[i];
  for (int c = 0; c < C1; ++c) {
    wt.b1[c] = b1 ? b1[c] : 0.0f;
    wt.b2[c] = b2 ? b2[c] : 0.0f;
  }
  if (in_type == LCE_T_FLOAT) return launch_stem2<float, false, C1>(in, wt, out, s, stream);
  if (in_type == LCE_T_INT8) return launch_stem2<int8_t, false, C1>(in, wt, out, s, stream);
  return launch_stem2<uint8_t, true, C1>(in, wt, out, s, stream);
}

int make_geom(const lce_f32_conv_desc* d, ConvGeom* g) {
  if (d->batch < 0 || d->in_h < 1 || d->in_w < 1 || d->in_c < 1 || d->out_c < 1 ||
      d->filter_h < 1 || d->filter_w < 1 || d->stride_h < 1 || d->stride_w < 1 ||
      d->dilation_h < 1 || d->dilation_w < 1)
    return fail("f32 conv: bad parameters");
  g->B = d->batch; g->H = d->in_h; g->W = d->in_w; g->Cin = d->in_c;
  g->KH = d->filter_h; g->KW = d->filter_w; g->Cout = d->out_c;
  g->sh = d->stride_h; g->sw = d->stride_w; g->dh = d->dilation_h; g->dw = d->dilation_w;
  g->OH = out_size(d->padding, d->in_h, d->filter_h, d->stride_h, d->dilation_h);
  g->OW = out_size(d->padding, d->in_w, d->filter_w, d->stride_w, d->dilation_w);
  g->ph = pad_before(d->stride_h, d->dilation_h, d->in_h, d->filter_h, g->OH);
  g->pw = pad_before(d->stride_w, d->dilation_w, d->in_w, d->filter_w, g->OW);
  g->act = d->activation;
  if (g->OH < 0) g->OH = 0;
  if (g->OW < 0) g->OW = 0;
  return 0;
}

// ---- grouped convolution (lce_b200_f32_grouped_conv2d): filter [Cout, KH, KW, Cin / G] ----
// Output channel o reads input channels [(o / (Cout / G)) * Cin / G, ...). Each output is the chain
// the other FMA convolution kernels run over its group's channels: acc = 0, fmaf over (fy, fx, ci)
// in that order, padded taps as fmaf(0, w, acc); then the bias once if present, the activation, and
// the optional BatchNorm behind it in the MUL and ADD builtins' roundings.
struct GroupedEpilogue {
  const float* bias;    // may be null
  const float* scale;   // may be null (no MUL)
  const float* shift;   // may be null (no ADD)
  int act, post_act;
};

__device__ __forceinline__ float grouped_epilogue(float acc, int o, const GroupedEpilogue& e) {
  float y = e.bias ? __fadd_rn(acc, __ldg(e.bias + o)) : acc;
  y = apply_act(y, e.act);
  if (e.scale) y = __fmul_rn(y, __ldg(e.scale + o));
  if (e.shift) y = __fadd_rn(y, __ldg(e.shift + o));
  return apply_act(y, e.post_act);
}

// Any shape: one thread per output element, operands straight from global memory.
__global__ void __launch_bounds__(256) grouped_conv_any_kernel(const float* __restrict__ in,
                                                               const float* __restrict__ filter,
                                                               float* __restrict__ out, ConvGeom g, int cin_g,
                                                               int cout_g, GroupedEpilogue e, long long n) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const int o = static_cast<int>(i % g.Cout);
    long long r = i / g.Cout;
    const int ox = static_cast<int>(r % g.OW);
    r /= g.OW;
    const int oy = static_cast<int>(r % g.OH);
    const long long b = r / g.OH;
    const float* wp = filter + static_cast<long long>(o) * g.KH * g.KW * cin_g;
    const int c0 = (o / cout_g) * cin_g;
    float acc = 0.0f;
    for (int fy = 0; fy < g.KH; ++fy) {
      const int iy = oy * g.sh - g.ph + fy * g.dh;
      for (int fx = 0; fx < g.KW; ++fx) {
        const int ix = ox * g.sw - g.pw + fx * g.dw;
        const bool inside = static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) &&
                            static_cast<unsigned>(ix) < static_cast<unsigned>(g.W);
        const float* src = in + ((b * g.H + (inside ? iy : 0)) * g.W + (inside ? ix : 0)) * g.Cin + c0;
        for (int ci = 0; ci < cin_g; ++ci) acc = fmaf(inside ? __ldg(src + ci) : 0.0f, __ldg(wp++), acc);
      }
    }
    out[i] = grouped_epilogue(acc, o, e);
  }
}

// 3x3, stride 1, dilation 1, CG -> OG channels in each of G groups (MeliusNet's stem: 8 -> 8 in 4
// groups, 4 -> 8 in 8). A block takes a 16 x 8 pixel tile of one image: the tile and its halo for all
// channels, and every group's weights, are staged in shared memory once. A warp takes two rows of
// the tile and one group, so its weight reads are one broadcast address; each lane owns one pixel and
// the group's OG outputs and stores them as float4. Input pixels sit CIN + 4 floats apart, so the
// float4 reads of eight consecutive lanes hit distinct banks. Padded taps read zeros from the tile.
constexpr int kGTW = 16, kGTH = 8;
template <int CG, int OG, int G>
__global__ void __launch_bounds__(256) grouped_conv3x3_kernel(const float* __restrict__ in,
                                                              const float* __restrict__ filter,
                                                              float* __restrict__ out, ConvGeom g,
                                                              GroupedEpilogue e) {
  constexpr int CIN = CG * G, COUT = OG * G, PS = CIN + 4, Q = OG / 4;
  constexpr int HW = kGTW + 2, HH = kGTH + 2;
  static_assert(CG % 4 == 0 && OG % 4 == 0, "whole float4s per group");
  __shared__ __align__(16) float x_s[HH * HW * PS];
  __shared__ __align__(16) float w_s[9 * CG * OG * G];   // [tap][ci][q][g][4]
  const int b = blockIdx.z;
  const int oy0 = blockIdx.y * kGTH, ox0 = blockIdx.x * kGTW;
  for (int i = threadIdx.x; i < 9 * CG * COUT; i += blockDim.x) {
    const int o = i / (9 * CG), rem = i - o * (9 * CG);
    const int gi = o / OG, oo = o - gi * OG;
    w_s[((rem * Q + (oo >> 2)) * G + gi) * 4 + (oo & 3)] = __ldg(filter + i);
  }
  const long long img = static_cast<long long>(b) * g.H * g.W;
  for (int i = threadIdx.x; i < HH * HW * (CIN / 4); i += blockDim.x) {
    const int p = i / (CIN / 4), c4 = i - p * (CIN / 4);
    const int py = p / HW, px = p - py * HW;
    const int iy = oy0 - g.ph + py, ix = ox0 - g.pw + px;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (static_cast<unsigned>(iy) < static_cast<unsigned>(g.H) && static_cast<unsigned>(ix) < static_cast<unsigned>(g.W))
      v = __ldg(reinterpret_cast<const float4*>(in + (img + static_cast<long long>(iy) * g.W + ix) * CIN) + c4);
    *reinterpret_cast<float4*>(x_s + p * PS + c4 * 4) = v;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col = lane & (kGTW - 1);
  // (row pair, group) tasks: kGTH / 2 * G of them over the block's 8 warps
  for (int task = warp; task < (kGTH / 2) * G; task += 8) {
    const int gi = task % G, row = (task / G) * 2 + (lane >> 4);
    float acc[OG];
#pragma unroll
    for (int k = 0; k < OG; ++k) acc[k] = 0.0f;
#pragma unroll
    for (int fy = 0; fy < 3; ++fy)
#pragma unroll
      for (int fx = 0; fx < 3; ++fx) {
        const float* xp = x_s + ((row + fy) * HW + col + fx) * PS + gi * CG;
#pragma unroll
        for (int c4 = 0; c4 < CG / 4; ++c4) {
          const float4 v = *reinterpret_cast<const float4*>(xp + c4 * 4);
          const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float4* wq =
                reinterpret_cast<const float4*>(w_s + (((fy * 3 + fx) * CG + c4 * 4 + k) * Q * G + gi) * 4);
#pragma unroll
            for (int q = 0; q < Q; ++q) {
              const float4 w = wq[q * G];
              acc[4 * q] = fmaf(xv[k], w.x, acc[4 * q]);
              acc[4 * q + 1] = fmaf(xv[k], w.y, acc[4 * q + 1]);
              acc[4 * q + 2] = fmaf(xv[k], w.z, acc[4 * q + 2]);
              acc[4 * q + 3] = fmaf(xv[k], w.w, acc[4 * q + 3]);
            }
          }
        }
      }
    const int oy = oy0 + row, ox = ox0 + col;
    if (oy < g.OH && ox < g.OW) {
      float4* o4 = reinterpret_cast<float4*>(out + ((static_cast<long long>(b) * g.OH + oy) * g.OW + ox) * COUT +
                                             gi * OG);
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const int o = gi * OG + 4 * q;
        o4[q] = make_float4(grouped_epilogue(acc[4 * q], o, e), grouped_epilogue(acc[4 * q + 1], o + 1, e),
                            grouped_epilogue(acc[4 * q + 2], o + 2, e), grouped_epilogue(acc[4 * q + 3], o + 3, e));
      }
    }
  }
}

}  // namespace

// DEQUANTIZE (TF/lite/kernels/internal/reference/dequantize.h:32-49): out = float(scale * (q - zp)),
// the product in double as there. 16 quantised values (one 128-bit load) per thread.
template <typename Q>
__global__ void __launch_bounds__(256) dequantize_affine_kernel(const Q* __restrict__ in, float* __restrict__ out,
                                                                long long n, double scale, int zp) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long n16 = n / 16;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n16; i += stride) {
    const uint4 v = __ldcs(reinterpret_cast<const uint4*>(in) + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float4* o = reinterpret_cast<float4*>(out) + i * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float r[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const Q q = static_cast<Q>((w[j] >> (8 * k)) & 0xFFu);
        r[k] = static_cast<float>(scale * static_cast<double>(static_cast<int>(q) - zp));
      }
      o[j] = make_float4(r[0], r[1], r[2], r[3]);
    }
  }
  for (long long i = n16 * 16 + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride)
    out[i] = static_cast<float>(scale * static_cast<double>(static_cast<int>(in[i]) - zp));
}


extern "C" {

int lce_b200_f32_conv_out_shape(const lce_f32_conv_desc* d, int* out_h, int* out_w) {
  ConvGeom g;
  if (make_geom(d, &g)) return 1;
  *out_h = g.OH;
  *out_w = g.OW;
  return 0;
}

// Whether conv2d_impl computes a convolution's floats on the same kernel with and without the
// signs of its output (Graph::FuseConvQuantize asks before it rewrites the graph, so that
// CONV_2D+LceQuantize equals CONV_2D then LceQuantize bit for bit). The tensor-core pointwise
// kernel packs whole 128-column tiles only: a 1x1 stride-1 convolution it takes without the signs
// (K a multiple of 32) but of another width, such as QuickNetSmall's 32 -> 64 transition, would
// run on another kernel with them.
int lce_b200_internal_conv_packs_alike(int filter_h, int filter_w, int stride_h, int stride_w,
                                       int in_c, int out_c) {
  const bool pw = filter_h == 1 && filter_w == 1 && stride_h == 1 && stride_w == 1 &&
                  in_c % 32 == 0 && in_c <= 4096;
  return !(pw && out_c % 32 == 0 && out_c % 128 != 0);
}

// The direct kernel's K threshold; LCE_B200_DIRECT_MAXK overrides it for experiments.
static int direct_max_k() {
  static const int k = [] {
    const char* e = getenv("LCE_B200_DIRECT_MAXK");
    return e ? atoi(e) : kDirectMaxK;
  }();
  return k;
}

// Whether conv2d_impl runs an ungrouped convolution of this geometry on the implicit-GEMM kernels
// (conv_igemm8x8_kernel, or conv_igemm_kernel under LCE_B200_IGEMM_8X4: the same chain per output)
// whatever its batch and wherever its tensors sit. conv2d_impl takes that path first for such a
// convolution, and Graph::FuseSubpixelConvs asks here before it replaces one by a kernel that
// repeats the igemm kernels' chain, so the two cannot disagree. Never: 1x1 stride-1 convolutions
// (tf32 pointwise and GEMM kernels), the 7x7 stride-2 3 -> 64 stem, K up to the direct kernel's
// threshold. A convolution refused here may still reach the igemm kernels as a fallback.
int lce_b200_internal_conv_runs_igemm(int in_h, int in_w, int in_c, int filter_h, int filter_w, int stride_h,
                                      int stride_w, int dilation_h, int dilation_w, int out_c) {
  if (filter_h == 1 && filter_w == 1 && stride_h == 1 && stride_w == 1) return 0;
  if (filter_h == 7 && filter_w == 7 && in_c == 3 && out_c == 64 && stride_h == 2 && stride_w == 2 &&
      dilation_h == 1 && dilation_w == 1)
    return 0;
  const long long K = static_cast<long long>(filter_h) * filter_w * in_c;
  if (K <= direct_max_k()) return 0;
  return K <= kIKMax && static_cast<long long>(in_h) * in_w * in_c < (1LL << 31);
}

static int igemm_conv(const ConvGeom& g, long long M, const float* in, const float* filter, const float* bias,
                      float* out, void* stream) {
  const int K = g.KH * g.KW * g.Cin;
  dim3 igrid(static_cast<unsigned>((M + kIM - 1) / kIM), (g.Cout + kIN - 1) / kIN);
  const size_t ksmem = static_cast<size_t>((K + kIK - 1) / kIK * kIK) * 2 * sizeof(int);
  static const bool use8x4 = [] {
    const char* e = getenv("LCE_B200_IGEMM_8X4");
    return e && e[0] == '1';
  }();
  // with the kernels' static tiles, the offset table of a K above about 3000 (DoReFaNet's 3x3x384
  // layers as float convolutions) passes the 48 KB a launch gets without opting in
  {
    static bool attr[64] = {};   // the attribute is per device
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr[dev]) {
      const int most = kIKMax * 2 * static_cast<int>(sizeof(int));
      cudaFuncSetAttribute(conv_igemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
      cudaFuncSetAttribute(conv_igemm8x8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
      if (dev >= 0 && dev < 64) attr[dev] = true;
    }
  }
  if (use8x4) {
    conv_igemm_kernel<<<igrid, 256, ksmem, as_stream(stream)>>>(in, filter, bias, out, g, M);
    return launch_check("conv_igemm_kernel");
  }
  conv_igemm8x8_kernel<<<igrid, 128, ksmem, as_stream(stream)>>>(in, filter, bias, out, g, M);
  return launch_check("conv_igemm8x8_kernel");
}

// `packed` (optional): LceQuantize of the output. Kernels that can emit it in their epilogue do
// and set *packed_done; the caller packs with the stand-alone kernel otherwise.
static int conv2d_impl(const lce_f32_conv_desc* d, const float* in, const float* filter,
                       const float* bias, float* out, int32_t* packed, bool* packed_done,
                       void* stream) {
  ConvGeom g;
  if (make_geom(d, &g)) return 1;
  const long long M = static_cast<long long>(g.B) * g.OH * g.OW;
  if (M == 0) return 0;
  const int K = g.KH * g.KW * g.Cin;
  if (lce_b200_internal_conv_runs_igemm(g.H, g.W, g.Cin, g.KH, g.KW, g.sh, g.sw, g.dh, g.dw, g.Cout))
    return igemm_conv(g, M, in, filter, bias, out, stream);
  // 1x1 stride-1 convolutions are plain GEMMs over the pixels: tensor cores first
  if (g.KH == 1 && g.KW == 1 && g.sh == 1 && g.sw == 1) {
    int32_t* pk = (packed && (g.Cout & 31) == 0) ? packed : nullptr;
    const int rc = lce_b200_internal::pw_tf32_conv(in, filter, bias, out, pk, M, g.Cout, K, g.act,
                                                   ((static_cast<long long>(g.OH) * g.OW) & 1) == 0, stream);
    if (rc >= 0) {
      if (rc == 0 && pk) *packed_done = true;
      return rc;
    }
  }
  if (g.KH == 7 && g.KW == 7 && g.Cin == 3 && g.Cout == 64 && g.sh == 2 && g.sw == 2 && g.dh == 1 && g.dw == 1) {
    const int rc = lce_b200_internal::stem7_tf32_conv(in, filter, bias, out, g.B, g.H, g.W, g.OH, g.OW, g.ph, g.pw, g.act,
                                                      stream);
    if (rc >= 0) return rc;
  }
  const int Gd = (g.Cout + 15) / 16;
  const size_t direct_smem =
      (static_cast<size_t>(K) * Gd * kDirectGroupStride + Gd * 16) * sizeof(float);
  if (K <= direct_max_k() && g.Cout <= kDirectMaxCout && !((uintptr_t)out & 15) &&
      M * Gd < (1LL << 30) && direct_smem <= 96 * 1024) {
    const int G = Gd;
    const long long threads = M * G;
    const size_t smem = direct_smem;
    if (smem > 48 * 1024) {
      static bool attr[64] = {};   // the attribute is per device
      int dev = 0;
      cudaGetDevice(&dev);
      if (dev < 0 || dev >= 64 || !attr[dev]) {
        cudaFuncSetAttribute(conv_direct16_kernel<0, 0, 0, 4>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (dev >= 0 && dev < 64) attr[dev] = true;
      }
    }
    // 128 threads = (128 / G) pixels x G groups, PX pixels each. PX trades shared-memory weight
    // reads per FMA against registers / resident warps: the two compile-time shapes are latency
    // bound at PX = 4 (236 / 130 registers, 12-18 % of the warp slots); measured best: stem PX = 2.
    static const int px_env = [] {
      const char* e = getenv("LCE_B200_DIRECT_PX");
      return e ? atoi(e) : 0;
    }();
    const bool stem = g.KH == 3 && g.KW == 3 && g.Cin == 3;
    const bool pw16 = g.KH == 1 && g.KW == 1 && g.Cin == 16 && !((uintptr_t)in & 15);
    int PX = stem ? 2 : 4;
    if ((stem || pw16) && (px_env == 1 || px_env == 2 || px_env == 4)) PX = px_env;
    const int px_per_blk = 128 / G;
    const long long tiles = (M + px_per_blk * PX - 1) / (px_per_blk * PX);
    // the pointwise 16 -> 64 layer stages 4 KB of weights per block for only 128 pixels: give a
    // block 8 tiles (measured 0.125 -> 0.109 ms); the stem is better off with more, smaller
    // blocks (0.168 -> 0.132 ms at PX = 2, one tile per block)
    const int tpb = (pw16 && PX == 4) ? static_cast<int>(std::max<long long>(
                                            1, std::min<long long>(8, tiles / (132 * 8))))
                                      : 1;
    const unsigned blocks = static_cast<unsigned>((tiles + tpb - 1) / tpb);
    (void)threads;
    cudaStream_t st = as_stream(stream);
    // fused LceQuantize: whole words per pixel, lane pairs hold the two halves of a word
    int32_t* pk = (packed && (g.Cout & 31) == 0 && (G & 1) == 0 && 128 % G == 0) ? packed : nullptr;
    if (pk) *packed_done = true;
#define LCE_DIRECT(KH_, KW_, CIN_, PX_) \
  conv_direct16_kernel<KH_, KW_, CIN_, PX_><<<blocks, 128, smem, st>>>(in, filter, bias, out, g, M, G, tpb, pk)
    if (stem) {
      if (PX == 1) LCE_DIRECT(3, 3, 3, 1);
      else if (PX == 2) LCE_DIRECT(3, 3, 3, 2);
      else LCE_DIRECT(3, 3, 3, 4);
    } else if (pw16) {
      if (PX == 1) LCE_DIRECT(1, 1, 16, 1);
      else if (PX == 2) LCE_DIRECT(1, 1, 16, 2);
      else
        conv_direct16_kernel<1, 1, 16, 4, true><<<blocks, 128, smem, st>>>(in, filter, bias, out, g,
                                                                           M, G, tpb, pk);
    } else {
      LCE_DIRECT(0, 0, 0, 4);
    }
#undef LCE_DIRECT
    return launch_check("conv_direct16_kernel");
  }
  const bool plain = g.KH == 1 && g.KW == 1 && g.sh == 1 && g.sw == 1 && (K & 3) == 0 &&
                     !((uintptr_t)in & 15) && !((uintptr_t)filter & 15) && !((uintptr_t)out & 15);
  if (plain && ((M + kPM - 1) / kPM) * ((g.Cout + kPN - 1) / kPN) < 74) {
    dim3 sgrid(static_cast<unsigned>((M + kSM_ - 1) / kSM_), (g.Cout + kSN_ - 1) / kSN_);
    gemm_small_m_kernel<<<sgrid, 256, 0, as_stream(stream)>>>(in, filter, bias, out, M, g.Cout, K,
                                                              g.act);
    return launch_check("gemm_small_m_kernel");
  }
  if (plain) {
    dim3 grid(static_cast<unsigned>((M + kPM - 1) / kPM), (g.Cout + kPN - 1) / kPN);
    int32_t* pk = (packed && (g.Cout & 31) == 0) ? packed : nullptr;
    if (pk) *packed_done = true;
    conv_gemm128_kernel<<<grid, 256, 0, as_stream(stream)>>>(in, filter, bias, out, M, g.Cout, K,
                                                             g.act, pk);
    return launch_check("conv_gemm128_kernel");
  }
  if (K <= kIKMax && static_cast<long long>(g.H) * g.W * g.Cin < (1LL << 31))
    return igemm_conv(g, M, in, filter, bias, out, stream);
  dim3 grid(static_cast<unsigned>((M + kGM - 1) / kGM), (g.Cout + kGN - 1) / kGN);
  conv_gemm_kernel<<<grid, 256, 0, as_stream(stream)>>>(in, filter, bias, out, g, M);
  return launch_check("conv_gemm_kernel");
}

int lce_b200_f32_conv2d(const lce_f32_conv_desc* d, const float* in, const float* filter,
                        const float* bias, float* out, void* stream) {
  bool done = false;
  return conv2d_impl(d, in, filter, bias, out, nullptr, &done, stream);
}

int lce_b200_f32_conv2d_packed(const lce_f32_conv_desc* d, const float* in, const float* filter,
                               const float* bias, float* out, int32_t* packed_out, void* stream) {
  if (!packed_out) return lce_b200_f32_conv2d(d, in, filter, bias, out, stream);
  bool done = false;
  if (conv2d_impl(d, in, filter, bias, out, packed_out, &done, stream)) return 1;
  if (done) return 0;
  int oh, ow;
  if (lce_b200_f32_conv_out_shape(d, &oh, &ow)) return 1;
  return lce_b200_quantize(LCE_T_FLOAT, out, static_cast<int64_t>(d->batch) * oh * ow, d->out_c, 0,
                           packed_out, stream);
}

int lce_b200_f32_depthwise_conv2d(const lce_f32_conv_desc* d, const float* in,
                                  const float* filter, const float* bias, float* out,
                                  void* stream) {
  ConvGeom g;
  if (make_geom(d, &g)) return 1;
  if (d->out_c != d->in_c) return fail("depthwise conv: depth_multiplier must be 1");
  const long long n = static_cast<long long>(g.B) * g.OH * g.OW * g.Cout;
  if (n == 0) return 0;
  const bool a16 = !((uintptr_t)in & 15) && !((uintptr_t)filter & 15) && !((uintptr_t)out & 15) &&
                   !((uintptr_t)bias & 15);
  if ((g.Cout & 3) == 0 && a16 && g.B <= 65535 && g.OH <= 65535) {
    const int C4 = g.Cout >> 2;
    dim3 grid((g.OW * C4 + 255) / 256, g.OH, g.B);
    if (g.KH == 3 && g.KW == 3)
      depthwise_v4_kernel<3><<<grid, 256, 0, as_stream(stream)>>>(
          reinterpret_cast<const float4*>(in), reinterpret_cast<const float4*>(filter),
          reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(out), g);
    else
      depthwise_v4_kernel<0><<<grid, 256, 0, as_stream(stream)>>>(
          reinterpret_cast<const float4*>(in), reinterpret_cast<const float4*>(filter),
          reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(out), g);
    return launch_check("depthwise_v4_kernel");
  }
  depthwise_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(in, filter, bias, out, g, n);
  return launch_check("depthwise_kernel");
}

int lce_b200_f32_pool_out_shape(const lce_f32_pool_desc* d, int* out_h, int* out_w) {
  if (d->filter_h < 1 || d->filter_w < 1 || d->stride_h < 1 || d->stride_w < 1)
    return fail("pool: bad parameters");
  *out_h = out_size(d->padding, d->in_h, d->filter_h, d->stride_h, 1);
  *out_w = out_size(d->padding, d->in_w, d->filter_w, d->stride_w, 1);
  return 0;
}

static int run_pool(bool is_max, const lce_f32_pool_desc* d, const float* in, float* out,
                    void* stream) {
  int oh, ow;
  if (lce_b200_f32_pool_out_shape(d, &oh, &ow)) return 1;
  const long long n = static_cast<long long>(d->batch) * oh * ow * d->channels;
  if (n <= 0) return 0;
  const int ph = pad_before(d->stride_h, 1, d->in_h, d->filter_h, oh);
  const int pw = pad_before(d->stride_w, 1, d->in_w, d->filter_w, ow);
  if ((d->channels & 3) == 0 && !((uintptr_t)in & 15) && !((uintptr_t)out & 15) &&
      d->batch <= 65535 && oh <= 65535) {
    const int C4 = d->channels >> 2;
    dim3 grid((ow * C4 + 255) / 256, oh, d->batch);
#define LCE_POOL_V4(MAXV, F)                                                                   \
  pool_v4_kernel<MAXV, F><<<grid, 256, 0, as_stream(stream)>>>(                                \
      reinterpret_cast<const float4*>(in), reinterpret_cast<float4*>(out), d->in_h, d->in_w,   \
      C4, oh, ow, d->filter_h, d->filter_w, d->stride_h, d->stride_w, ph, pw, d->activation)
    const int f = (d->filter_h == d->filter_w && (d->filter_h == 2 || d->filter_h == 3))
                      ? d->filter_h : 0;
    if (is_max) {
      if (f == 2) LCE_POOL_V4(true, 2); else if (f == 3) LCE_POOL_V4(true, 3); else LCE_POOL_V4(true, 0);
    } else {
      if (f == 2) LCE_POOL_V4(false, 2); else if (f == 3) LCE_POOL_V4(false, 3); else LCE_POOL_V4(false, 0);
    }
#undef LCE_POOL_V4
    return launch_check("pool_v4_kernel");
  }
  if (is_max)
    pool_kernel<true><<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(
        in, out, d->batch, d->in_h, d->in_w, d->channels, oh, ow, d->filter_h, d->filter_w,
        d->stride_h, d->stride_w, ph, pw, d->activation);
  else
    pool_kernel<false><<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(
        in, out, d->batch, d->in_h, d->in_w, d->channels, oh, ow, d->filter_h, d->filter_w,
        d->stride_h, d->stride_w, ph, pw, d->activation);
  return launch_check("pool_kernel");
}
int lce_b200_f32_max_pool(const lce_f32_pool_desc* d, const float* in, float* out, void* s) {
  return run_pool(true, d, in, out, s);
}
int lce_b200_f32_avg_pool(const lce_f32_pool_desc* d, const float* in, float* out, void* s) {
  return run_pool(false, d, in, out, s);
}

static bool vec4_ok(const void* a, const void* b, const void* o, int64_t n, int64_t b_len) {
  return b_len == n && (n & 3) == 0 && !((uintptr_t)a & 15) && !((uintptr_t)b & 15) &&
         !((uintptr_t)o & 15);
}
int lce_b200_f32_maxpool2x2_depthwise3x3(const lce_f32_pool_desc* pool, const lce_f32_conv_desc* dw,
                                         const float* in, const float* filter, const float* bias,
                                         float* out, void* stream) {
  int ph_, pw_;
  if (lce_b200_f32_pool_out_shape(pool, &ph_, &pw_)) return 1;
  if (pool->filter_h != 2 || pool->filter_w != 2 || pool->stride_h != 1 || pool->stride_w != 1 ||
      pool->padding != LCE_PADDING_VALID || pool->activation != LCE_ACT_NONE)
    return fail("maxpool2x2_depthwise3x3: the pool must be 2x2, stride 1, VALID, no activation");
  ConvGeom g;
  if (make_geom(dw, &g)) return 1;
  if (dw->filter_h != 3 || dw->filter_w != 3 || dw->dilation_h != 1 || dw->dilation_w != 1 ||
      dw->out_c != dw->in_c || (dw->in_c & 3) || dw->in_c != pool->channels ||
      dw->in_h != ph_ || dw->in_w != pw_ || dw->batch != pool->batch)
    return fail("maxpool2x2_depthwise3x3: unsupported depthwise shape");
  if (((uintptr_t)in & 15) || ((uintptr_t)filter & 15) || ((uintptr_t)out & 15) ||
      ((uintptr_t)bias & 15) || g.B > 65535 || g.OH > 65535)
    return fail("maxpool2x2_depthwise3x3: unaligned pointers or too many rows");
  const long long n = static_cast<long long>(g.B) * g.OH * g.OW * g.Cout;
  if (n == 0) return 0;
  const int C4 = g.Cout >> 2;
  dim3 grid((g.OW * C4 + 255) / 256, g.OH, g.B);
  pool2_dw3_v4_kernel<<<grid, 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(in), reinterpret_cast<const float4*>(filter),
      reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(out), pool->in_h,
      pool->in_w, C4, ph_, pw_, g.OH, g.OW, g.sh, g.sw, g.ph, g.pw, g.act);
  return launch_check("pool2_dw3_v4_kernel");
}

int lce_b200_f32_stem_conv_dw(const lce_f32_conv_desc* conv1, const lce_f32_conv_desc* dw, int in_type, const void* in,
                              double in_scale, int32_t in_zero_point, const float* w1, const float* b1, const float* w2,
                              const float* b2, float* out, void* stream) {
  ConvGeom g1, g2;
  if (make_geom(conv1, &g1) || make_geom(dw, &g2)) return 1;
  const bool ok = g1.KH == 3 && g1.KW == 3 && g1.sh == 2 && g1.sw == 2 && g1.dh == 1 && g1.dw == 1 && g1.Cin == 3 &&
                  (g1.Cout == 8 || g1.Cout == 16) && g2.KH == 3 && g2.KW == 3 && g2.sh == 2 && g2.sw == 2 &&
                  g2.dh == 1 && g2.dw == 1 && g2.Cin == g1.Cout && g2.Cout == g1.Cout && g2.H == g1.OH &&
                  g2.W == g1.OW && g2.B == g1.B;
  if (!ok) return fail("stem_conv_dw: unsupported shapes (3x3/s2 3 -> 8 or 16, depthwise 3x3/s2)");
  if (in_type != LCE_T_FLOAT && in_type != LCE_T_INT8 && in_type != LCE_T_BOOL) return fail("stem_conv_dw: bad input type");
  if ((uintptr_t)out & 15) return fail("stem_conv_dw: unaligned output");
  if (g1.B == 0 || g2.OH == 0 || g2.OW == 0) return 0;
  Stem2Geom s{};
  s.B = g1.B; s.H = g1.H; s.W = g1.W; s.OH1 = g1.OH; s.OW1 = g1.OW; s.ph1 = g1.ph; s.pw1 = g1.pw;
  s.OH2 = g2.OH; s.OW2 = g2.OW; s.ph2 = g2.ph; s.pw2 = g2.pw; s.act1 = g1.act; s.act2 = g2.act;
  s.n_rt = (g2.OH + kS2R - 1) / kS2R;
  s.n_ct = (g2.OW + kS2TW - 1) / kS2TW;
  s.in_scale = in_scale; s.in_zero_point = in_zero_point;
  const int es = in_type == LCE_T_FLOAT ? 4 : 1;
  // every image row starts 16-byte aligned, so a fetch that starts at a 16-column boundary and ends
  // at the row's end or 240 columns on is a whole number of 16-byte chunks
  s.aligned = (((uintptr_t)in & 15) == 0 && (static_cast<long long>(g1.W) * 3 * es) % 16 == 0) ? 1 : 0;
  if (!w1 || !w2) return fail("stem_conv_dw: the filters must be host pointers");
  if (g1.Cout == 8) return stem2_run<8>(in_type, in, w1, b1, w2, b2, out, s, stream);
  return stem2_run<16>(in_type, in, w1, b1, w2, b2, out, s, stream);
}

int lce_b200_f32_add(const float* a, const float* b, float* out, int64_t n, int64_t b_len,
                     int act, void* stream) {
  if (n <= 0) return 0;
  if (b_len <= 0 || n % b_len) return fail("add: operand shapes do not broadcast");
  eltwise_kernel<0><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      a, b, out, n, b_len, act, vec4_ok(a, b, out, n, b_len));
  return launch_check("eltwise_kernel<add>");
}
int lce_b200_f32_mul(const float* a, const float* b, float* out, int64_t n, int64_t b_len,
                     int act, void* stream) {
  if (n <= 0) return 0;
  if (b_len <= 0 || n % b_len) return fail("mul: operand shapes do not broadcast");
  eltwise_kernel<1><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      a, b, out, n, b_len, act, vec4_ok(a, b, out, n, b_len));
  return launch_check("eltwise_kernel<mul>");
}
int lce_b200_f32_activation(const float* in, float* out, int64_t n, int act, void* stream) {
  if (n <= 0) return 0;
  eltwise_kernel<2><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      in, in, out, n, n, act, vec4_ok(in, in, out, n, n));
  return launch_check("eltwise_kernel<act>");
}

int lce_b200_f32_maximum(const float* a, const float* b, float* out, int64_t n, int64_t b_len,
                         void* stream) {
  if (n <= 0) return 0;
  if (b_len <= 0 || n % b_len) return fail("maximum: operand shapes do not broadcast");
  eltwise_kernel<3><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      a, b, out, n, b_len, LCE_ACT_NONE, vec4_ok(a, b, out, n, b_len));
  return launch_check("eltwise_kernel<maximum>");
}
int lce_b200_f32_minimum(const float* a, const float* b, float* out, int64_t n, int64_t b_len,
                         void* stream) {
  if (n <= 0) return 0;
  if (b_len <= 0 || n % b_len) return fail("minimum: operand shapes do not broadcast");
  eltwise_kernel<4><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      a, b, out, n, b_len, LCE_ACT_NONE, vec4_ok(a, b, out, n, b_len));
  return launch_check("eltwise_kernel<minimum>");
}
int lce_b200_f32_div(const float* a, const float* b, float* out, int64_t n, int64_t b_len, int act,
                     void* stream) {
  if (n <= 0) return 0;
  if (b_len <= 0 || n % b_len) return fail("div: operand shapes do not broadcast");
  eltwise_kernel<5><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      a, b, out, n, b_len, act, vec4_ok(a, b, out, n, b_len));
  return launch_check("eltwise_kernel<div>");
}
int lce_b200_f32_round(const float* in, float* out, int64_t n, void* stream) {
  if (n <= 0) return 0;
  eltwise_kernel<6><<<grid_for(n / 4 + 1, 256), 256, 0, as_stream(stream)>>>(
      in, in, out, n, n, LCE_ACT_NONE, vec4_ok(in, in, out, n, n));
  return launch_check("eltwise_kernel<round>");
}

int lce_b200_f32_chain_sign(const float* x, const lce_chain_desc* chain, int64_t rows, int channels,
                            float* out, int32_t* packed, void* stream) {
  if (rows < 0 || channels <= 0) return fail("chain_sign: bad shape (%lld rows, %d channels)",
                                             static_cast<long long>(rows), channels);
  if (rows == 0 || (out == nullptr && packed == nullptr)) return 0;
  const lce_chain_desc ch = chain ? *chain : lce_chain_desc{nullptr, nullptr, nullptr, nullptr};
  const int cw = (channels + 31) / 32;
  const long long n = packed ? rows * cw * 32 : rows * static_cast<long long>(channels);
  const int grid = grid_for(n, 256);
  cudaStream_t s = as_stream(stream);
  // 32-bit index arithmetic where it fits (the row / channel split is a division per element)
  const bool narrow = n + 256LL * grid < (1LL << 31);
  if (packed) {
    if (narrow)
      chain_sign_kernel<true, int><<<grid, 256, 0, s>>>(x, ch, static_cast<int>(rows), channels, cw, out, packed);
    else
      chain_sign_kernel<true, long long><<<grid, 256, 0, s>>>(x, ch, rows, channels, cw, out, packed);
  } else {
    if (narrow)
      chain_sign_kernel<false, int><<<grid, 256, 0, s>>>(x, ch, static_cast<int>(rows), channels, cw, out, packed);
    else
      chain_sign_kernel<false, long long><<<grid, 256, 0, s>>>(x, ch, rows, channels, cw, out, packed);
  }
  return launch_check("chain_sign_kernel");
}

int lce_b200_f32_gate_sign(const float* x, const lce_gate_desc* gate, const float* residual, int act,
                           int64_t batch, int64_t pixels, int channels, float* out, int32_t* packed,
                           void* stream) {
  if (batch < 0 || pixels < 0 || channels <= 0)
    return fail("gate_sign: bad shape (%lld images, %lld pixels, %d channels)",
                static_cast<long long>(batch), static_cast<long long>(pixels), channels);
  if (!gate || !gate->gate) return fail("gate_sign: the gate tensor is required");
  if (act < LCE_ACT_NONE || act > LCE_ACT_RELU6) return fail("gate_sign: unknown activation %d", act);
  const long long rows = batch * pixels;
  if (rows == 0 || (out == nullptr && packed == nullptr)) return 0;
  const int cw = (channels + 31) / 32;
  const long long n = packed ? rows * cw * 32 : rows * static_cast<long long>(channels);
  const int grid = grid_for(n, 256);
  cudaStream_t s = as_stream(stream);
  const bool narrow = n + 256LL * grid < (1LL << 31) && batch * static_cast<long long>(channels) < (1LL << 31);
  if (packed) {
    if (narrow)
      gate_sign_kernel<true, int><<<grid, 256, 0, s>>>(x, *gate, residual, act, static_cast<int>(rows),
                                                       static_cast<int>(pixels), channels, cw, out, packed);
    else
      gate_sign_kernel<true, long long><<<grid, 256, 0, s>>>(x, *gate, residual, act, rows, pixels, channels,
                                                             cw, out, packed);
  } else {
    if (narrow)
      gate_sign_kernel<false, int><<<grid, 256, 0, s>>>(x, *gate, residual, act, static_cast<int>(rows),
                                                        static_cast<int>(pixels), channels, cw, out, packed);
    else
      gate_sign_kernel<false, long long><<<grid, 256, 0, s>>>(x, *gate, residual, act, rows, pixels, channels,
                                                              cw, out, packed);
  }
  return launch_check("gate_sign_kernel");
}

int lce_b200_f32_scale_sign(const float* x, const lce_scale_desc* scale, const float* residual, int act,
                            int64_t batch, int64_t pixels, int channels, float* out, int32_t* packed,
                            void* stream) {
  if (batch < 0 || pixels < 0 || channels <= 0)
    return fail("scale_sign: bad shape (%lld images, %lld pixels, %d channels)",
                static_cast<long long>(batch), static_cast<long long>(pixels), channels);
  if (!scale || !scale->scale) return fail("scale_sign: the scale tensor is required");
  if (act < LCE_ACT_NONE || act > LCE_ACT_RELU6) return fail("scale_sign: unknown activation %d", act);
  const long long rows = batch * pixels;
  if (rows == 0 || (out == nullptr && packed == nullptr)) return 0;
  const lce_gate_desc gd{scale->scale, nullptr, scale->sign_scale, scale->sign_shift};
  const int cw = (channels + 31) / 32;
  const long long n = packed ? rows * cw * 32 : rows * static_cast<long long>(channels);
  const int grid = grid_for(n, 256);
  cudaStream_t s = as_stream(stream);
  const bool narrow = n + 256LL * grid < (1LL << 31);   // pixels * channels <= rows * channels too
  if (packed) {
    if (narrow)
      gate_sign_kernel<true, int, true><<<grid, 256, 0, s>>>(x, gd, residual, act, static_cast<int>(rows),
                                                             static_cast<int>(pixels), channels, cw, out, packed);
    else
      gate_sign_kernel<true, long long, true><<<grid, 256, 0, s>>>(x, gd, residual, act, rows, pixels,
                                                                   channels, cw, out, packed);
  } else {
    if (narrow)
      gate_sign_kernel<false, int, true><<<grid, 256, 0, s>>>(x, gd, residual, act, static_cast<int>(rows),
                                                              static_cast<int>(pixels), channels, cw, out, packed);
    else
      gate_sign_kernel<false, long long, true><<<grid, 256, 0, s>>>(x, gd, residual, act, rows, pixels,
                                                                    channels, cw, out, packed);
  }
  return launch_check("gate_sign_kernel (per position)");
}

int lce_b200_f32_affine_sign(const float* x, int64_t x_pixel_stride, int64_t rows, int channels,
                             const float* scale, const float* shift, int32_t* packed, float* copy,
                             int64_t copy_pixel_stride, void* stream) {
  if (rows < 0 || channels <= 0 || x_pixel_stride < channels ||
      (copy != nullptr && copy_pixel_stride < channels))
    return fail("affine_sign: bad shape (%lld rows, %d channels, pixel strides %lld and %lld)",
                static_cast<long long>(rows), channels, static_cast<long long>(x_pixel_stride),
                static_cast<long long>(copy_pixel_stride));
  if (packed == nullptr) return fail("affine_sign: the packed output is required");
  if (rows == 0) return 0;
  const int cw = (channels + 31) / 32;
  const long long n = rows * cw * 32;
  const int grid = grid_for(n, 256);
  cudaStream_t s = as_stream(stream);
  // 32-bit index arithmetic where it fits (the row / channel split is a division per element)
  const long long widest = std::max<long long>(x_pixel_stride, copy ? copy_pixel_stride : 0);
  if (n + 256LL * grid < (1LL << 31) && rows * widest < (1LL << 31))
    affine_sign_kernel<int><<<grid, 256, 0, s>>>(x, static_cast<int>(x_pixel_stride), static_cast<int>(rows),
                                                 channels, cw, scale, shift, packed, copy,
                                                 static_cast<int>(copy_pixel_stride));
  else
    affine_sign_kernel<long long><<<grid, 256, 0, s>>>(x, x_pixel_stride, rows, channels, cw, scale, shift,
                                                       packed, copy, copy_pixel_stride);
  return launch_check("affine_sign_kernel");
}

int lce_b200_f32_maxpool_affine_sign(const float* x, int batch, int in_h, int in_w, int channels,
                                     int filter_h, int filter_w, int stride_h, int stride_w, int padding,
                                     int activation, const float* scale, const float* shift,
                                     int32_t* packed, void* stream) {
  if (batch < 0 || in_h <= 0 || in_w <= 0 || channels <= 0)
    return fail("maxpool_affine_sign: bad shape (%d x %d x %d x %d)", batch, in_h, in_w, channels);
  if (padding != LCE_PADDING_SAME && padding != LCE_PADDING_VALID)
    return fail("maxpool_affine_sign: unknown padding %d", padding);
  if (packed == nullptr) return fail("maxpool_affine_sign: the packed output is required");
  const lce_f32_pool_desc d{batch, in_h, in_w, channels, filter_h, filter_w, stride_h, stride_w, padding,
                            activation};
  int oh, ow;
  if (lce_b200_f32_pool_out_shape(&d, &oh, &ow)) return 1;
  if (batch == 0 || oh <= 0 || ow <= 0) return 0;
  const int ph = pad_before(stride_h, 1, in_h, filter_h, oh);
  const int pw = pad_before(stride_w, 1, in_w, filter_w, ow);
  const int cw = (channels + 31) / 32;
  const long long words = static_cast<long long>(batch) * oh * ow * cw;
  const int grid = grid_for(words * 32, 256);
  cudaStream_t s = as_stream(stream);
  const int f = filter_h == filter_w && (filter_h == 2 || filter_h == 3) ? filter_h : 0;
  // 32-bit index arithmetic where the input and the word count fit
  const bool narrow = static_cast<long long>(batch) * in_h * in_w * channels < (1LL << 31) &&
                      words + 8LL * grid < (1LL << 31);
#define LCE_MAXPOOL_SIGN(F, I)                                                                            \
  maxpool_affine_sign_kernel<F, I><<<grid, 256, 0, s>>>(x, in_h, in_w, channels, oh, ow, cw, filter_h,   \
                                                        filter_w, stride_h, stride_w, ph, pw, activation, \
                                                        scale, shift, packed, static_cast<I>(words))
  if (narrow) {
    if (f == 2) LCE_MAXPOOL_SIGN(2, int); else if (f == 3) LCE_MAXPOOL_SIGN(3, int); else LCE_MAXPOOL_SIGN(0, int);
  } else {
    if (f == 2) LCE_MAXPOOL_SIGN(2, long long); else if (f == 3) LCE_MAXPOOL_SIGN(3, long long);
    else LCE_MAXPOOL_SIGN(0, long long);
  }
#undef LCE_MAXPOOL_SIGN
  return launch_check("maxpool_affine_sign_kernel");
}

int lce_b200_f32_quant2_planes(const float* x, int batch, int in_h, int in_w, int channels, int filter_h,
                               int filter_w, int stride_h, int stride_w, int padding, int activation,
                               int32_t* planes, void* stream) {
  if (batch < 0 || in_h <= 0 || in_w <= 0 || channels <= 0)
    return fail("quant2_planes: bad shape (%d x %d x %d x %d)", batch, in_h, in_w, channels);
  if (channels % 32) return fail("quant2_planes: channels (%d) must be a multiple of 32", channels);
  if (planes == nullptr) return fail("quant2_planes: the planes output is required");
  const bool pooled = filter_h != 0 || filter_w != 0;
  int oh = in_h, ow = in_w, ph = 0, pw = 0;
  if (pooled) {
    if (padding != LCE_PADDING_SAME && padding != LCE_PADDING_VALID)
      return fail("quant2_planes: unknown padding %d", padding);
    const lce_f32_pool_desc d{batch, in_h, in_w, channels, filter_h, filter_w, stride_h, stride_w, padding,
                              activation};
    if (lce_b200_f32_pool_out_shape(&d, &oh, &ow)) return 1;
    ph = pad_before(stride_h, 1, in_h, filter_h, oh);
    pw = pad_before(stride_w, 1, in_w, filter_w, ow);
  }
  if (batch == 0 || oh <= 0 || ow <= 0) return 0;
  const int cw = channels / 32;
  const long long words = static_cast<long long>(batch) * oh * ow * cw;
  const int grid = grid_for(words * 32, 256);
  cudaStream_t s = as_stream(stream);
  const int f = !pooled ? 1 : filter_h == 3 && filter_w == 3 ? 3 : 0;
  // 32-bit index arithmetic where the input, the output and the word count fit
  const bool narrow = static_cast<long long>(batch) * in_h * in_w * channels < (1LL << 31) &&
                      3 * words + 8LL * grid < (1LL << 31);
#define LCE_QUANT2(F, I)                                                                                  \
  quant2_planes_kernel<F, I><<<grid, 256, 0, s>>>(x, in_h, in_w, channels, oh, ow, cw, filter_h, filter_w, \
                                                  stride_h, stride_w, ph, pw, activation, planes,         \
                                                  static_cast<I>(words))
  if (narrow) {
    if (f == 1) LCE_QUANT2(1, int); else if (f == 3) LCE_QUANT2(3, int); else LCE_QUANT2(0, int);
  } else {
    if (f == 1) LCE_QUANT2(1, long long); else if (f == 3) LCE_QUANT2(3, long long);
    else LCE_QUANT2(0, long long);
  }
#undef LCE_QUANT2
  return launch_check("quant2_planes_kernel");
}

int lce_b200_f32_shift_sign_planes(const float* x, int64_t pixels, int channels, int n_planes,
                                   const float* shifts, int32_t* const* planes, void* stream) {
  if (pixels < 0 || channels <= 0) return fail("shift_sign_planes: bad shape (%lld x %d)",
                                               static_cast<long long>(pixels), channels);
  if (channels % 32) return fail("shift_sign_planes: channels (%d) must be a multiple of 32", channels);
  if (n_planes < 1 || n_planes > 8) return fail("shift_sign_planes: 1 to 8 planes, not %d", n_planes);
  if (!shifts || !planes) return fail("shift_sign_planes: the shifts and planes are required");
  ShiftPlanes sp{};
  for (int k = 0; k < n_planes; ++k) {
    if (!planes[k]) return fail("shift_sign_planes: plane %d is NULL", k);
    sp.shift[k] = shifts[k];
    sp.planes[k] = planes[k];
  }
  if (pixels == 0) return 0;
  const int cw = channels / 32;
  const long long words = pixels * cw;
  const int grid = grid_for(words * 32, 256);
  cudaStream_t s = as_stream(stream);
  // 32-bit index arithmetic where the input and the word count fit
  if (pixels * channels + 8LL * 32 * grid < (1LL << 31))
    shift_sign_planes_kernel<int><<<grid, 256, 0, s>>>(x, channels, cw, n_planes, sp, static_cast<int>(words));
  else
    shift_sign_planes_kernel<long long><<<grid, 256, 0, s>>>(x, channels, cw, n_planes, sp, words);
  return launch_check("shift_sign_planes_kernel");
}

int lce_b200_f32_grouped_conv2d(const lce_f32_conv_desc* d, int groups, const float* in, const float* filter,
                                const float* bias, const float* scale, const float* shift, int post_activation,
                                float* out, void* stream) {
  ConvGeom g;
  if (d == nullptr) return fail("grouped conv: no descriptor");
  if (make_geom(d, &g)) return 1;
  if (groups < 1 || g.Cin % groups || g.Cout % groups)
    return fail("grouped conv: %d groups must divide the %d input and %d output channels", groups, g.Cin, g.Cout);
  if (d->padding != LCE_PADDING_SAME && d->padding != LCE_PADDING_VALID)
    return fail("grouped conv: unknown padding %d", d->padding);
  const long long n = static_cast<long long>(g.B) * g.OH * g.OW * g.Cout;
  if (n == 0) return 0;
  if (in == nullptr || filter == nullptr || out == nullptr) return fail("grouped conv: null tensor");
  const int cg = g.Cin / groups, og = g.Cout / groups;
  const GroupedEpilogue e{bias, scale, shift, g.act, post_activation};
  cudaStream_t s = as_stream(stream);
  const bool a16 = !((uintptr_t)in & 15) && !((uintptr_t)out & 15);
  if (g.KH == 3 && g.KW == 3 && g.sh == 1 && g.sw == 1 && g.dh == 1 && g.dw == 1 && a16 && g.B <= 65535) {
    const dim3 grid((g.OW + kGTW - 1) / kGTW, (g.OH + kGTH - 1) / kGTH, g.B);
    if (cg == 8 && og == 8 && groups == 4) {
      grouped_conv3x3_kernel<8, 8, 4><<<grid, 256, 0, s>>>(in, filter, out, g, e);
      return launch_check("grouped_conv3x3_kernel");
    }
    if (cg == 4 && og == 8 && groups == 8) {
      grouped_conv3x3_kernel<4, 8, 8><<<grid, 256, 0, s>>>(in, filter, out, g, e);
      return launch_check("grouped_conv3x3_kernel");
    }
  }
  grouped_conv_any_kernel<<<grid_for(n, 256), 256, 0, s>>>(in, filter, out, g, cg, og, e, n);
  return launch_check("grouped_conv_any_kernel");
}

int lce_b200_f32_logistic(const float* in, float* out, int64_t n, void* stream) {
  if (n < 0) return fail("logistic: bad size %lld", static_cast<long long>(n));
  if (n == 0) return 0;
  logistic_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(in, out, n);
  return launch_check("logistic_kernel");
}

}  // extern "C"

namespace {
// The reference's scale, in float: in / out, or (in - 1) / (out - 1) with align_corners and out > 1
ResizeAxis resize_axis(int in, int out, int align_corners) {
  const float scale = align_corners && out > 1 ? static_cast<float>(in - 1) / static_cast<float>(out - 1)
                                               : static_cast<float>(in) / static_cast<float>(out);
  return ResizeAxis{in, out, scale};
}
int resize_geom(const char* op, int batch, int in_h, int in_w, int channels, int out_h, int out_w,
                int align_corners, int half_pixel_centers, ResizeGeom* g) {
  if (batch < 0 || in_h <= 0 || in_w <= 0 || channels <= 0 || out_h <= 0 || out_w <= 0)
    return fail("%s: bad shape (%d x %d x %d x %d to %d x %d)", op, batch, in_h, in_w, channels, out_h, out_w);
  if (static_cast<long long>(std::max(in_w, out_w)) * ((channels + 31) / 32 * 32) >= (1LL << 31) - (1LL << 22))
    return fail("%s: a row of %d x %d floats is too wide", op, std::max(in_w, out_w), channels);
  g->y = resize_axis(in_h, out_h, align_corners);
  g->x = resize_axis(in_w, out_w, align_corners);
  g->batch = batch;
  g->C = channels;
  g->align_corners = align_corners ? 1 : 0;
  g->half_pixel_centers = half_pixel_centers ? 1 : 0;
  return 0;
}
// blockIdx.y over the output rows, blockIdx.x over one row's `per_row` units of work
dim3 row_grid(long long rows, long long per_row, int per_block) {
  return dim3(static_cast<unsigned>(std::min<long long>((per_row + per_block - 1) / per_block, 1024)),
              static_cast<unsigned>(std::min<long long>(rows, 65535)));
}
template <bool BILINEAR>
int resize_run(const char* op, const float* in, int batch, int in_h, int in_w, int channels, int out_h,
               int out_w, int align_corners, int half_pixel_centers, float* out, void* stream) {
  ResizeGeom g;
  if (resize_geom(op, batch, in_h, in_w, channels, out_h, out_w, align_corners, half_pixel_centers, &g)) return 1;
  if (BILINEAR && align_corners && half_pixel_centers)
    return fail("%s: align_corners and half_pixel_centers cannot both be set", op);
  if (batch == 0) return 0;
  if (!in || !out) return fail("%s: null tensor", op);
  const long long row_len = static_cast<long long>(out_w) * channels;
  const bool vec = row_len % 4 == 0 && !((uintptr_t)out & 15);
  const dim3 grid = row_grid(static_cast<long long>(batch) * out_h, vec ? row_len / 4 : row_len, 256);
  cudaStream_t s = as_stream(stream);
  if (BILINEAR) {
    if (vec) resize_bilinear_kernel<4><<<grid, 256, 0, s>>>(in, out, g);
    else resize_bilinear_kernel<1><<<grid, 256, 0, s>>>(in, out, g);
    return launch_check("resize_bilinear_kernel");
  }
  if (vec) resize_nearest_kernel<4><<<grid, 256, 0, s>>>(in, out, g);
  else resize_nearest_kernel<1><<<grid, 256, 0, s>>>(in, out, g);
  return launch_check("resize_nearest_kernel");
}

template <int NCOL, int TN>
int subpixel_launch(const float* in, const float* filter, const float* bias, const float* img, float* out,
                    const SubpixelGeom& g, unsigned M, cudaStream_t s) {
  using Tile = SubpixelTile<NCOL, TN>;
  const int Kpad = (g.KH * g.KW * g.Cin + kIK - 1) / kIK * kIK;
  const size_t smem = Tile::kFloats * sizeof(float) + 2 * static_cast<size_t>(Kpad) * sizeof(int);
  static bool attr[64] = {};   // the attribute is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64 || !attr[dev]) {
    cudaFuncSetAttribute(subpixel_conv_kernel<NCOL, TN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         static_cast<int>(Tile::kFloats * sizeof(float) + 2 * kIKMax * sizeof(int)));
    if (dev >= 0 && dev < 64) attr[dev] = true;
  }
  const unsigned blocks = (M + Tile::BM - 1) / Tile::BM;
  subpixel_conv_kernel<NCOL, TN><<<blocks, 128, smem, s>>>(in, filter, bias, img, out, g, M);
  return launch_check("subpixel_conv_kernel");
}
}  // namespace

extern "C" {

int lce_b200_f32_resize_nearest(const float* in, int batch, int in_h, int in_w, int channels, int out_h, int out_w,
                                int align_corners, int half_pixel_centers, float* out, void* stream) {
  return resize_run<false>("resize_nearest", in, batch, in_h, in_w, channels, out_h, out_w, align_corners,
                           half_pixel_centers, out, stream);
}

int lce_b200_f32_resize_bilinear(const float* in, int batch, int in_h, int in_w, int channels, int out_h,
                                 int out_w, int align_corners, int half_pixel_centers, float* out, void* stream) {
  return resize_run<true>("resize_bilinear", in, batch, in_h, in_w, channels, out_h, out_w, align_corners,
                          half_pixel_centers, out, stream);
}

int lce_b200_f32_upsample_add_sign(const float* u, int batch, int in_h, int in_w, int channels, int out_h,
                                   int out_w, int align_corners, int half_pixel_centers, const float* skip,
                                   int activation, float* out, int32_t* packed, void* stream) {
  ResizeGeom g;
  if (resize_geom("upsample_add_sign", batch, in_h, in_w, channels, out_h, out_w, align_corners,
                  half_pixel_centers, &g))
    return 1;
  if (activation < LCE_ACT_NONE || activation > LCE_ACT_RELU6)
    return fail("upsample_add_sign: unknown activation %d", activation);
  if (!u || !skip) return fail("upsample_add_sign: u and skip are required");
  if (batch == 0 || (out == nullptr && packed == nullptr)) return 0;
  const int cw = (channels + 31) / 32;
  const dim3 grid = row_grid(static_cast<long long>(batch) * out_h, static_cast<long long>(out_w) * cw, 8);
  upsample_add_sign_kernel<<<grid, 256, 0, as_stream(stream)>>>(u, skip, g, cw, activation, out, packed);
  return launch_check("upsample_add_sign_kernel");
}

// Rows of at least this many elements (at inner == 1) take a warp each; shorter rows a thread each.
constexpr int kArgmaxWarpRow = 64;

int lce_b200_f32_argmax(const float* in, int64_t outer, int n, int64_t inner, int out_int64, void* out,
                        void* stream) {
  if (outer < 0 || inner < 0 || n <= 0)
    return fail("argmax: bad shape (%lld x %d x %lld)", static_cast<long long>(outer), n,
                static_cast<long long>(inner));
  if (outer == 0 || inner == 0) return 0;
  if (!in || !out) return fail("argmax: null tensor");
  cudaStream_t s = as_stream(stream);
  if (inner == 1 && n >= kArgmaxWarpRow) {
    const int grid = grid_for(outer, 8);
    if (out_int64) argmax_warp_kernel<int64_t><<<grid, 256, 0, s>>>(in, outer, n, static_cast<int64_t*>(out));
    else argmax_warp_kernel<int32_t><<<grid, 256, 0, s>>>(in, outer, n, static_cast<int32_t*>(out));
    return launch_check("argmax_warp_kernel");
  }
  const int grid = grid_for(outer * inner, 256);
  if (out_int64) argmax_kernel<int64_t><<<grid, 256, 0, s>>>(in, outer, n, inner, static_cast<int64_t*>(out));
  else argmax_kernel<int32_t><<<grid, 256, 0, s>>>(in, outer, n, inner, static_cast<int32_t*>(out));
  return launch_check("argmax_kernel");
}

int lce_b200_f32_reduce_max(const float* in, int64_t outer, int64_t n, int64_t inner, float* out, void* stream) {
  if (outer < 0 || inner < 0 || n < 0)
    return fail("reduce_max: bad shape (%lld x %lld x %lld)", static_cast<long long>(outer), static_cast<long long>(n),
                static_cast<long long>(inner));
  if (outer == 0 || inner == 0) return 0;
  if (!out || (n > 0 && !in)) return fail("reduce_max: null tensor");
  cudaStream_t s = as_stream(stream);
  if (inner == 1 && n >= kArgmaxWarpRow) {
    reduce_max_warp_kernel<<<grid_for(outer, 8), 256, 0, s>>>(in, outer, n, out);
    return launch_check("reduce_max_warp_kernel");
  }
  reduce_max_kernel<<<grid_for(outer * inner, 256), 256, 0, s>>>(in, outer, n, inner, out);
  return launch_check("reduce_max_kernel");
}

// The two staged source rows of bilinear_argmax_kernel fit the default 48 KB of dynamic shared memory.
constexpr int kBilinearArgmaxMaxRowFloats = 48 * 1024 / 2 / static_cast<int>(sizeof(float));

int lce_b200_resize_bilinear_argmax_max_row_floats(void) { return kBilinearArgmaxMaxRowFloats; }

int lce_b200_f32_resize_bilinear_argmax(const float* in, int batch, int in_h, int in_w, int channels, int out_h,
                                        int out_w, int align_corners, int half_pixel_centers, int out_int64,
                                        void* out, void* stream) {
  ResizeGeom g;
  if (resize_geom("resize_bilinear_argmax", batch, in_h, in_w, channels, out_h, out_w, align_corners,
                  half_pixel_centers, &g))
    return 1;
  if (align_corners && half_pixel_centers)
    return fail("resize_bilinear_argmax: align_corners and half_pixel_centers cannot both be set");
  if (static_cast<long long>(in_w) * channels > kBilinearArgmaxMaxRowFloats)
    return fail("resize_bilinear_argmax: a source row of %d x %d floats does not fit shared memory (at most %d)",
                in_w, channels, kBilinearArgmaxMaxRowFloats);
  if (batch == 0) return 0;
  if (!in || !out) return fail("resize_bilinear_argmax: null tensor");
  const dim3 grid = row_grid(static_cast<long long>(batch) * out_h, 1, 1);
  const int threads = std::min(256, (out_w + 31) / 32 * 32);
  const size_t smem = 2 * static_cast<size_t>(in_w) * channels * sizeof(float);
  cudaStream_t s = as_stream(stream);
  if (out_int64) bilinear_argmax_kernel<int64_t><<<grid, threads, smem, s>>>(in, g, static_cast<int64_t*>(out));
  else bilinear_argmax_kernel<int32_t><<<grid, threads, smem, s>>>(in, g, static_cast<int32_t*>(out));
  return launch_check("bilinear_argmax_kernel");
}

int lce_b200_f32_depth_to_space(const float* in, int batch, int in_h, int in_w, int channels, int block_size,
                                float* out, void* stream) {
  if (batch < 0 || in_h <= 0 || in_w <= 0 || channels <= 0 || block_size <= 0)
    return fail("depth_to_space: bad shape (%d x %d x %d x %d, block size %d)", batch, in_h, in_w, channels,
                block_size);
  const int r = block_size;
  if (channels % (static_cast<long long>(r) * r))
    return fail("depth_to_space: %d channels are not a multiple of block_size^2 = %lld", channels,
                static_cast<long long>(r) * r);
  const int run = channels / r;   // r * C'
  const long long row_len = static_cast<long long>(in_w) * run;
  if (row_len >= (1LL << 31) - (1LL << 22) || static_cast<long long>(in_h) * r > INT_MAX)
    return fail("depth_to_space: an output row of %lld floats is too wide", row_len);
  if (batch == 0) return 0;
  if (!in || !out) return fail("depth_to_space: null tensor");
  const bool vec = run % 4 == 0 && !((uintptr_t)in & 15) && !((uintptr_t)out & 15);
  const long long rows = static_cast<long long>(batch) * in_h * r;
  const dim3 grid = row_grid(rows, vec ? row_len / 4 : row_len, 256);
  cudaStream_t s = as_stream(stream);
  if (vec) depth_to_space_kernel<4><<<grid, 256, 0, s>>>(in, out, in_h, in_w, channels, r, rows);
  else depth_to_space_kernel<1><<<grid, 256, 0, s>>>(in, out, in_h, in_w, channels, r, rows);
  return launch_check("depth_to_space_kernel");
}

int lce_b200_f32_transpose_conv2d(const lce_f32_transpose_conv_desc* d, const float* in, const float* filter,
                                  const float* bias, float* out, void* stream) {
  if (!d) return fail("transpose_conv2d: null descriptor");
  const TConvGeom g{d->batch, d->in_h, d->in_w, d->in_c, d->filter_h, d->filter_w, d->out_c, d->out_h, d->out_w,
                    d->stride_h, d->stride_w, d->pad_h, d->pad_w, d->activation};
  if (g.B < 0 || g.H <= 0 || g.W <= 0 || g.Cin <= 0 || g.KH <= 0 || g.KW <= 0 || g.Cout <= 0 || g.OH <= 0 ||
      g.OW <= 0)
    return fail("transpose_conv2d: bad shape (input %d x %d x %d x %d, filter %d x %d x %d, output %d x %d)", g.B,
                g.H, g.W, g.Cin, g.Cout, g.KH, g.KW, g.OH, g.OW);
  if (g.sh <= 0 || g.sw <= 0) return fail("transpose_conv2d: strides must be positive");
  if (g.ph < 0 || g.pw < 0) return fail("transpose_conv2d: padding must not be negative");
  if (g.act < LCE_ACT_NONE || g.act > LCE_ACT_RELU6) return fail("transpose_conv2d: unknown activation %d", g.act);
  if (static_cast<long long>(g.OH) + g.ph + g.KH >= INT_MAX || static_cast<long long>(g.OW) + g.pw + g.KW >= INT_MAX)
    return fail("transpose_conv2d: the output is too large");
  const long long total = static_cast<long long>(g.B) * g.OH * g.OW * ((g.Cout + 3) / 4);
  if (total == 0) return 0;
  if (!in || !filter || !out) return fail("transpose_conv2d: null tensor");
  const bool vec = g.Cin % 4 == 0 && !((uintptr_t)in & 15) && !((uintptr_t)filter & 15);
  cudaStream_t s = as_stream(stream);
  const unsigned grid = grid_for(total, 256);
  if (vec) transpose_conv_kernel<true><<<grid, 256, 0, s>>>(in, filter, bias, out, g, total);
  else transpose_conv_kernel<false><<<grid, 256, 0, s>>>(in, filter, bias, out, g, total);
  return launch_check("transpose_conv_kernel");
}

int lce_b200_subpixel_conv_max_out_channels(void) { return SubpixelTile<8, 8>::BN; }

int lce_b200_f32_subpixel_conv(const lce_f32_conv_desc* d, const float* in, const float* filter, const float* bias,
                               int block_size, const float* img, int img_h, int img_w, int align_corners,
                               int half_pixel_centers, int add_activation, float* out, void* stream) {
  ConvGeom cg;
  if (make_geom(d, &cg)) return 1;
  const int r = block_size;
  if (cg.sh != 1 || cg.sw != 1 || cg.dh != 1 || cg.dw != 1 || d->padding != LCE_PADDING_SAME)
    return fail("subpixel_conv: the convolution must have stride 1, dilation 1 and SAME padding");
  if (r <= 0 || cg.Cout % (r * r))
    return fail("subpixel_conv: %d output channels are not a multiple of block_size^2 (block size %d)", cg.Cout, r);
  if (cg.Cout > lce_b200_subpixel_conv_max_out_channels())
    return fail("subpixel_conv: %d output channels are more than %d", cg.Cout,
                lce_b200_subpixel_conv_max_out_channels());
  const long long K = static_cast<long long>(cg.KH) * cg.KW * cg.Cin;
  const long long M = static_cast<long long>(cg.B) * cg.H * cg.W;
  if (K > kIKMax || static_cast<long long>(cg.H) * cg.W * cg.Cin >= (1LL << 31) || M > (1LL << 31))
    return fail("subpixel_conv: the convolution is too large (K = %lld, %lld pixels)", K, M);
  SubpixelGeom g{cg.B, cg.H, cg.W, cg.Cin, cg.KH, cg.KW, cg.ph, cg.pw, cg.Cout, r, cg.Cout / (r * r),
                 cg.act, add_activation, {}};
  if (static_cast<long long>(cg.H) * r > INT_MAX || static_cast<long long>(cg.W) * r * g.Cp >= (1LL << 31) - (1LL << 22))
    return fail("subpixel_conv: an output row of %d x %d floats is too wide", cg.W * r, g.Cp);
  if (img) {
    if (resize_geom("subpixel_conv", cg.B, img_h, img_w, g.Cp, cg.H * r, cg.W * r, align_corners, half_pixel_centers,
                    &g.img))
      return 1;
    if (align_corners && half_pixel_centers)
      return fail("subpixel_conv: align_corners and half_pixel_centers cannot both be set");
  }
  if (M == 0) return 0;
  if (!in || !filter || !out) return fail("subpixel_conv: null tensor");
  cudaStream_t s = as_stream(stream);
  const unsigned m = static_cast<unsigned>(M);
  if (cg.Cout <= SubpixelTile<4, 4>::BN) return subpixel_launch<4, 4>(in, filter, bias, img, out, g, m, s);
  if (cg.Cout <= SubpixelTile<4, 8>::BN) return subpixel_launch<4, 8>(in, filter, bias, img, out, g, m, s);
  return subpixel_launch<8, 8>(in, filter, bias, img, out, g, m, s);
}

int lce_b200_f32_mean_hw_act(const float* in, float* out, int batch, int h, int w, int c, int pre_activation,
                             void* stream) {
  if (batch <= 0 || c <= 0) return 0;
  if (h * w <= 0) return fail("mean: empty spatial extent");
  mean_hw_kernel<<<(batch * c + 255) / 256, 256, 0, as_stream(stream)>>>(in, out, batch, h * w, c, pre_activation);
  return launch_check("mean_hw_kernel");
}

int lce_b200_f32_mean_hw(const float* in, float* out, int batch, int h, int w, int c,
                         void* stream) {
  return lce_b200_f32_mean_hw_act(in, out, batch, h, w, c, LCE_ACT_NONE, stream);
}

int lce_b200_f32_softmax(const float* in, float* out, int64_t rows, int cols, float beta,
                         void* stream) {
  if (rows <= 0 || cols <= 0) return 0;
  if (rows > 0x7fffffffLL) return fail("softmax: too many rows");
  softmax_kernel<<<static_cast<unsigned>(rows), 128, 0, as_stream(stream)>>>(in, out, cols, beta);
  return launch_check("softmax_kernel");
}

int lce_b200_dequantize_affine(int in_type, const void* in, float* out, int64_t n, double scale,
                               int32_t zero_point, void* stream) {
  if (n <= 0) return 0;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) != 0 || (reinterpret_cast<uintptr_t>(out) & 15u) != 0)
    return fail("dequantize: buffers must be 16-byte aligned");
  const unsigned grid = static_cast<unsigned>(std::min<long long>((n / 16 + 256) / 256, 132 * 16));
  if (in_type == LCE_T_INT8) {
    dequantize_affine_kernel<int8_t><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const int8_t*>(in), out, n, scale,
                                                                          zero_point);
  } else if (in_type == LCE_T_BOOL) {   // the uint8 code of the LCE_T_* enum
    dequantize_affine_kernel<uint8_t><<<grid, 256, 0, as_stream(stream)>>>(static_cast<const uint8_t*>(in), out, n, scale,
                                                                           zero_point);
  } else {
    return fail("dequantize: unsupported quantised type %d", in_type);
  }
  return launch_check("dequantize_affine_kernel");
}

int lce_b200_pad4d_32(const void* in, void* out, const int32_t* in_dims,
                      const int32_t* pad_before, const int32_t* pad_after, uint32_t fill_bits,
                      void* stream) {
  Pad4 p;
  long long total = 1;
  for (int i = 0; i < 4; ++i) {
    if (in_dims[i] < 0 || pad_before[i] < 0 || pad_after[i] < 0)
      return fail("pad: negative dimension or padding");
    p.in[i] = in_dims[i];
    p.before[i] = pad_before[i];
    p.out[i] = in_dims[i] + pad_before[i] + pad_after[i];
    total *= p.out[i];
  }
  if (total == 0) return 0;
  pad4d32_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, as_stream(stream)>>>(
      static_cast<const uint32_t*>(in), static_cast<uint32_t*>(out), p, fill_bits, total);
  return launch_check("pad4d32_kernel");
}

}  // extern "C"
