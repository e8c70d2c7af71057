// lce_b200_pw.cuh -- the fp32 pointwise (1x1, stride 1) CONV_2D either side of the binary path,
// on the tensor cores: out[M][N] = act(A[M][K] * W[N][K]^T + bias[N])  (TFLite reference
// semantics: tensorflow/lite/kernels/internal/reference/conv.h:27; the QuickNet transition and
// stem pointwise layers and Bi-RealNet's shortcut convolutions).
//
// An fp32 FMA GEMM of these shapes is issue-bound well above its HBM time. wgmma .tf32 uses only
// the tf32 part of its operands, so the kernel splits every operand once,
//     hi = rna_tf32(x),  lo = rna_tf32(x - hi)                (x - hi is exact in fp32)
// and accumulates hi*hi + hi*lo + lo*hi in fp32 registers: the dropped terms are ~2^-22 |a||w|
// with random sign, the same order as the rounding of an fp32 FMA chain of this length.
//
// Per CTA (persistent, one per SM), items = (128-row tile, 128-column tile):
//   warp 8      TMA: A[128 x 32 floats] (+ W[128 x 32]) per K block, SWIZZLE_128B, 3 stages
//   warps 0-7   two math warpgroups, 64 rows each: split the W tile hi | lo in shared memory
//               (elementwise, so the swizzle needs no decoding), read their A fragments from the
//               swizzled tile and split them in registers, 12 x wgmma m64n128k8 per K block, then
//               + bias (staged in shared memory once per column tile), activation (+ LceQuantize
//               bits from the accumulators); each warpgroup writes its 64 x 128 results to its
//               own staging tile and one of its threads stores them by TMA, so the stores drain
//               while the warpgroup runs its next item
// 162 registers, no spills; 216,064 B of shared memory (A / W ring 144 KB, output staging 64 KB).
// On an H100 80GB HBM3 at a 700 W power limit, QuickNet batch 256 (per-node CUDA events, 200
// steps), operands read once and results written once: 16 -> 64 106.8 us (2.47 TB/s), 64 -> 128
// 69.5 us (2.26 TB/s), 128 -> 256 63.9 us (1.23 TB/s), 256 -> 512 55.3 us (0.71 TB/s), against
// 187.0, 108.8, 103.4 and 71.9 us when every thread stored float2 pairs straight from its
// accumulators. The two wider layers are bound by their K loop, not by HBM.
// K = 16 (QuickNet's 16 -> 64 pointwise) runs as pixel PAIRS: A'[M/2][32] is the same memory,
// W' = diag(W, W) is built in shared memory once, out'[M/2][128] is the same memory as out.
#ifndef LCE_B200_PW_CUH_
#define LCE_B200_PW_CUH_

#include "lce_b200_tc.cuh"

namespace lce {
namespace pw {

using namespace lce::tc;

constexpr int kPwMathThreads = 256;       // two warpgroups
constexpr int kPwThreads = kPwMathThreads + 32;   // + TMA producer warp
constexpr int kPwNS = 3;                  // A / W stages
constexpr int kPwTile = 16384;            // 128 rows x 128 B
constexpr int kPwWStage = 2 * kPwTile;    // W: hi | lo
constexpr int kPwOBox = 64 * 128;         // output staging: 64 rows x 32 floats
constexpr int kPwOStage = 4 * kPwOBox;    // one warpgroup's 64 x 128 results
constexpr int kPwBarBytes = 1024;
constexpr size_t kPwSmem = kPwNS * (kPwTile + kPwWStage) + 2 * kPwOStage + 1024 + kPwBarBytes + 1024;

struct PwParams {
  long long M;          // rows (pixel pairs in pairs mode)
  int N, KB;            // columns (multiple of 128), K blocks of 32 floats
  int n_tiles, m_tiles;
  int act;              // LCE_ACT_*
  int pairs;            // K = 16, N = 64 run as [M/2][32] x diag(W, W)
  int w_resident;       // n_tiles == 1 and KB <= kPwNS: the weights are staged and split once
  int bias_mask;        // column -> bias index (pairs: & 63)
  const float* filter;  // [N][K] (read directly only in pairs mode)
  const float* bias;    // may be null
  int32_t* packed;      // optional LceQuantize of the output, [M][N / 32]
};

// K-major SWIZZLE_128B operand: 8-row atoms of 1024 B (SBO), layout type 1 (128-byte swizzle)
__device__ __forceinline__ uint32_t sdesc_lo(uint32_t saddr) { return ((saddr & 0x3FFFFu) >> 4) | (1u << 16); }
constexpr uint32_t kSdescHi = (1024u >> 4) | (1u << 30);

// round-to-nearest (ties away from zero) to tf32, as cvt.rna.tf32.f32 does -- but on the integer
// ALU at full rate.
// (No Inf / NaN handling: a value within 2^-11 of FLT_MAX would round to Inf.)
__device__ __forceinline__ float to_tf32(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
__device__ __forceinline__ void split4(float4 x, float4* hi, float4* lo) {
  float4 h = make_float4(to_tf32(x.x), to_tf32(x.y), to_tf32(x.z), to_tf32(x.w));
  *hi = h;
  *lo = make_float4(to_tf32(x.x - h.x), to_tf32(x.y - h.y), to_tf32(x.z - h.z), to_tf32(x.w - h.w));
}
// split one 16 KB tile in place (hi) and into the tile 16 KB above it (lo); 256 threads. All
// loads first: the in-place stores alias the loads.
__device__ __forceinline__ void split_tile(unsigned char* tile, int t) {
  float4* c = reinterpret_cast<float4*>(tile) + t;
  float4 x[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) x[j] = c[kPwMathThreads * j];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float4 h, l;
    split4(x[j], &h, &l);
    c[kPwMathThreads * j] = h;
    c[kPwMathThreads * j + kPwTile / 16] = l;
  }
}
// element (row, k) of a K-major SWIZZLE_128B tile of 32-float rows
__device__ __forceinline__ float swz_at(const unsigned char* tile, int row, int k) {
  return *reinterpret_cast<const float*>(tile + row * 128 + ((((k >> 2) ^ (row & 7))) << 4) + (k & 3) * 4);
}

__device__ __forceinline__ float apply_act(float y, int act) {
  if (act == LCE_ACT_RELU) return fmaxf(y, 0.f);
  if (act == LCE_ACT_RELU6) return fminf(fmaxf(y, 0.f), 6.f);
  if (act == LCE_ACT_RELU_N1_TO_1) return fminf(fmaxf(y, -1.f), 1.f);
  return y;
}

template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc, uint32_t scale_d) {
  if constexpr (N == 128) wgmma_tf32_n128(d, a, desc, scale_d);
  else wgmma_tf32_n64(d, a, desc, scale_d);
}

// The three tf32 passes of one 32-float K block: a_hi / a_lo are the warpgroup's A fragments of
// the four k8 steps, w_lo the descriptor start of the W hi tile (its lo tile follows `lo_ofs`
// bytes above). The small cross terms first, hi*hi last.
template <int N>
__device__ __forceinline__ void tf32_3pass(float (&d)[N / 2], uint32_t (&a_hi)[4][4], uint32_t (&a_lo)[4][4], uint32_t w_lo,
                                           uint32_t lo_ofs, bool first) {
#pragma unroll
  for (int k8 = 0; k8 < 4; ++k8) { fence_regs(a_hi[k8]); fence_regs(a_lo[k8]); }
  wgmma_fence();
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    const uint32_t w = w_lo + (pass == 1 ? (lo_ofs >> 4) : 0);
#pragma unroll
    for (int k8 = 0; k8 < 4; ++k8)
      wgmma_tf32<N>(d, pass == 0 ? a_lo[k8] : a_hi[k8], make_desc(w + 2 * k8, kSdescHi), (!first || pass != 0 || k8 != 0) ? 1u : 0u);
  }
  wgmma_commit();
  wgmma_wait_all();
  fence_regs(d);
}

__global__ void __launch_bounds__(kPwThreads, 1)
pw_tf32_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
               const __grid_constant__ CUtensorMap tm_o, const PwParams p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  unsigned char* a_st = smem;                               // [kPwNS] raw A tiles
  unsigned char* w_st = a_st + kPwNS * kPwTile;             // [kPwNS][hi | lo]
  unsigned char* o_st = w_st + kPwNS * kPwWStage;           // [2 warpgroups] output staging
  float* s_bias = reinterpret_cast<float*>(o_st + 2 * kPwOStage);   // [2 warpgroups][128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(o_st + 2 * kPwOStage + 1024);
  uint64_t* full = bars;                  // TMA landed                          (1 + tx)
  uint64_t* empty = bars + kPwNS;         // MMAs of the stage retired           (8 math warps)

  const int tid = threadIdx.x;
  const int wid = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < kPwNS; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int items = p.n_tiles * p.m_tiles;

  if (wid == 8) {
    // ------------------------------------------------ TMA producer
    uint32_t cnt = 0;
    bool first = true;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
      const int mt = it / p.n_tiles, nt = it - mt * p.n_tiles;
      for (int kb = 0; kb < p.KB; ++kb, ++cnt) {
        const int s = cnt % kPwNS;
        mbar_wait_tc(&empty[s], ((cnt / kPwNS) & 1) ^ 1, 1);
        const bool load_w = !p.pairs && (!p.w_resident || first);
        const int ws = p.w_resident ? kb : s;
        if (elect_one()) {
          mbar_arrive_expect_tx(&full[s], load_w ? 2 * kPwTile : kPwTile);
          tma_load_2d(a_st + s * kPwTile, &tm_a, &full[s], kb * 32, mt * 128);
          if (load_w) tma_load_2d(w_st + ws * kPwWStage, &tm_w, &full[s], kb * 32, nt * 128);
        }
        __syncwarp();
      }
      first = false;
    }
    return;
  }

  // ------------------------------------------------ math warpgroups
  const int g = lane >> 2, t = lane & 3;
  const int wg = wid >> 2, wtid = tid & 127;
  const int r0 = wg * 64 + (wid & 3) * 16 + g;   // tile rows r0 and r0 + 8
  const int pw = p.N >> 5;   // packed words per row
  uint32_t cnt = 0;
  bool first = true;
  for (int it = blockIdx.x; it < items; it += gridDim.x, first = false) {
    const int mt = it / p.n_tiles, nt = it - mt * p.n_tiles;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < p.KB; ++kb, ++cnt) {
      const int s = cnt % kPwNS;
      const int ws = p.w_resident ? kb : s;
      if (p.pairs && first && tid < 128) {
        // W' = diag(W, W): row n' = tid, 32 floats (8 cells of 16 B, swizzled by row & 7)
        unsigned char* row = w_st + ws * kPwWStage + tid * 128;
        const float* src = p.filter + (tid & 63) * 16;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
          if ((c >> 2) == (tid >> 6)) x = __ldg(reinterpret_cast<const float4*>(src) + (c & 3));
          float4 h, l;
          split4(x, &h, &l);
          float4* cell = reinterpret_cast<float4*>(row + ((c ^ (tid & 7)) << 4));
          *cell = h;
          *(cell + kPwTile / 16) = l;
        }
      }
      mbar_wait_tc(&full[s], (cnt / kPwNS) & 1, 4);
      const bool split_w = !p.pairs && (!p.w_resident || first);
      if (split_w) split_tile(w_st + ws * kPwWStage, tid);
      if (split_w || (p.pairs && first)) {
        // both warpgroups read the whole W tile: all of it must be split (and visible to the
        // tensor cores' async proxy) first
        fence_proxy_async();
        named_bar_sync(1, kPwMathThreads);
      }
      const unsigned char* at = a_st + s * kPwTile;
      uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
      for (int k8 = 0; k8 < 4; ++k8)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          // fragment register r: row r0 + 8 * (r & 1), column 8 * k8 + t + 4 * (r >> 1)
          const float x = swz_at(at, r0 + 8 * (r & 1), 8 * k8 + t + 4 * (r >> 1));
          const float h = to_tf32(x);
          a_hi[k8][r] = __float_as_uint(h);
          a_lo[k8][r] = __float_as_uint(to_tf32(x - h));
        }
      tf32_3pass<128>(acc, a_hi, a_lo, sdesc_lo(smem_u32(w_st + ws * kPwWStage)), kPwTile, kb == 0);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // epilogue: register i of block j is row r0 + 8 * ((i >> 1) & 1), column 8j + 2t + (i & 1).
    // The warpgroup stages its 64 x 128 results in shared memory, as four 32-column SWIZZLE_128B
    // boxes, and one thread stores them by TMA; the stores drain while the warpgroup runs its next
    // item. Rows past M and columns past N are outside the tensor map and are not written.
    unsigned char* ost = o_st + wg * kPwOStage;
    float* sb = s_bias + wg * 128;
    if (wtid == 0) bulk_wait_read();   // the previous item's stores have read the staging tile
    if (p.bias != nullptr && (first || p.n_tiles > 1)) {
      const int n = nt * 128 + wtid;
      sb[wtid] = n < p.N ? __ldg(p.bias + (n & p.bias_mask)) : 0.f;
    }
    named_bar_sync(2 + wg, 128);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int rl = (wid & 3) * 16 + g + 8 * rr;   // row in the warpgroup's 64
      const long long row = static_cast<long long>(mt) * 128 + wg * 64 + rl;
      const bool row_ok = row < p.M;
#pragma unroll
      for (int gq = 0; gq < 4; ++gq) {
        uint32_t bits = 0;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j = 4 * gq + jj;
          const float2 bi = p.bias != nullptr ? *reinterpret_cast<const float2*>(sb + 8 * j + 2 * t) : make_float2(0.f, 0.f);
          const float y0 = apply_act(__fadd_rn(acc[4 * j + 2 * rr], bi.x), p.act);
          const float y1 = apply_act(__fadd_rn(acc[4 * j + 2 * rr + 1], bi.y), p.act);
          bits |= ((y0 < 0.0f ? 1u : 0u) | (y1 < 0.0f ? 2u : 0u)) << (8 * jj + 2 * t);
          // box gq, 16-byte cell (2 jj + t / 2) ^ (rl & 7) of row rl
          *reinterpret_cast<float2*>(ost + gq * kPwOBox + rl * 128 + (((2 * jj + (t >> 1)) ^ (rl & 7)) << 4) + (t & 1) * 8) =
              make_float2(y0, y1);
        }
        if (p.packed != nullptr) {
          bits = quad_or(bits);
          if (t == 0 && row_ok) p.packed[row * pw + nt * 4 + gq] = static_cast<int32_t>(bits);
        }
      }
    }
    fence_proxy_async();
    named_bar_sync(2 + wg, 128);
    const long long row0 = static_cast<long long>(mt) * 128 + wg * 64;
    if (wtid == 0 && row0 < p.M) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (nt * 128 + 32 * q < p.N) tma_store_2d(&tm_o, ost + q * kPwOBox, nt * 128 + 32 * q, static_cast<int>(row0));
      bulk_commit();
    }
  }
  if (wtid == 0) bulk_wait();
}


// ------------------------------------------------------------------ 7x7 / stride 2 stem on wgmma .tf32
// Bi-RealNet's first layer, CONV_2D 7x7 stride 2, 3 -> 64 channels: K = 147 (five 32-float K
// blocks, zero-padded), N = 64. Same 3-pass split as above; what differs is the A operand: no
// im2col tensor exists, so no TMA -- each thread gathers the input values of its A fragment (21
// contiguous floats per filter row; neighbours share them through L1) and splits them in
// registers. The filter (37 KB) is split into shared memory once per CTA. Each of the two
// warpgroups of a CTA takes 64-pixel tiles on its own.
constexpr int kS7Threads = 256;
constexpr int kS7K = 147, kS7KB = 5, kS7N = 64;
constexpr int kS7WTile = 64 * 128;                 // 64 rows x 32 floats
constexpr size_t kS7Smem = kS7KB * 2 * kS7WTile + 1024;
struct Stem7Params {
  long long M;           // output pixels
  int H, W, OH, OW, ph, pw;
  int m_tiles, act;      // m_tiles: 64-pixel tiles
  const float* in;       // [B][H][W][3]
  const float* filter;   // [64][7][7][3]
  const float* bias;
  float* out;            // [M][64]
};

__global__ void __launch_bounds__(kS7Threads, 2)
stem7_tf32_kernel(const Stem7Params p) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* w_st = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  const int tid = threadIdx.x;
  const int wid = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int lane = tid & 31;
  // the filter, split hi | lo, in the K-major SWIZZLE_128B image the MMA reads (K padded with zeros)
  for (int i = tid; i < kS7KB * 64 * 8; i += kS7Threads) {
    const int c = i & 7, row = (i >> 3) & 63, kb = i >> 9;
    float4 x;
    float* xp = reinterpret_cast<float*>(&x);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = kb * 32 + c * 4 + q;
      xp[q] = k < kS7K ? __ldg(p.filter + row * kS7K + k) : 0.0f;
    }
    float4 hh, ll;
    split4(x, &hh, &ll);
    float4* cell = reinterpret_cast<float4*>(w_st + kb * 2 * kS7WTile + row * 128 + ((c ^ (row & 7)) << 4));
    *cell = hh;
    *(cell + kS7WTile / 16) = ll;
  }
  fence_proxy_async();
  __syncthreads();

  const int g = lane >> 2, t = lane & 3;
  const int r0 = (wid & 3) * 16 + g;   // rows r0 and r0 + 8 of a 64-pixel tile
  const int row_pitch = p.W * 3;
  const long long ohw = static_cast<long long>(p.OH) * p.OW;
  for (int it = blockIdx.x * 2 + (wid >> 2); it < p.m_tiles; it += gridDim.x * 2) {
    const float* base[2];
    uint32_t rowmask[2];
    int e_lo[2], e_hi[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long m = static_cast<long long>(it) * 64 + r0 + 8 * rr;
      const long long mm = m < p.M ? m : p.M - 1;          // rows past the end gather a valid pixel; never stored
      const int bi = static_cast<int>(mm / ohw);
      const int rem = static_cast<int>(mm - bi * ohw);
      const int oy = rem / p.OW, ox = rem - oy * p.OW;
      const int iy0 = oy * 2 - p.ph, ix0 = ox * 2 - p.pw;
      rowmask[rr] = 0;
#pragma unroll
      for (int fy = 0; fy < 7; ++fy)
        if (static_cast<unsigned>(iy0 + fy) < static_cast<unsigned>(p.H)) rowmask[rr] |= 1u << fy;
      e_lo[rr] = 3 * max(0, -ix0);
      e_hi[rr] = 3 * min(7, p.W - ix0);
      base[rr] = p.in + ((static_cast<long long>(bi) * p.H + iy0) * p.W + ix0) * 3;
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll 1
    for (int kb = 0; kb < kS7KB; ++kb) {
      uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
      for (int k8 = 0; k8 < 4; ++k8)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int rr = r & 1;
          const int k = kb * 32 + 8 * k8 + t + 4 * (r >> 1);
          const int fy = k / 21, e = k - fy * 21;
          float x = 0.0f;
          if (k < kS7K && ((rowmask[rr] >> fy) & 1u) && e >= e_lo[rr] && e < e_hi[rr]) x = __ldg(base[rr] + fy * row_pitch + e);
          const float h = to_tf32(x);
          a_hi[k8][r] = __float_as_uint(h);
          a_lo[k8][r] = __float_as_uint(to_tf32(x - h));
        }
      tf32_3pass<kS7N>(acc, a_hi, a_lo, sdesc_lo(smem_u32(w_st + kb * 2 * kS7WTile)), kS7WTile, kb == 0);
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long m = static_cast<long long>(it) * 64 + r0 + 8 * rr;
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < kS7N / 8; ++j) {
        const int n = 8 * j + 2 * t;
        float y[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float bi = p.bias ? __ldg(p.bias + n + e) : 0.f;
          y[e] = apply_act(__fadd_rn(acc[4 * j + 2 * rr + e], bi), p.act);
        }
        *reinterpret_cast<float2*>(p.out + m * kS7N + n) = make_float2(y[0], y[1]);
      }
    }
  }
}

}  // namespace pw
}  // namespace lce

#endif  // LCE_B200_PW_CUH_
