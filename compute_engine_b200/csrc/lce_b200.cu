// lce_b200.cu -- implementation of the C-ABI CUDA layer declared in
// include/lce_b200.h. Host-side logic restates what the reference's op shell
// does around its kernels (LCE = /root/reference/larq_compute_engine):
//   shape inference          LCE/tflite/kernels/bconv2d.cc:169-248,
//                            tensorflow/lite/kernels/padding.h:32-82
//   output-transform fold    LCE/tflite/kernels/bconv2d.cc:353-389 (in double, on the host)
// and launches the kernels of lce_b200_kernels.cuh. There is no CPU compute path.
#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "lce_b200.h"
#include "lce_b200_kernels.cuh"
#include "lce_b200_imma.cuh"
#include "lce_b200_pair.cuh"
#include "lce_b200_tc.cuh"
#include "lce_b200_pw.cuh"

namespace {
thread_local std::string g_err;
std::atomic<uint64_t> g_launches{0};
std::atomic<uint64_t> g_path[3] = {};   // inner-product launches: wgmma / mma.sync / XOR + POPC
}  // namespace

// shared with lce_b200_builtins.cu
namespace lce_b200_internal {
int fail(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return 1;
}
int launch_check(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("launch of %s failed: %s", what, cudaGetErrorString(e));
  return 0;
}
}  // namespace lce_b200_internal
using lce_b200_internal::fail;
using lce_b200_internal::launch_check;

namespace {

#define CUDA_OK(expr)                                                            \
  do {                                                                           \
    cudaError_t e__ = (expr);                                                    \
    if (e__ != cudaSuccess)                                                      \
      return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

inline cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }
// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: one flag per (kernel
// instantiation, device), so a process that drives several GPUs raises the limit on each of them.
struct PerDeviceOnce {
  bool done[64] = {};
  bool need() {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return true;
    if (done[dev]) return false;
    done[dev] = true;
    return true;
  }
};
// per-channel vectors (multiplier, bias, thresholds) are padded by one widest channel tile
constexpr int kChanPad = 128;
inline int cdiv(int a, int b) { return (a + b - 1) / b; }

int grid_for(long long work_items, int per_block, int max_blocks = 132 * 16) {
  long long b = (work_items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return static_cast<int>(b);
}

// tensorflow/lite/kernels/padding.h:42-60
int out_size(int padding, int image, int filter, int stride, int dil) {
  const int eff = (filter - 1) * dil + 1;
  if (stride == 0) return 0;
  if (padding == LCE_PADDING_SAME) return (image + stride - 1) / stride;
  if (padding == LCE_PADDING_VALID) return (image + stride - eff) / stride;
  return 0;
}
// tensorflow/lite/kernels/padding.h:32-40
int pad_before(int stride, int dil, int in, int filter, int out) {
  const int eff = (filter - 1) * dil + 1;
  int total = (out - 1) * stride + eff - in;
  if (total < 0) total = 0;
  return total / 2;
}

bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// Copy `bytes` from a host-or-device pointer into fresh device memory of
// `alloc_bytes` (zero padded).
int to_device(const void* src, size_t bytes, size_t alloc_bytes, void** dst) {
  CUDA_OK(cudaMalloc(dst, alloc_bytes));
  CUDA_OK(cudaMemset(*dst, 0, alloc_bytes));
  if (bytes)
    CUDA_OK(cudaMemcpy(*dst, src, bytes,
                       is_device_ptr(src) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  return 0;
}
int to_host(const void* src, size_t bytes, void* dst) {
  CUDA_OK(cudaMemcpy(dst, src, bytes,
                     is_device_ptr(src) ? cudaMemcpyDeviceToHost : cudaMemcpyHostToHost));
  return 0;
}

// The part of a plan that the implicit-GEMM kernel needs, shared by LceBconv2d
// and the plain BGEMM.
struct GemmCore {
  int V = 1;            // words per smem vector (largest of 4,2,1 dividing Cw_pg)
  int Cw_pg = 0, taps = 1, Kv = 0, Kc_v = 0, n_chunks = 1;
  int cout = 0, cout_pg = 0, groups = 1, tiles_per_group = 1;
  int out_type = LCE_OUT_FLOAT;
  int clamp_min = 0, clamp_max = 0;
  int32_t* wt = nullptr;        // tiled weights
  float* mul = nullptr;         // folded, padded
  float* bias = nullptr;
  int32_t* thr = nullptr;
  int32_t* tap_popc = nullptr;  // zero-padding correction table
  size_t smem_bytes = 0;
  // mma.sync inner product (lce_b200_imma.cuh); absent when LCE_B200_BCONV_IMMA=0 or ineligible
  int32_t* wt_nat = nullptr;    // weights in mma B-fragment order: packed b1, or expanded to int8
  int32_t* wpop = nullptr;      // popcount of each channel's filter row (padded by BN)
  bool imma_b1 = false;         // b1 fragments (default) or int8 ones (LCE_B200_BCONV_B1=0)
  bool imma_win = false;        // b1 group windows: groups of 32 * odd output channels (GW)
  // a 32-channel layer the pair kernel takes: its b1 fragments for that kernel alone (wpop filled
  // too); the plan's own launches stay on the kernels below, which take every other channel count
  int32_t* pair_wt = nullptr;
  int imma_Kc_v = 0, imma_chunks = 1;
  size_t imma_smem = 0;
  // wgmma inner product (lce_b200_tc.cuh); absent when LCE_B200_BCONV_TC=0 or ineligible
  bool tc_ok = false;
  uint8_t* tc_wt = nullptr;        // [n_tiles][S_t][BN x 128 B] int8 stage images
  int32_t* tc_wpop2 = nullptr;     // 2 * popcount of each filter row, padded
  int32_t* tc_tap_popc_t = nullptr;  // [taps][ldc], zero-padding correction
  float* tc_zpc_cache = nullptr;     // [4][eff_h][eff_w][ldc], the optimised kernels' float corrections
  int tc_BN = 0, tc_n_tiles = 0, tc_CcB = 0, tc_n_chunks = 1, tc_flat = 0, tc_V = 1;
  int tc_S_full = 0, tc_S_last = 0, tc_S_t = 0, tc_ldc = 0;
  // shape-dependent part, cached per input shape
  long long tc_key_M = -1;
  int tc_key_H = 0, tc_key_W = 0, tc_max_px = 0;

  void release() {
    cudaFree(wt); cudaFree(mul); cudaFree(bias); cudaFree(thr); cudaFree(tap_popc);
    cudaFree(wt_nat); cudaFree(wpop); cudaFree(pair_wt);
    cudaFree(tc_wt); cudaFree(tc_wpop2); cudaFree(tc_tap_popc_t); cudaFree(tc_zpc_cache);
    wt = wt_nat = wpop = pair_wt = nullptr; mul = bias = nullptr; thr = tap_popc = nullptr;
    tc_wt = nullptr; tc_wpop2 = tc_tap_popc_t = nullptr; tc_zpc_cache = nullptr; tc_ok = false;
  }
};

// Dynamic shared memory one CTA may use so that kCtasPerSm CTAs stay resident on an SM
// (227 KB per SM, 1 KB reserved per CTA, a little static shared memory).
size_t cta_smem_budget() {
  return (227u * 1024u / lce::kCtasPerSm - 1024u - 256u) & ~size_t{127};
}

template <int V, int OUT>
int launch_conv_vo(const lce::ConvKParams& p, dim3 grid, size_t smem, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(lce::bconv_kernel<V, OUT>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(cta_smem_budget())));
  lce::bconv_kernel<V, OUT><<<grid, lce::kThreads, smem, s>>>(p);
  g_path[2].fetch_add(1, std::memory_order_relaxed);
  return launch_check("bconv_kernel");
}
size_t imma_smem_budget(int V, bool b1) {
  const int ctas = b1 ? lce::kB1SmemCtas : lce::imma_ctas_per_sm(V);
  return (227u * 1024u / ctas - 1024u - 256u) & ~size_t{127};
}

template <int V, int OUT, bool B1, bool CHAIN = false, bool GATE = false, bool SLICE = false,
          bool SPATIAL = false, bool GW = false, bool SHUFFLE = false, bool FCMAX = false>
int launch_imma_vo(const lce::ConvKParams& p, dim3 grid, size_t smem, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(lce::bconv_imma_kernel<V, OUT, B1, CHAIN, GATE, SLICE, SPATIAL, GW, SHUFFLE, FCMAX>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(imma_smem_budget(V, B1))));
  lce::bconv_imma_kernel<V, OUT, B1, CHAIN, GATE, SLICE, SPATIAL, GW, SHUFFLE, FCMAX>
      <<<grid, lce::kIThreads, smem, s>>>(p);
  g_path[1].fetch_add(1, std::memory_order_relaxed);
  return launch_check("bconv_imma_kernel");
}
// Epilogue tails of the float output beyond run_fused's (bconv_run_impl decides).
// kScale: p.gate indexed by position within the image (lce_b200_bconv2d_run_fused_scale)
// kShuffle: the pixel-shuffled store of lce_b200_bconv2d_run_fused_shuffle (p.shuf_*), b1 only
// kFcMax: lce_b200_bconv2d_run_fused_fc_max's per-image column max (p.shuf_*, p.max_keys), b1 only
enum class Tail { kNone, kChain, kGate, kScale, kSlice, kShuffle, kFcMax };   // p.chain / p.gate / p.out_stride in the epilogue

// group-window plans (b1 only): every tail but the slice store
template <int V>
int launch_imma_win_v(int out_type, Tail tail, const lce::ConvKParams& p, dim3 grid, size_t smem,
                      cudaStream_t s) {
  constexpr int F = LCE_OUT_FLOAT;
  switch (tail) {
    case Tail::kChain: return launch_imma_vo<V, F, true, true, false, false, false, true>(p, grid, smem, s);
    case Tail::kGate: return launch_imma_vo<V, F, true, false, true, false, false, true>(p, grid, smem, s);
    case Tail::kScale: return launch_imma_vo<V, F, true, false, true, false, true, true>(p, grid, smem, s);
    case Tail::kSlice: return fail("bconv2d: the slice store takes no grouped plan with 32 * odd channels per group");
    case Tail::kShuffle:
    case Tail::kFcMax: return fail("bconv2d: the shuffle store takes no grouped plan");
    case Tail::kNone: break;
  }
  if (out_type == LCE_OUT_BITPACKED)
    return launch_imma_vo<V, LCE_OUT_BITPACKED, true, false, false, false, false, true>(p, grid, smem, s);
  return launch_imma_vo<V, F, true, false, false, false, false, true>(p, grid, smem, s);
}

template <int V>
int launch_imma_v(int out_type, bool b1, Tail tail, const lce::ConvKParams& p, dim3 grid,
                  size_t smem, cudaStream_t s) {
  if (tail == Tail::kChain) {
    if (b1) return launch_imma_vo<V, LCE_OUT_FLOAT, true, true>(p, grid, smem, s);
    return launch_imma_vo<V, LCE_OUT_FLOAT, false, true>(p, grid, smem, s);
  }
  if (tail == Tail::kGate) {
    if (b1) return launch_imma_vo<V, LCE_OUT_FLOAT, true, false, true>(p, grid, smem, s);
    return launch_imma_vo<V, LCE_OUT_FLOAT, false, false, true>(p, grid, smem, s);
  }
  if (tail == Tail::kScale) {
    if (b1) return launch_imma_vo<V, LCE_OUT_FLOAT, true, false, true, false, true>(p, grid, smem, s);
    return launch_imma_vo<V, LCE_OUT_FLOAT, false, false, true, false, true>(p, grid, smem, s);
  }
  if (tail == Tail::kSlice) {
    if (b1) return launch_imma_vo<V, LCE_OUT_FLOAT, true, false, false, true>(p, grid, smem, s);
    return launch_imma_vo<V, LCE_OUT_FLOAT, false, false, false, true>(p, grid, smem, s);
  }
  if (tail == Tail::kShuffle) {
    if (!b1) return fail("bconv2d: the shuffle store needs the b1 inner product");
    return launch_imma_vo<V, LCE_OUT_FLOAT, true, false, false, false, false, false, true>(p, grid, smem, s);
  }
  if (tail == Tail::kFcMax) {
    if (!b1) return fail("bconv2d: the max epilogue needs the b1 inner product");
    return launch_imma_vo<V, LCE_OUT_FLOAT, true, false, false, false, false, false, false, true>(p, grid, smem, s);
  }
  if (b1) {
    if (out_type == LCE_OUT_FLOAT) return launch_imma_vo<V, LCE_OUT_FLOAT, true>(p, grid, smem, s);
    if (out_type == LCE_OUT_BITPACKED) return launch_imma_vo<V, LCE_OUT_BITPACKED, true>(p, grid, smem, s);
    return launch_imma_vo<V, LCE_OUT_RAW_ACC, true>(p, grid, smem, s);
  }
  if (out_type == LCE_OUT_FLOAT) return launch_imma_vo<V, LCE_OUT_FLOAT, false>(p, grid, smem, s);
  if (out_type == LCE_OUT_BITPACKED) return launch_imma_vo<V, LCE_OUT_BITPACKED, false>(p, grid, smem, s);
  return launch_imma_vo<V, LCE_OUT_RAW_ACC, false>(p, grid, smem, s);
}

template <int V>
int launch_conv_v(int out_type, const lce::ConvKParams& p, dim3 grid, size_t smem,
                  cudaStream_t s) {
  switch (out_type) {
    case LCE_OUT_FLOAT: return launch_conv_vo<V, LCE_OUT_FLOAT>(p, grid, smem, s);
    case LCE_OUT_INT8: return launch_conv_vo<V, LCE_OUT_INT8>(p, grid, smem, s);
    case LCE_OUT_BITPACKED: return launch_conv_vo<V, LCE_OUT_BITPACKED>(p, grid, smem, s);
    case LCE_OUT_RAW_ACC: return launch_conv_vo<V, LCE_OUT_RAW_ACC>(p, grid, smem, s);
  }
  return fail("unsupported output type %d", out_type);
}
int tc_launch(GemmCore& c, const lce::ConvKParams& p, cudaStream_t s);

// The plan's output goes through the mma.sync kernel (launch_conv's first choice).
bool takes_imma(const GemmCore& c, const lce::ConvKParams& p) { return c.wt_nat != nullptr && p.vec_store; }

int launch_conv(GemmCore& c, lce::ConvKParams& p, cudaStream_t s, Tail tail = Tail::kNone) {
  p.fd_ohw = lce::make_fastdiv(static_cast<uint32_t>(p.OH) * p.OW);
  p.fd_ow = lce::make_fastdiv(p.OW);
  p.fd_cwv = lce::make_fastdiv(p.CwV);
  p.fd_kw = lce::make_fastdiv(p.KW);
  p.fd_tpg = lce::make_fastdiv(p.tiles_per_group);
  p.img_words = static_cast<long long>(p.H) * p.W * p.Cw_total;
  if (p.M <= 0) return 0;  // empty batch: nothing to do
  const long long m_tiles = (p.M + lce::kBM - 1) / lce::kBM;
  if (m_tiles > INT_MAX) return fail("too many output pixels");
  if (p.img_words >= (1LL << 31)) return fail("input image too large (>= 2^31 packed words)");
  // Which inner product: on H100 the mma.sync kernel (native b1 BMMA, or int8 fragments with
  // LCE_B200_BCONV_B1=0) runs the QuickNet graph faster than the wgmma kernel (bench.py reports
  // both in one run), so it takes every plan it can (full 64-channel tiles, float, bitpacked or
  // raw-accumulator output); the wgmma kernel takes the rest it is eligible for (int8 outputs,
  // other channel counts), XOR + POPC what is left. All produce the same int32 accumulators.
  if (takes_imma(c, p)) {
    // mma.sync inner product: 128 x 64 tiles, the same int32 accumulators as bconv_kernel
    lce::ConvKParams q = p;
    q.wt = c.wt_nat; q.wpop = c.wpop;
    q.Kc_v = c.imma_Kc_v; q.n_chunks = c.imma_chunks;
    q.res_stage = 0;
    const size_t ismem = c.imma_smem;
    dim3 igrid(static_cast<unsigned>((p.M + lce::kIBM - 1) / lce::kIBM),
               static_cast<unsigned>(c.groups * c.tiles_per_group));
    if (c.imma_win) {
      // K = taps x the window's two groups of input words; 64-channel tiles over all channels
      q.Kv = 2 * p.Kv;
      q.CwV = 2 * p.CwV;
      q.fd_cwv = lce::make_fastdiv(q.CwV);
      q.win_step = 8 % (2 * c.Cw_pg);
      igrid.y = static_cast<unsigned>(cdiv(c.cout, lce::kBN));
      switch (c.V) {
        case 4: return launch_imma_win_v<4>(c.out_type, tail, q, igrid, ismem, s);
        case 2: return launch_imma_win_v<2>(c.out_type, tail, q, igrid, ismem, s);
        default: return launch_imma_win_v<1>(c.out_type, tail, q, igrid, ismem, s);
      }
    }
    switch (c.V) {
      case 4: return launch_imma_v<4>(c.out_type, c.imma_b1, tail, q, igrid, ismem, s);
      case 2: return launch_imma_v<2>(c.out_type, c.imma_b1, tail, q, igrid, ismem, s);
      default: return launch_imma_v<1>(c.out_type, c.imma_b1, tail, q, igrid, ismem, s);
    }
  }
  if (tail != Tail::kNone)
    return fail("bconv2d: the chain, gate, scale, slice and shuffle epilogues need the mma.sync kernel");
  if (c.tc_ok) {
    // wgmma inner product: persistent 128 x BN tiles
    const int rc = tc_launch(c, p, s);
    if (rc >= 0) return rc;
  }
  dim3 grid(static_cast<unsigned>(m_tiles), static_cast<unsigned>(c.groups * c.tiles_per_group));
  const size_t smem = c.smem_bytes + (p.res_stage ? lce::kResStageBytes : 0);
  switch (c.V) {
    case 4: return launch_conv_v<4>(c.out_type, p, grid, smem, s);
    case 2: return launch_conv_v<2>(c.out_type, p, grid, smem, s);
    default: return launch_conv_v<1>(c.out_type, p, grid, smem, s);
  }
}


// ------------------------------------------------------------------------- //
// wgmma path (lce_b200_tc.cuh): plan-time weight images and the launch.
// ------------------------------------------------------------------------- //
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder() {
  static EncodeTiledFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess) {
      cudaGetLastError();
      f = nullptr;
    }
    return reinterpret_cast<EncodeTiledFn>(f);
  }();
  return fn;
}
int num_sms() {
  static int cache[64] = {};
  int dev = 0, v = 132;
  cudaGetDevice(&dev);
  if (dev >= 0 && dev < 64 && cache[dev]) return cache[dev];
  cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
  if (dev >= 0 && dev < 64) cache[dev] = v;
  return v;
}
constexpr size_t kTcSmemBudget = 226u * 1024u;   // dynamic shared memory of the one CTA per SM

bool tc_enabled() {
  const char* e = getenv("LCE_B200_BCONV_TC");  // read per plan: A/B in one process
  return !(e && e[0] == '0');
}

// Weight stage images, 2 * popc(filter row) and the transposed tap popcounts. Eligibility that
// does not depend on the input shape is decided here; the rest in tc_launch.
int build_tc_weights(GemmCore* c, const int32_t* d_filter, bool want_tap_popc) {
  c->tc_ok = false;
  if (!tc_enabled() || c->groups != 1 || tensor_map_encoder() == nullptr) return 0;
  if ((c->out_type == LCE_OUT_FLOAT || c->out_type == LCE_OUT_RAW_ACC) && (c->cout % 4 != 0 || c->cout < 32))
    return 0;  // two-channel stores, 32-channel sign words
  if (want_tap_popc && c->taps > 64) return 0;
  const int Cw = c->Cw_pg;
  // 64-channel tiles: their kernel fits two CTAs per SM (128-channel tiles need too many registers)
  c->tc_BN = c->cout > 32 ? 64 : 32;
  c->tc_n_tiles = cdiv(c->cout, c->tc_BN);
  if (Cw % 4 == 0) {
    c->tc_flat = 0; c->tc_V = 4;
    c->tc_CcB = std::min(Cw, 32);   // halo stage = pixels x 128 B at most
  } else {
    c->tc_flat = 1; c->tc_V = (Cw % 2 == 0) ? 2 : 1;
    c->tc_CcB = Cw;
    if (Cw > 64) return 0;
  }
  c->tc_n_chunks = cdiv(Cw, c->tc_CcB);
  const int cc_last = Cw - (c->tc_n_chunks - 1) * c->tc_CcB;
  c->tc_S_full = cdiv(c->taps * c->tc_CcB, lce::tc::kWS);
  c->tc_S_last = cdiv(c->taps * cc_last, lce::tc::kWS);
  c->tc_S_t = (c->tc_n_chunks - 1) * c->tc_S_full + c->tc_S_last;
  c->tc_ldc = c->tc_n_tiles * c->tc_BN;
  const long long units = static_cast<long long>(c->tc_n_tiles) * c->taps * Cw * c->tc_BN;
  CUDA_OK(cudaMalloc(&c->tc_wt, static_cast<size_t>(units) * 32));
  lce::tc::expand_weights_tc_kernel<<<grid_for(units, 256, 1 << 22), 256>>>(
      d_filter, c->tc_wt, c->cout, c->taps, Cw, c->tc_CcB, c->tc_BN, units);
  if (launch_check("expand_weights_tc_kernel")) return 1;
  CUDA_OK(cudaMalloc(&c->tc_wpop2, static_cast<size_t>(c->tc_ldc) * 4));
  CUDA_OK(cudaMemset(c->tc_wpop2, 0, static_cast<size_t>(c->tc_ldc) * 4));
  lce::tc::wpop2_kernel<<<cdiv(c->cout, 256), 256>>>(d_filter, c->tc_wpop2, c->cout, c->taps * Cw);
  if (launch_check("wpop2_kernel")) return 1;
  if (want_tap_popc) {
    const size_t n = static_cast<size_t>(c->taps) * c->tc_ldc;
    CUDA_OK(cudaMalloc(&c->tc_tap_popc_t, n * 4));
    CUDA_OK(cudaMemset(c->tc_tap_popc_t, 0, n * 4));
    lce::tc::tap_popc_t_kernel<<<cdiv(c->cout * c->taps, 256), 256>>>(d_filter, c->tc_tap_popc_t, c->cout, c->taps,
                                                                       Cw, c->tc_ldc);
    if (launch_check("tap_popc_t_kernel")) return 1;
  }
  c->tc_ok = true;
  return 0;
}

// Largest halo (input pixels touched by one 128-pixel tile) over all tiles of this shape: the same
// arithmetic as lce::tc::tile_halo, run once per (plan, input shape).
int tc_max_halo_px(const lce::ConvKParams& p) {
  long long best = 1;
  const long long ohw = static_cast<long long>(p.OH) * p.OW;
  const long long total_px = (p.M / ohw) * p.H * p.W;
  auto flat = [&](long long m, int fy, int fx) {
    const long long b = m / ohw, r = m - b * ohw;
    const long long oy = r / p.OW, ox = r - oy * p.OW;
    return (b * p.H + (oy * p.sh - p.ph + fy * p.dh)) * p.W + (ox * p.sw - p.pw + fx * p.dw);
  };
  for (long long m0 = 0; m0 < p.M; m0 += lce::tc::kBM) {
    const long long m1 = std::min<long long>(m0 + lce::tc::kBM, p.M) - 1;
    long long lo = std::max<long long>(flat(m0, 0, 0), 0);
    const long long hi = std::min<long long>(flat(m1, p.KH - 1, p.KW - 1) + 1, total_px);
    if (lo > total_px - 1) lo = total_px - 1;
    best = std::max(best, std::max<long long>(hi - lo, 1));
  }
  return static_cast<int>(std::min<long long>(best, INT_MAX));
}

template <int V, int OUT, int BN>
int launch_tc_vob(const CUtensorMap& tm_in, const lce::tc::TcParams& t, int grid, size_t smem, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(lce::tc::bconv_tc_kernel<V, OUT, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kTcSmemBudget)));
  lce::tc::bconv_tc_kernel<V, OUT, BN><<<grid, lce::tc::kThreads, smem, s>>>(tm_in, t);
  g_path[0].fetch_add(1, std::memory_order_relaxed);
  return launch_check("bconv_tc_kernel");
}
template <int V, int OUT>
int launch_tc_vo(const CUtensorMap& tm_in, const lce::tc::TcParams& t, int grid, size_t smem, cudaStream_t s) {
  switch (t.BN) {
    case 64: return launch_tc_vob<V, OUT, 64>(tm_in, t, grid, smem, s);
    default: return launch_tc_vob<V, OUT, 32>(tm_in, t, grid, smem, s);
  }
}
template <int V>
int launch_tc_v(int out_type, const CUtensorMap& tm_in, const lce::tc::TcParams& t, int grid, size_t smem, cudaStream_t s) {
  switch (out_type) {
    case LCE_OUT_FLOAT: return launch_tc_vo<V, LCE_OUT_FLOAT>(tm_in, t, grid, smem, s);
    case LCE_OUT_INT8: return launch_tc_vo<V, LCE_OUT_INT8>(tm_in, t, grid, smem, s);
    case LCE_OUT_BITPACKED: return launch_tc_vo<V, LCE_OUT_BITPACKED>(tm_in, t, grid, smem, s);
    default: return launch_tc_vo<V, LCE_OUT_RAW_ACC>(tm_in, t, grid, smem, s);
  }
}

// Returns -1 when this launch is not eligible (the caller falls through to the mma.sync / XOR
// kernels), else the launch status.
int tc_launch(GemmCore& c, const lce::ConvKParams& p, cudaStream_t s) {
  namespace T = lce::tc;
  if (!c.tc_ok || p.M >= (1LL << 31)) return -1;
  const long long ohw = static_cast<long long>(p.OH) * p.OW;
  const long long batch = p.M / ohw;
  const long long total_px = batch * p.H * p.W;
  const long long total_words = total_px * p.Cw_total;
  if (total_words >= (1LL << 31) || total_px < 1) return -1;
  if ((reinterpret_cast<uintptr_t>(p.in) & 15u) != 0) return -1;
  // the epilogue stores two channels at a time
  if ((reinterpret_cast<uintptr_t>(p.out) & 7u) != 0) return -1;
  if (p.residual != nullptr && (reinterpret_cast<uintptr_t>(p.residual) & 7u) != 0) return -1;
  if (c.tc_key_M != p.M || c.tc_key_H != p.H || c.tc_key_W != p.W) {
    c.tc_max_px = tc_max_halo_px(p);
    c.tc_key_M = p.M; c.tc_key_H = p.H; c.tc_key_W = p.W;
  }
  T::TcParams t;
  memset(&t, 0, sizeof(t));
  t.M = p.M; t.total_px = total_px;
  t.H = p.H; t.W = p.W; t.OH = p.OH; t.OW = p.OW; t.KH = p.KH; t.KW = p.KW;
  t.sh = p.sh; t.sw = p.sw; t.dh = p.dh; t.dw = p.dw; t.ph = p.ph; t.pw = p.pw;
  t.taps = p.KH * p.KW;
  t.Cw = c.Cw_pg; t.CcB = c.tc_CcB; t.n_chunks = c.tc_n_chunks; t.mode_flat = c.tc_flat;
  t.cout = c.cout; t.BN = c.tc_BN; t.n_tiles = c.tc_n_tiles;
  t.m_tiles = static_cast<int>((p.M + T::kBM - 1) / T::kBM);
  t.S_full = c.tc_S_full; t.S_last = c.tc_S_last; t.S_t = c.tc_S_t;
  // shared memory: weights | halo stages | barriers
  size_t raw_stage;
  if (c.tc_flat) raw_stage = static_cast<size_t>(cdiv(c.tc_max_px * c.Cw_pg + 3, 256)) * 1024;
  else raw_stage = static_cast<size_t>(cdiv(c.tc_max_px, 128)) * 128 * c.tc_CcB * 4;
  raw_stage = (raw_stage + 1023) & ~size_t{1023};
  t.raw_stage_bytes = static_cast<int>(raw_stage);
  const size_t stage_bytes = static_cast<size_t>(c.tc_BN) * 32 * T::kWS;     // one ring slot
  const size_t resident_bytes = static_cast<size_t>(c.tc_BN) * 32 * t.taps * c.Cw_pg;  // all K words, dense
  const size_t fixed = T::kNR * raw_stage + T::kBarBytes;
  // two CTAs per SM where a layout fits half the shared memory, else one with all of it
  constexpr size_t kHalfBudget = (227u * 1024u / 2 - 1024u) & ~size_t{1023};
  const int ctas = fixed + 2 * stage_bytes <= kHalfBudget ? 2 : 1;
  const size_t budget = ctas == 2 ? kHalfBudget : kTcSmemBudget;
  if (fixed + 2 * stage_bytes > budget) return -1;
  const size_t room = budget - fixed;
  size_t b_bytes;
  if (c.tc_n_tiles == 1 && c.tc_S_t <= T::kMaxNB && room >= ((resident_bytes + 1023) & ~size_t{1023})) {
    t.b_resident = 1;
    t.nB = c.tc_S_t;
    b_bytes = (resident_bytes + 1023) & ~size_t{1023};
  } else {
    // the weights stream through a ring of as many stages as fit (2 .. kMaxRing)
    t.b_resident = 0;
    t.nB = static_cast<int>(std::min<size_t>(T::kMaxRing, room / stage_bytes));
    b_bytes = t.nB * stage_bytes;
  }
  t.Kw_total = t.taps * c.Cw_pg;
  t.off_raw = static_cast<int>(b_bytes);
  t.off_bar = t.off_raw + T::kNR * t.raw_stage_bytes;
  const size_t smem = static_cast<size_t>(t.off_bar) + T::kBarBytes;
  t.clamp_min = p.clamp_min; t.clamp_max = p.clamp_max;
  t.has_res = p.residual != nullptr ? 1 : 0; t.residual_act = p.residual_act;
  t.cw_out = p.cw_out; t.zp_half = p.zp_half; t.ldc = c.tc_ldc;
  t.wt = c.tc_wt; t.mul = p.mul; t.bias = p.bias; t.wpop2 = c.tc_wpop2; t.thr = p.thr;
  t.tap_popc_t = p.tap_popc != nullptr ? c.tc_tap_popc_t : nullptr;
  t.zp_float = p.zp_float; t.cin_pg = p.cin_pg;
  t.zpc_cache = c.tc_zpc_cache;
  if (t.zp_float && t.zpc_cache == nullptr) return -1;
  t.residual = p.residual;
  t.out = p.out; t.packed_out = p.packed_out;
  t.fd_ohw = lce::make_fastdiv(static_cast<uint32_t>(ohw));
  t.fd_ow = lce::make_fastdiv(p.OW);
  t.fd_kw = lce::make_fastdiv(p.KW);
  t.fd_mt = lce::make_fastdiv(t.m_tiles);

  EncodeTiledFn enc = tensor_map_encoder();
  CUtensorMap tm_in;
  cuuint32_t es[2] = {1, 1};
  if (c.tc_flat) {
    cuuint64_t gd[1] = {static_cast<cuuint64_t>(total_words)};
    cuuint64_t gs[1] = {0};
    cuuint32_t box[1] = {256};
    if (enc(&tm_in, CU_TENSOR_MAP_DATA_TYPE_INT32, 1, const_cast<int32_t*>(p.in), gd, gs, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail("cuTensorMapEncodeTiled (activations, flat) failed");
  } else {
    cuuint64_t gd[2] = {static_cast<cuuint64_t>(p.Cw_total), static_cast<cuuint64_t>(total_px)};
    cuuint64_t gs[1] = {static_cast<cuuint64_t>(p.Cw_total) * 4};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(c.tc_CcB), 128};
    if (enc(&tm_in, CU_TENSOR_MAP_DATA_TYPE_INT32, 2, const_cast<int32_t*>(p.in), gd, gs, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail("cuTensorMapEncodeTiled (activations) failed");
  }
  const long long items = static_cast<long long>(t.n_tiles) * t.m_tiles;
  const int grid = static_cast<int>(std::min<long long>(items, static_cast<long long>(ctas) * num_sms()));
  switch (c.tc_V) {
    case 4: return launch_tc_v<4>(c.out_type, tm_in, t, grid, smem, s);
    case 2: return launch_tc_v<2>(c.out_type, tm_in, t, grid, smem, s);
    default: return launch_tc_v<1>(c.out_type, tm_in, t, grid, smem, s);
  }
}

// fp32 pointwise convolution on the tensor cores (lce_b200_pw.cuh), called by the CONV_2D builtin
// (lce_b200_builtins.cu). 0 = launched, -1 = shape not eligible (the caller's FMA kernels take
// it), > 0 = error.
std::atomic<uint64_t> g_pw_launches{0};
}  // namespace
namespace lce_b200_internal {
int pw_tf32_conv(const float* in, const float* filter, const float* bias, float* out, int32_t* packed, long long M, int N,
                 int K, int act, int pairs_ok, void* stream) {
  static const bool enabled = [] { const char* e = getenv("LCE_B200_PW_TF32"); return !(e && e[0] == '0'); }();
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enabled || enc == nullptr) return -1;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(filter) | reinterpret_cast<uintptr_t>(out) |
       reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(packed)) & 15)
    return -1;
  // Which kernel runs must not depend on the batch (an image's result must not change with its
  // batch mates): eligibility looks at the layer's shape only; `pairs_ok` = even pixels per image.
  const bool pairs = K == 16 && N == 64 && pairs_ok && (M & 1) == 0;
  // N: whole 128-column tiles, or (no packed output) any multiple of 4 -- TMA zero-fills the filter
  // rows past N and the stores are guarded by n < N (FULLY_CONNECTED's 1000 logits)
  if (!pairs && ((K & 31) != 0 || K > 4096 || (N & 3) != 0 || ((N & 127) != 0 && packed != nullptr))) return -1;
  namespace P = lce::pw;
  P::PwParams p{};
  p.M = pairs ? M / 2 : M;
  p.N = pairs ? 128 : N;
  p.KB = pairs ? 1 : K / 32;
  p.n_tiles = (p.N + 127) / 128;
  const long long m_tiles = (p.M + 127) / 128;
  if (m_tiles > (1 << 22)) return -1;
  p.m_tiles = static_cast<int>(m_tiles);
  p.act = act;
  p.pairs = pairs ? 1 : 0;
  p.w_resident = (p.n_tiles == 1 && p.KB <= P::kPwNS) ? 1 : 0;
  p.bias_mask = pairs ? 63 : 0x7fffffff;
  p.filter = filter;
  p.bias = bias;
  p.packed = packed;
  const int Kp = pairs ? 32 : K;
  CUtensorMap tm_a, tm_w;
  cuuint32_t es[2] = {1, 1};
  cuuint32_t box_ld[2] = {32, 128};
  {
    cuuint64_t gd[2] = {static_cast<cuuint64_t>(Kp), static_cast<cuuint64_t>(p.M)};
    cuuint64_t gs[1] = {static_cast<cuuint64_t>(Kp) * 4};
    if (enc(&tm_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(in), gd, gs, box_ld, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail("cuTensorMapEncodeTiled (pointwise input) failed");
  }
  tm_w = tm_a;
  if (!pairs) {
    cuuint64_t gd[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(N)};
    cuuint64_t gs[1] = {static_cast<cuuint64_t>(K) * 4};
    if (enc(&tm_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(filter), gd, gs, box_ld, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail("cuTensorMapEncodeTiled (pointwise filter) failed");
  }
  CUtensorMap tm_o;
  {
    // the output, stored by TMA from 64-row x 32-column SWIZZLE_128B staging boxes
    cuuint64_t gd[2] = {static_cast<cuuint64_t>(p.N), static_cast<cuuint64_t>(p.M)};
    cuuint64_t gs[1] = {static_cast<cuuint64_t>(p.N) * 4};
    cuuint32_t box_o[2] = {32, 64};
    if (enc(&tm_o, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, out, gd, gs, box_o, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail("cuTensorMapEncodeTiled (pointwise output) failed");
  }
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(P::pw_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P::kPwSmem)));
  const int grid = static_cast<int>(std::min<long long>(m_tiles * p.n_tiles, num_sms()));
  P::pw_tf32_kernel<<<grid, P::kPwThreads, P::kPwSmem, static_cast<cudaStream_t>(stream)>>>(tm_a, tm_w, tm_o, p);
  g_pw_launches.fetch_add(1, std::memory_order_relaxed);
  return launch_check("pw_tf32_kernel");
}
uint64_t pw_tf32_launches() { return g_pw_launches.load(); }
// CONV_2D 7x7 / stride 2 / 3 -> 64 (Bi-RealNet's stem) on wgmma tf32 (lce_b200_pw.cuh):
// 0 = launched, -1 = not this shape, > 0 = error.
int stem7_tf32_conv(const float* in, const float* filter, const float* bias, float* out, int B, int H, int W, int OH, int OW,
                    int ph, int pw, int act, void* stream) {
  static const bool enabled = [] { const char* e = getenv("LCE_B200_PW_TF32"); return !(e && e[0] == '0'); }();
  EncodeTiledFn enc = tensor_map_encoder();
  if (!enabled || enc == nullptr) return -1;
  if ((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(bias)) & 15) return -1;
  namespace P = lce::pw;
  P::Stem7Params p{};
  p.M = static_cast<long long>(B) * OH * OW;
  const long long m_tiles = (p.M + 63) / 64;
  if (m_tiles > (1 << 24)) return -1;
  p.H = H; p.W = W; p.OH = OH; p.OW = OW; p.ph = ph; p.pw = pw;
  p.m_tiles = static_cast<int>(m_tiles);
  p.act = act;
  p.in = in; p.filter = filter; p.bias = bias; p.out = out;
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(P::stem7_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(P::kS7Smem)));
  // two warpgroups per CTA, two CTAs per SM
  const int grid = static_cast<int>(std::min<long long>((m_tiles + 1) / 2, 2LL * num_sms()));
  P::stem7_tf32_kernel<<<grid, P::kS7Threads, P::kS7Smem, static_cast<cudaStream_t>(stream)>>>(p);
  g_pw_launches.fetch_add(1, std::memory_order_relaxed);
  return launch_check("stem7_tf32_kernel");
}
}  // namespace lce_b200_internal
namespace {

// A kernel-selection switch set to 0 (read per plan: A/B in one process)
bool env_off(const char* name) {
  const char* e = getenv(name);
  return e && e[0] == '0';
}

// Build the tiled weights (+ optional tap popcounts) from an OHWI-packed filter
// [cout][taps][Cw_pg] that may live on the host or the device. pair_b1: a 32-channel layer the
// pair kernel takes (pair_layer_refusal), which gets the pair kernel's fragments as well.
int build_core_weights(GemmCore* c, const int32_t* filter, bool want_tap_popc, bool pair_b1 = false) {
  const size_t filter_words = static_cast<size_t>(c->cout) * c->taps * c->Cw_pg;
  int32_t* d_filter = nullptr;
  const bool on_dev = is_device_ptr(filter);
  if (!on_dev) {
    void* tmp = nullptr;
    if (to_device(filter, filter_words * 4, filter_words * 4 + 16, &tmp)) return 1;
    d_filter = static_cast<int32_t*>(tmp);
  } else {
    d_filter = const_cast<int32_t*>(filter);
  }
  c->V = (c->Cw_pg % 4 == 0) ? 4 : (c->Cw_pg % 2 == 0) ? 2 : 1;
  const int CwV = c->Cw_pg / c->V;
  c->Kv = c->taps * CwV;
  const int max_kc_v = lce::kMaxChunkWords / c->V;
  c->n_chunks = cdiv(c->Kv, max_kc_v);
  c->Kc_v = cdiv(c->Kv, c->n_chunks);
  c->smem_bytes = static_cast<size_t>(c->Kc_v) * (lce::kBM + lce::kBN) * c->V * 4;
  c->tiles_per_group = cdiv(c->cout_pg, lce::kBN);
  const long long total = static_cast<long long>(c->groups) * c->tiles_per_group * c->Kv *
                          lce::kBN * c->V;
  CUDA_OK(cudaMalloc(&c->wt, total * 4));
  lce::tile_weights_kernel<<<grid_for(total, 256, 1 << 20), 256>>>(
      d_filter, c->wt, c->cout_pg, c->tiles_per_group, c->taps, c->Cw_pg, c->V, c->Kv, total, 0);
  if (launch_check("tile_weights_kernel")) return 1;
  // mma.sync inner product (lce_b200_imma.cuh) where a plan is eligible: full 64-channel
  // tiles, float, bitpacked or raw-accumulator output. LCE_B200_BCONV_IMMA=0 leaves every plan
  // to the wgmma / XOR + POPC kernels (bench.py reports both). LCE_B200_BCONV_B1=0 keeps the
  // int8 fragments instead of the packed b1 ones; both give the same accumulators.
  // Grouped plans with 32 * odd output channels per group take the b1 fragments over group
  // windows (bconv_imma_kernel's GW); with int8 fragments they stay on the kernels below.
  const bool imma_on = !env_off("LCE_B200_BCONV_IMMA") && c->out_type != LCE_OUT_INT8;
  c->imma_win = imma_on && c->groups > 1 && c->cout_pg % lce::kBN == 32 && !env_off("LCE_B200_BCONV_B1");
  if (imma_on && (c->cout_pg % lce::kBN == 0 || c->imma_win)) {
    const int Kw = c->taps * c->Cw_pg;
    c->imma_b1 = !env_off("LCE_B200_BCONV_B1");
    const size_t budget = imma_smem_budget(c->V, c->imma_b1);
    if (c->imma_b1) {
      const int win = c->imma_win ? 2 : 1;   // a group window holds two groups' words per tap
      const int n_slices = cdiv(win * Kw, 8);  // 8-word k-slices, the last one padded to 4 or 8 words
      const long long n_tiles = c->imma_win ? cdiv(c->cout, lce::kBN) : c->groups * c->tiles_per_group;
      const long long total = n_tiles * n_slices * 256;
      CUDA_OK(cudaMalloc(&c->wt_nat, total * 8));
      lce::pack_weights_b1_kernel<<<grid_for(total, 256, 1 << 22), 256>>>(
          d_filter, reinterpret_cast<uint2*>(c->wt_nat), c->cout_pg, c->tiles_per_group, win * Kw,
          n_slices, total, c->imma_win ? c->Cw_pg : 0, c->groups);
      if (launch_check("pack_weights_b1_kernel")) return 1;
      // K staging: one chunk when it fits kB1SmemCtas CTAs per SM, else a two-deep ring of
      // chunks of whole 8-word slices
      const int Kvp = lce::b1_padded_vectors(win * c->Kv, c->V);
      const size_t slice_bytes = lce::kB1BytesPerSlice;
      if (n_slices * slice_bytes <= budget) {
        c->imma_chunks = 1;
        c->imma_Kc_v = Kvp;
        c->imma_smem = n_slices * slice_bytes;
      } else {
        const int ring_slices = std::max(static_cast<int>(budget / (2 * slice_bytes)), 1);
        c->imma_chunks = cdiv(n_slices, ring_slices);
        const int chunk_slices = cdiv(n_slices, c->imma_chunks);
        c->imma_Kc_v = chunk_slices * 8 / c->V;
        c->imma_smem = 2 * chunk_slices * slice_bytes;
      }
    } else {
      const long long xtotal = static_cast<long long>(c->groups) * c->tiles_per_group * Kw * 256;
      CUDA_OK(cudaMalloc(&c->wt_nat, xtotal * 8));
      lce::expand_weights_imma_kernel<<<grid_for(xtotal, 256, 1 << 22), 256>>>(
          d_filter, reinterpret_cast<uint2*>(c->wt_nat), c->cout_pg, c->tiles_per_group, c->taps,
          c->Cw_pg, xtotal);
      if (launch_check("expand_weights_imma_kernel")) return 1;
      // K staging: everything in one chunk when it fits the CTA's shared-memory share, else a
      // two-deep ring of equal chunks. 3 CTAs per SM for uint4 operands, 4 otherwise (registers).
      const int single_max = static_cast<int>(budget / lce::kIBytesPerWord) / c->V;      // vectors
      const int ring_max = static_cast<int>(budget / (2 * lce::kIBytesPerWord)) / c->V;
      c->imma_chunks = c->Kv <= single_max ? 1 : cdiv(c->Kv, std::max(ring_max, 1));
      c->imma_Kc_v = cdiv(c->Kv, c->imma_chunks);
      c->imma_smem = static_cast<size_t>(c->imma_Kc_v) * c->V * lce::kIBytesPerWord *
                     (c->imma_chunks > 1 ? 2 : 1);  // two-deep ring
    }
    CUDA_OK(cudaMalloc(&c->wpop, static_cast<size_t>(c->cout + lce::kBN) * 4));
    CUDA_OK(cudaMemset(c->wpop, 0, static_cast<size_t>(c->cout + lce::kBN) * 4));
    lce::tap_popc_kernel<<<cdiv(c->cout, 256), 256>>>(d_filter, c->wpop, c->cout, 1, Kw);
    if (launch_check("tap_popc_kernel")) return 1;
  } else if (pair_b1) {
    // one 64-channel tile of b1 fragments whose channels 32-63 are zero (PairShape<1>)
    const int Kw = c->taps * c->Cw_pg;
    const int n_slices = cdiv(Kw, 8);
    const long long total = static_cast<long long>(n_slices) * 256;
    CUDA_OK(cudaMalloc(&c->pair_wt, total * 8));
    lce::pack_weights_b1_kernel<<<grid_for(total, 256, 1 << 22), 256>>>(
        d_filter, reinterpret_cast<uint2*>(c->pair_wt), c->cout_pg, 1, Kw, n_slices, total);
    if (launch_check("pack_weights_b1_kernel")) return 1;
    CUDA_OK(cudaMalloc(&c->wpop, static_cast<size_t>(c->cout + lce::kBN) * 4));
    CUDA_OK(cudaMemset(c->wpop, 0, static_cast<size_t>(c->cout + lce::kBN) * 4));
    lce::tap_popc_kernel<<<cdiv(c->cout, 256), 256>>>(d_filter, c->wpop, c->cout, 1, Kw);
    if (launch_check("tap_popc_kernel")) return 1;
  }
  if (build_tc_weights(c, d_filter, want_tap_popc)) return 1;
  if (want_tap_popc) {
    const size_t n = static_cast<size_t>(c->cout + lce::kBN) * c->taps;
    CUDA_OK(cudaMalloc(&c->tap_popc, n * 4));
    CUDA_OK(cudaMemset(c->tap_popc, 0, n * 4));
    lce::tap_popc_kernel<<<cdiv(c->cout * c->taps, 256), 256>>>(d_filter, c->tap_popc, c->cout,
                                                                c->taps, c->Cw_pg);
    if (launch_check("tap_popc_kernel")) return 1;
  }
  CUDA_OK(cudaDeviceSynchronize());
  if (!on_dev) cudaFree(d_filter);
  return 0;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// What keeps a layer off the pair kernel (lce_b200_pair.cuh), or nullptr: it takes 3x3, stride 1,
// dilation 1, ungrouped, SAME one-padded layers with float output and channels_in ==
// channels_out in {32, 64, 128}, on the b1 mma.sync inner product.
const char* pair_layer_refusal(const lce_bconv2d_desc& d) {
  if (d.out_type != LCE_OUT_FLOAT) return "float output";
  if (d.filter_h != 3 || d.filter_w != 3 || d.stride_h != 1 || d.stride_w != 1 ||
      d.dilation_h != 1 || d.dilation_w != 1 || d.groups != 1)
    return "an ungrouped 3x3 filter with stride 1 and dilation 1";
  if (d.padding != LCE_PADDING_SAME || d.pad_value != 1) return "SAME padding with pad_values = 1";
  if (d.channels_in != d.channels_out ||
      (d.channels_out != 32 && d.channels_out != 64 && d.channels_out != 128))
    return "channels_in == channels_out, 32, 64 or 128";
  if (env_off("LCE_B200_BCONV_IMMA") || env_off("LCE_B200_BCONV_B1"))
    return "the b1 mma.sync inner product (LCE_B200_BCONV_IMMA / _B1 are 0)";
  return nullptr;
}

// the pair kernel's output tile for C channels (32, 64 or 128)
void pair_tile(int C, int* th, int* tw) {
  *th = C == 32 ? lce::PairShape<1>::TH : C == 64 ? lce::PairShape<2>::TH : lce::PairShape<4>::TH;
  *tw = C == 32 ? lce::PairShape<1>::TW : C == 64 ? lce::PairShape<2>::TW : lce::PairShape<4>::TW;
}

// What keeps a plan off lce_b200_bconv2d_run_slice, or nullptr: float output and the mma.sync
// weight fragments, which a plan has when it was created with LCE_B200_BCONV_IMMA not 0 and full
// 64-channel tiles. c == nullptr: for a plan not created yet.
const char* slice_refusal(const lce_bconv2d_desc& d, const GemmCore* c) {
  if (d.out_type != LCE_OUT_FLOAT) return "float output";
  const bool imma = c != nullptr ? c->wt_nat != nullptr
                                 : !env_off("LCE_B200_BCONV_IMMA") && d.groups > 0 &&
                                       (d.channels_out / d.groups) % lce::kBN == 0;
  if (!imma)
    return "the mma.sync weight fragments (channels_out a multiple of 64, LCE_B200_BCONV_IMMA not 0)";
  return nullptr;
}

// What keeps a plan off lce_b200_bconv2d_run_fused_shuffle with an s_h x s_w shuffle, or nullptr: an
// ungrouped 1x1 / stride 1 / dilation 1 plan with float output, no fused activation and no zero
// padding, channels_out = s_h * s_w * C with C a multiple of 64, on the b1 mma.sync weight fragments.
// c == nullptr: for a plan not created yet.
const char* shuffle_refusal(const lce_bconv2d_desc& d, int s_h, int s_w, const GemmCore* c) {
  if (d.out_type != LCE_OUT_FLOAT || d.activation != LCE_ACT_NONE) return "float output without a fused activation";
  if (d.groups != 1 || d.filter_h != 1 || d.filter_w != 1 || d.stride_h != 1 || d.stride_w != 1 ||
      d.dilation_h != 1 || d.dilation_w != 1 || (d.padding == LCE_PADDING_SAME && d.pad_value == 0))
    return "an ungrouped 1x1 convolution with stride 1, dilation 1 and no zero padding";
  if (s_h <= 0 || s_w <= 0 || d.channels_out % (s_h * s_w) != 0 || (d.channels_out / (s_h * s_w)) % lce::kBN != 0)
    return "channels_out = s_h * s_w * C with C a multiple of 64";
  const bool b1 = c != nullptr ? c->wt_nat != nullptr && c->imma_b1 && !c->imma_win
                               : !env_off("LCE_B200_BCONV_IMMA") && !env_off("LCE_B200_BCONV_B1");
  if (!b1) return "the b1 mma.sync inner product (LCE_B200_BCONV_IMMA / _B1 are 0)";
  return nullptr;
}

// Whether lce_b200_bconv2d_run_fused / _run_fused_chain take packed output for the plan: every
// ungrouped plan, and grouped float-output plans with channels_out / groups a multiple of 32 on the
// b1 mma.sync weight fragments, whose epilogue packs whole 32-channel words of one CTA.
// c == nullptr: for a plan not created yet (LCE_B200_BCONV_IMMA and _B1 not 0).
bool grouped_packs(const lce_bconv2d_desc& d, const GemmCore* c) {
  if (d.groups == 1) return true;
  if (d.out_type != LCE_OUT_FLOAT || d.groups < 1 || (d.channels_out / d.groups) % 32 != 0) return false;
  if (c != nullptr) return c->wt_nat != nullptr && c->imma_b1;
  return !env_off("LCE_B200_BCONV_IMMA") && !env_off("LCE_B200_BCONV_B1");
}

template <int CW>
int launch_pair(const lce::PairParams& p, int grid, cudaStream_t s) {
  constexpr int smem = lce::PairShape<CW>::smem_bytes;
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(lce::bconv_pair_kernel<CW>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  lce::bconv_pair_kernel<CW><<<grid, lce::kPThreads, smem, s>>>(p);
  g_path[1].fetch_add(1, std::memory_order_relaxed);
  return launch_check("bconv_pair_kernel");
}

// OneTimeSetup's fold of the float / int8 output transform (bconv2d.cc:353-389), in double on the
// host: fm = -mul / scale, fb = (bias + K * mul) / scale + zero_point for each output channel.
int fold_output_transform(const lce_bconv2d_desc& d, const float* post_mul, const float* post_bias,
                          float* fm, float* fb) {
  const int cout = d.channels_out;
  std::vector<float> pm(cout), pb(cout);
  if (to_host(post_mul, cout * sizeof(float), pm.data()) || to_host(post_bias, cout * sizeof(float), pb.data()))
    return 1;
  const int32_t backtransform_add = d.filter_h * d.filter_w * (d.channels_in / d.groups);
  const double scale = d.out_type == LCE_OUT_INT8 ? static_cast<double>(d.out_scale) : 1.0;
  const double zp = d.out_type == LCE_OUT_INT8 ? static_cast<double>(d.out_zero_point) : 0.0;
  for (int i = 0; i < cout; ++i) {
    const double m = pm[i], b = pb[i];
    fm[i] = static_cast<float>(-1 * m / scale);
    fb[i] = static_cast<float>((b + static_cast<double>(backtransform_add) * m) / scale + zp);
  }
  return 0;
}

// ABC-Net bases kernel (bconv_bases_kernel): the M bases' fragments stay in shared memory, the
// planes stream through a two-deep ring of whole-K planes (reuse) or of K chunks. Returns what a
// layer with `n_slices` 8-word k-slices and `m_bases` bases stages, or a refusal.
constexpr size_t kBasesSmemMax = 226u * 1024u;   // one CTA per SM, its 1 KB of static shared memory aside
const char* bases_staging(int n_slices, int m_bases, int* chunk_slices, int* chunks, int* reuse,
                          size_t* smem) {
  const size_t w = static_cast<size_t>(m_bases) * n_slices * (8 * 32 * 8);
  const size_t slice_a = static_cast<size_t>(lce::kIBM) * 32;
  if (w + 2 * slice_a > kBasesSmemMax)
    return "the bases' weights for one 64-channel tile do not fit in shared memory";
  const size_t avail = kBasesSmemMax - w;
  if (2 * n_slices * slice_a <= avail) {
    *reuse = 1; *chunks = 1; *chunk_slices = n_slices;
  } else {
    const int ring = static_cast<int>(avail / (2 * slice_a));
    *reuse = 0;
    *chunks = cdiv(n_slices, ring);
    *chunk_slices = cdiv(n_slices, *chunks);
  }
  *smem = w + 2 * static_cast<size_t>(*chunk_slices) * slice_a;
  return nullptr;
}

template <int V>
int launch_bases(const lce::BasesParams& bp, dim3 grid, size_t smem, cudaStream_t s) {
  static PerDeviceOnce once;
  if (once.need())
    CUDA_OK(cudaFuncSetAttribute(lce::bconv_bases_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(kBasesSmemMax)));
  lce::bconv_bases_kernel<V><<<grid, lce::kIThreads, smem, s>>>(bp);
  g_path[1].fetch_add(1, std::memory_order_relaxed);
  return launch_check("bconv_bases_kernel");
}

// What keeps terms of this shape off the bases kernel, or nullptr
const char* bases_refusal(const lce_bconv2d_desc& d, int m_bases, int n_planes) {
  if (m_bases < 1 || n_planes < 1 || m_bases > lce::kMaxBases || n_planes > lce::kMaxBases)
    return "1 to 8 bases and 1 to 8 planes";
  if (d.out_type != LCE_OUT_FLOAT || d.activation != LCE_ACT_NONE)
    return "float output without a fused activation";
  if (d.groups != 1 || d.channels_out % lce::kBN != 0 || d.channels_in % 32 != 0)
    return "ungrouped terms with channels_in % 32 == 0 and channels_out % 64 == 0";
  if (d.padding == LCE_PADDING_SAME && d.pad_value == 0)
    return "one-padded or VALID terms (zero padding needs the per-term float correction)";
  if (env_off("LCE_B200_BCONV_IMMA") || env_off("LCE_B200_BCONV_B1"))
    return "the b1 mma.sync inner product (LCE_B200_BCONV_IMMA / _B1 are 0)";
  const int Kw = d.filter_h * d.filter_w * (d.channels_in / 32);
  int cs, nc, reuse;
  size_t smem;
  return bases_staging(cdiv(Kw, 8), m_bases, &cs, &nc, &reuse, &smem);
}

}  // namespace

// ------------------------------------------------------------------------- //
struct lce_b200_bconv2d {
  lce_bconv2d_desc d;
  int zp_mode = LCE_ZERO_PADDING_REFERENCE;
  int out_h = 0, out_w = 0, pad_h = 0, pad_w = 0;
  GemmCore core;
  int32_t* packed_scratch = nullptr;  // run_f32: packed activations
  size_t packed_scratch_words = 0;
  void* h2d_in = nullptr;             // run_host staging
  void* d2h_out = nullptr;
  size_t h2d_bytes = 0, d2h_bytes = 0;
};

struct lce_b200_bgemm {
  GemmCore core;
  int N = 0, Kw = 0;
};

extern "C" {

int lce_b200_abi_version(void) { return LCE_B200_ABI_VERSION; }
const char* lce_b200_last_error(void) { return g_err.c_str(); }
uint64_t lce_b200_launch_count(void) { return g_launches.load(); }
void lce_b200_path_counts(uint64_t out[3]) {
  for (int i = 0; i < 3; ++i) out[i] = g_path[i].load();
}
int lce_b200_tc_debug(int32_t out[8]) {
  int flag = 0;
  if (cudaMemcpyFromSymbol(&flag, lce::tc::g_tc_abort, sizeof(int)) != cudaSuccess) return 1;
  if (cudaMemcpyFromSymbol(out, lce::tc::g_tc_dbg, 8 * sizeof(int)) != cudaSuccess) return 1;
  out[7] = flag;
  if (flag) {
    const int zero = 0;
    cudaMemcpyToSymbol(lce::tc::g_tc_abort, &zero, sizeof(int));
  }
  return 0;
}

int lce_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

// ------------------------------ LceQuantize ------------------------------ //
int lce_b200_quantize(int in_type, const void* in_dev, int64_t rows, int64_t cols,
                      int32_t zero_point, int32_t* out_dev, void* stream) {
  if (rows < 0 || cols < 0) return fail("quantize: negative shape");
  if (rows == 0 || cols == 0) return 0;
  if (cols > INT_MAX) return fail("quantize: last dimension too large");
  cudaStream_t s = as_stream(stream);
  const int cw = static_cast<int>((cols + 31) / 32);
  const long long n_words = rows * cw;
  switch (in_type) {
    case LCE_T_FLOAT:
      if (cols % 32 == 0 && aligned16(in_dev)) {
        lce::pack_f32_flat_kernel<<<grid_for(n_words * 4, 256), 256, 0, s>>>(
            static_cast<const float4*>(in_dev), out_dev, n_words);
        return launch_check("pack_f32_flat_kernel");
      }
      lce::pack_generic_kernel<float><<<grid_for(n_words * 32, 256), 256, 0, s>>>(
          static_cast<const float*>(in_dev), out_dev, rows, static_cast<int>(cols), cw, 0);
      return launch_check("pack_generic_kernel<float>");
    case LCE_T_INT8:
      lce::pack_generic_kernel<int8_t><<<grid_for(n_words * 32, 256), 256, 0, s>>>(
          static_cast<const int8_t*>(in_dev), out_dev, rows, static_cast<int>(cols), cw,
          zero_point);
      return launch_check("pack_generic_kernel<int8>");
    case LCE_T_BOOL:
      lce::pack_generic_kernel<uint8_t><<<grid_for(n_words * 32, 256), 256, 0, s>>>(
          static_cast<const uint8_t*>(in_dev), out_dev, rows, static_cast<int>(cols), cw, 1);
      return launch_check("pack_generic_kernel<bool>");
  }
  return fail("quantize: unsupported input type %d", in_type);
}

// ----------------------------- LceDequantize ----------------------------- //
int lce_b200_dequantize(int out_type, const int32_t* in_dev, int64_t rows, int64_t cols,
                        float scale, int32_t zero_point, void* out_dev, void* stream) {
  if (rows < 0 || cols < 0) return fail("dequantize: negative shape");
  if (rows == 0 || cols == 0) return 0;
  if (cols > INT_MAX) return fail("dequantize: last dimension too large");
  cudaStream_t s = as_stream(stream);
  const int cw = static_cast<int>((cols + 31) / 32);
  const int grid = grid_for(rows * cols, 256);
  switch (out_type) {
    case LCE_T_FLOAT:
      lce::unpack_kernel<float><<<grid, 256, 0, s>>>(in_dev, static_cast<float*>(out_dev), rows,
                                                     static_cast<int>(cols), cw, 1.0f, -1.0f);
      return launch_check("unpack_kernel<float>");
    case LCE_T_INT8: {
      // quantization.cc:130-138
      const int offset = static_cast<int>(std::round(1.0f / scale));
      const int8_t zero_bit = static_cast<int8_t>(std::min(127, zero_point + offset));
      const int8_t one_bit = static_cast<int8_t>(std::max(-128, zero_point - offset));
      lce::unpack_kernel<int8_t><<<grid, 256, 0, s>>>(in_dev, static_cast<int8_t*>(out_dev), rows,
                                                      static_cast<int>(cols), cw, zero_bit,
                                                      one_bit);
      return launch_check("unpack_kernel<int8>");
    }
    case LCE_T_BOOL:
      lce::unpack_kernel<uint8_t><<<grid, 256, 0, s>>>(in_dev, static_cast<uint8_t*>(out_dev),
                                                       rows, static_cast<int>(cols), cw,
                                                       uint8_t(1), uint8_t(0));
      return launch_check("unpack_kernel<bool>");
  }
  return fail("dequantize: unsupported output type %d", out_type);
}

// ----------------------------- LceBMaxPool2d ----------------------------- //
int lce_b200_bmaxpool_out_shape(const lce_bmaxpool_desc* d, int* out_h, int* out_w) {
  // bmaxpool.cc:51-54
  if (!d->stride_h || !d->stride_w || !d->filter_h || !d->filter_w)
    return fail("bmaxpool: strides and filter sizes must be non-zero");
  if (d->padding != LCE_PADDING_SAME && d->padding != LCE_PADDING_VALID)
    return fail("bmaxpool: unknown padding %d", d->padding);
  *out_h = out_size(d->padding, d->in_h, d->filter_h, d->stride_h, 1);
  *out_w = out_size(d->padding, d->in_w, d->filter_w, d->stride_w, 1);
  return 0;
}

int lce_b200_bmaxpool(const lce_bmaxpool_desc* d, const int32_t* in_dev, int32_t* out_dev,
                      void* stream) {
  int oh, ow;
  if (lce_b200_bmaxpool_out_shape(d, &oh, &ow)) return 1;
  const long long n = static_cast<long long>(d->batch) * oh * ow * d->channels_packed;
  if (n <= 0) return 0;
  const int ph = pad_before(d->stride_h, 1, d->in_h, d->filter_h, oh);
  const int pw = pad_before(d->stride_w, 1, d->in_w, d->filter_w, ow);
  lce::bmaxpool_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(
      in_dev, out_dev, d->batch, d->in_h, d->in_w, d->channels_packed, oh, ow, d->filter_h,
      d->filter_w, d->stride_h, d->stride_w, ph, pw);
  return launch_check("bmaxpool_kernel");
}

// ------------------------------- LceBconv2d ------------------------------ //
int lce_b200_bconv2d_out_shape(const lce_bconv2d_desc* d, int* out_h, int* out_w, int* pad_h,
                               int* pad_w) {
  if (d->pad_value != 0 && d->pad_value != 1)
    return fail("Attribute pad_values must be 0 or 1.");  // bconv2d.cc:113-116
  if (d->padding != LCE_PADDING_SAME && d->padding != LCE_PADDING_VALID)
    return fail("bconv2d: unknown padding %d", d->padding);
  if (d->groups < 1 || d->channels_in < 1 || d->channels_out < 1 || d->filter_h < 1 ||
      d->filter_w < 1 || d->stride_h < 1 || d->stride_w < 1 || d->dilation_h < 1 ||
      d->dilation_w < 1)
    return fail("bconv2d: non-positive parameter");
  // bconv2d.cc:169-186
  if (d->channels_in % d->groups != 0)
    return fail("bconv2d: channels_in %d not divisible by groups %d", d->channels_in, d->groups);
  if (d->groups > 1 && (d->channels_in / d->groups) % 32 != 0)
    return fail("bconv2d: grouped convolutions need channels_in/groups %% 32 == 0");
  if (d->channels_out % d->groups != 0)
    return fail("bconv2d: channels_out %d not divisible by groups %d", d->channels_out,
                d->groups);
  *out_h = out_size(d->padding, d->in_h, d->filter_h, d->stride_h, d->dilation_h);
  *out_w = out_size(d->padding, d->in_w, d->filter_w, d->stride_w, d->dilation_w);
  *pad_h = pad_before(d->stride_h, d->dilation_h, d->in_h, d->filter_h, *out_h);
  *pad_w = pad_before(d->stride_w, d->dilation_w, d->in_w, d->filter_w, *out_w);
  if (*out_h < 0) *out_h = 0;
  if (*out_w < 0) *out_w = 0;
  return 0;
}

int lce_b200_bconv2d_create(const lce_bconv2d_desc* d, const int32_t* filter,
                            const float* post_mul, const float* post_bias,
                            const int32_t* thresholds, lce_b200_bconv2d** out_plan) {
  *out_plan = nullptr;
  if (lce_b200_device_count() < 1) return fail("no CUDA device: this library has no CPU path");
  int oh, ow, ph, pw;
  if (lce_b200_bconv2d_out_shape(d, &oh, &ow, &ph, &pw)) return 1;
  if (d->out_type != LCE_OUT_FLOAT && d->out_type != LCE_OUT_INT8 &&
      d->out_type != LCE_OUT_BITPACKED)
    return fail("Supported output types are int8, int32, and float32.");  // bconv2d.cc:158-162
  const bool zero_pad = d->padding == LCE_PADDING_SAME && d->pad_value == 0;
  // bconv2d.cc:188-200: the reference kernel's rule (even channels_in) or the optimised kernels'
  // (float output, no fused activation); the plan starts in the mode whose rule holds
  const bool zp_ref_rule = d->channels_in % 2 == 0;
  const bool zp_opt_rule = d->out_type == LCE_OUT_FLOAT && d->activation == LCE_ACT_NONE;
  if (zero_pad && !zp_ref_rule && !zp_opt_rule)
    return fail("Zero-padding is only supported by the reference kernel with an even number of "
                "input channels, or when using float output with no fused activation function.");
  if (d->out_type == LCE_OUT_BITPACKED) {
    if (!thresholds) return fail("bconv2d: bitpacked output needs the thresholds input");
  } else if (!post_mul || !post_bias) {
    return fail("bconv2d: float/int8 output needs post_activation_multiplier and bias");
  }
  if (!filter) return fail("bconv2d: filter is null");

  auto* plan = new lce_b200_bconv2d();
  plan->d = *d;
  plan->zp_mode = (zero_pad && !zp_ref_rule) ? LCE_ZERO_PADDING_CORRECTION : LCE_ZERO_PADDING_REFERENCE;
  plan->out_h = oh; plan->out_w = ow; plan->pad_h = ph; plan->pad_w = pw;
  GemmCore& c = plan->core;
  c.groups = d->groups;
  c.cout = d->channels_out;
  c.cout_pg = d->channels_out / d->groups;
  c.Cw_pg = cdiv(d->channels_in / d->groups, 32);
  c.taps = d->filter_h * d->filter_w;
  c.out_type = d->out_type;
  int rc = build_core_weights(&c, filter, zero_pad,
                              d->channels_out == 32 && pair_layer_refusal(*d) == nullptr);

  const size_t padded = static_cast<size_t>(c.cout) + kChanPad;
  if (!rc && d->out_type != LCE_OUT_BITPACKED) {
    // OneTimeSetup (bconv2d.cc:353-389): fold in double on the host.
    std::vector<float> fm(padded, 0.f), fb(padded, 0.f);
    rc = fold_output_transform(*d, post_mul, post_bias, fm.data(), fb.data());
    const int32_t backtransform_add = d->filter_h * d->filter_w * (d->channels_in / d->groups);
    int32_t nmin, nmax;  // CalculateActivationRange<int32>, kernel_util.h:285-300
    switch (d->activation) {
      case LCE_ACT_RELU: nmin = 0; nmax = INT32_MAX; break;
      case LCE_ACT_RELU6: nmin = 0; nmax = 6; break;
      case LCE_ACT_RELU_N1_TO_1: nmin = -1; nmax = 1; break;
      default: nmin = INT32_MIN; nmax = INT32_MAX; break;
    }
    nmin = std::max(nmin, -backtransform_add);
    nmax = std::min(nmax, backtransform_add);
    c.clamp_min = -nmax + backtransform_add;
    c.clamp_max = -nmin + backtransform_add;
    void *dm = nullptr, *db = nullptr;
    rc = rc || to_device(fm.data(), padded * 4, padded * 4, &dm) ||
         to_device(fb.data(), padded * 4, padded * 4, &db);
    c.mul = static_cast<float*>(dm);
    c.bias = static_cast<float*>(db);
    if (!rc && zero_pad && zp_opt_rule && c.tc_ok && c.tc_tap_popc_t != nullptr) {
      // the optimised kernels' correction cache (zero_padding_correction.h:39-176), once per plan
      const int eff_h = (d->filter_h - 1) * d->dilation_h + 1, eff_w = (d->filter_w - 1) * d->dilation_w + 1;
      const size_t n = static_cast<size_t>(4) * eff_h * eff_w * c.tc_ldc;
      if (cudaMalloc(&c.tc_zpc_cache, n * 4) != cudaSuccess || cudaMemset(c.tc_zpc_cache, 0, n * 4) != cudaSuccess) {
        rc = fail("bconv2d: cannot allocate the zero-padding correction cache");
      } else {
        const int total = 4 * eff_h * eff_w * c.cout;
        lce::tc::zpc_cache_kernel<<<cdiv(total, 256), 256>>>(c.tc_tap_popc_t, c.mul, c.tc_zpc_cache, c.cout, c.tc_ldc,
                                                           d->filter_h, d->filter_w, d->dilation_h, d->dilation_w,
                                                           d->channels_in / d->groups);
        rc = launch_check("zpc_cache_kernel");
        if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = fail("zpc_cache_kernel failed");
      }
    }
  } else if (!rc) {
    void* dt = nullptr;
    rc = to_device(thresholds, c.cout * 4, padded * 4, &dt);
    c.thr = static_cast<int32_t*>(dt);
  }
  if (rc) {
    c.release();
    delete plan;
    return 1;
  }
  *out_plan = plan;
  return 0;
}

int lce_b200_bconv2d_set_input_shape(lce_b200_bconv2d* plan, int batch, int in_h, int in_w) {
  lce_bconv2d_desc d = plan->d;
  d.batch = batch; d.in_h = in_h; d.in_w = in_w;
  if (batch < 0 || in_h < 1 || in_w < 1) return fail("bconv2d: bad input shape");
  int oh, ow, ph, pw;
  if (lce_b200_bconv2d_out_shape(&d, &oh, &ow, &ph, &pw)) return 1;
  plan->d = d;
  plan->out_h = oh; plan->out_w = ow; plan->pad_h = ph; plan->pad_w = pw;
  return 0;
}

int lce_b200_bconv2d_set_zero_padding_mode(lce_b200_bconv2d* plan, int mode) {
  const lce_bconv2d_desc& d = plan->d;
  if (mode == LCE_ZERO_PADDING_CORRECTION) {
    if (d.padding == LCE_PADDING_SAME && d.pad_value == 0 &&
        !(d.out_type == LCE_OUT_FLOAT && d.activation == LCE_ACT_NONE))
      return fail("Zero-padding is only supported by the reference kernel with an even number of "
                  "input channels, or when using float output with no fused activation function.");
  } else if (mode == LCE_ZERO_PADDING_REFERENCE) {
    if (d.padding == LCE_PADDING_SAME && d.pad_value == 0 && d.channels_in % 2 != 0)
      return fail("Zero-padding is only supported by the reference kernel with an even number of "
                  "input channels, or when using float output with no fused activation function.");
  } else {
    return fail("bconv2d: unknown zero-padding mode %d", mode);
  }
  plan->zp_mode = mode;
  return 0;
}

int lce_b200_bconv2d_get_desc(const lce_b200_bconv2d* plan, lce_bconv2d_desc* d, int* out_h,
                              int* out_w) {
  *d = plan->d;
  *out_h = plan->out_h;
  *out_w = plan->out_w;
  return 0;
}

static size_t bconv_out_bytes(const lce_b200_bconv2d* plan) {
  const size_t px = static_cast<size_t>(plan->d.batch) * plan->out_h * plan->out_w;
  switch (plan->d.out_type) {
    case LCE_OUT_BITPACKED: return px * cdiv(plan->d.channels_out, 32) * 4;
    case LCE_OUT_INT8: return px * plan->d.channels_out;
    default: return px * plan->d.channels_out * 4;
  }
}

static int bconv_run_impl(lce_b200_bconv2d* plan, const int32_t* in_dev, void* out_dev,
                          const float* residual, int residual_act, int32_t* packed_out,
                          const lce_chain_desc* chain, void* stream,
                          const lce_gate_desc* gate = nullptr, int64_t out_stride = 0,
                          float* scratch = nullptr, bool gate_per_position = false,
                          const lce::ConvKParams* shuffle = nullptr) {
  const lce_bconv2d_desc& d = plan->d;
  GemmCore& c = plan->core;
  cudaStream_t s = as_stream(stream);
  lce::ConvKParams p;
  memset(&p, 0, sizeof(p));
  p.in = in_dev; p.wt = c.wt; p.out = out_dev;
  p.mul = c.mul; p.bias = c.bias; p.thr = c.thr; p.tap_popc = c.tap_popc;
  p.residual = residual; p.packed_out = packed_out; p.residual_act = residual_act;
  p.M = static_cast<long long>(d.batch) * plan->out_h * plan->out_w;
  p.H = d.in_h; p.W = d.in_w;
  p.Cw_total = cdiv(d.channels_in, 32);
  p.Cw_pg = c.Cw_pg; p.CwV = c.Cw_pg / c.V;
  p.KH = d.filter_h; p.KW = d.filter_w;
  p.sh = d.stride_h; p.sw = d.stride_w; p.dh = d.dilation_h; p.dw = d.dilation_w;
  p.ph = plan->pad_h; p.pw = plan->pad_w; p.OH = plan->out_h; p.OW = plan->out_w;
  p.cout = c.cout; p.cout_pg = c.cout_pg; p.tiles_per_group = c.tiles_per_group;
  p.Kv = c.Kv; p.Kc_v = c.Kc_v; p.n_chunks = c.n_chunks;
  p.clamp_min = c.clamp_min; p.clamp_max = c.clamp_max;
  p.cw_out = cdiv(c.cout, 32);
  p.zp_half = (d.channels_in / d.groups) / 2;
  if (d.out_type == LCE_OUT_INT8)
    p.vec_store = (c.cout % 8 == 0 && c.cout_pg % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(out_dev) & 7u) == 0);
  else
    p.vec_store = (c.cout % 4 == 0 && c.cout_pg % 4 == 0 && aligned16(out_dev));
  p.bp_fast = (c.groups == 1 || c.cout_pg % 32 == 0);
  // Stage the shortcut rows through shared memory when every tile is full (so each thread
  // owns 8 valid, 16-byte aligned channels) and the extra 16 KB keep the CTAs/SM resident.
  static const bool res_stage_on = [] {
    const char* e = getenv("LCE_B200_RES_STAGE");
    return !(e && e[0] == '0');
  }();
  p.res_stage = res_stage_on && residual != nullptr && d.out_type == LCE_OUT_FLOAT &&
                p.vec_store && c.cout_pg % lce::kBN == 0 &&
                c.smem_bytes + lce::kResStageBytes <= cta_smem_budget();
  if (p.M == 0) return 0;
  // The 4V-byte cp.async gathers need 4V-byte aligned pixels.
  if ((reinterpret_cast<uintptr_t>(in_dev) & (4u * c.V - 1)) != 0)
    return fail("bconv2d: input pointer must be %d-byte aligned", 4 * c.V);
  if (d.out_type == LCE_OUT_BITPACKED && !p.bp_fast)
    CUDA_OK(cudaMemsetAsync(out_dev, 0, bconv_out_bytes(plan), s));
  const bool zp_float = c.tap_popc != nullptr && plan->zp_mode == LCE_ZERO_PADDING_CORRECTION;
  if (chain != nullptr) {
    if (!zp_float && takes_imma(c, p)) {
      p.chain = *chain;
      return launch_conv(c, p, s, Tail::kChain);
    }
    // every other kernel: the fused tail without the pack, then the chain pass in place
    const int rc = bconv_run_impl(plan, in_dev, out_dev, residual, residual_act, nullptr, nullptr,
                                  stream);
    if (rc) return rc;
    float* out = static_cast<float*>(out_dev);
    return lce_b200_f32_chain_sign(out, chain, p.M, c.cout, out, packed_out, stream);
  }
  if (gate != nullptr) {
    // gate_per_position: gate->gate is a scale [OH * OW][C] and gate->alpha is NULL
    if (!zp_float && takes_imma(c, p) && p.M < (1LL << 31)) {   // the epilogue's 32-bit image index
      p.gate = *gate;
      return launch_conv(c, p, s, gate_per_position ? Tail::kScale : Tail::kGate);
    }
    // every other kernel: the convolution alone, then the whole tail in one pass in place
    const int rc = bconv_run_impl(plan, in_dev, out_dev, nullptr, LCE_ACT_NONE, nullptr, nullptr,
                                  stream);
    if (rc) return rc;
    float* out = static_cast<float*>(out_dev);
    const int64_t pixels = static_cast<int64_t>(p.OH) * p.OW;
    if (gate_per_position) {
      const lce_scale_desc sd{gate->gate, gate->sign_scale, gate->sign_shift};
      return lce_b200_f32_scale_sign(out, &sd, residual, residual_act, d.batch, pixels, c.cout, out,
                                     packed_out, stream);
    }
    return lce_b200_f32_gate_sign(out, gate, residual, residual_act, d.batch, pixels, c.cout, out,
                                  packed_out, stream);
  }
  if (shuffle != nullptr) {
    // run_fused_shuffle (the caller checked that the b1 mma.sync kernel takes the plan): its shuf_*
    // fields, and the signs' words per output pixel of C channels
    p.shuf_sh = shuffle->shuf_sh; p.shuf_sw = shuffle->shuf_sw; p.shuf_c = shuffle->shuf_c;
    p.shuf_act = shuffle->shuf_act; p.shuf_bias = shuffle->shuf_bias; p.shuf_k = shuffle->shuf_k;
    p.shuf_alpha = shuffle->shuf_alpha; p.shuf_scale = shuffle->shuf_scale; p.shuf_shift = shuffle->shuf_shift;
    p.shuf_act2 = shuffle->shuf_act2;
    p.max_keys = shuffle->max_keys; p.fd_pts = shuffle->fd_pts;
    p.cw_out = shuffle->shuf_c / 32;
    if (!takes_imma(c, p)) return fail("bconv2d_run_fused_shuffle / _fc: the plan does not run on the mma.sync kernel");
    return launch_conv(c, p, s, shuffle->max_keys != nullptr ? Tail::kFcMax : Tail::kShuffle);
  }
  // run_slice / run_slice_add: the mma.sync kernel's strided store, and the residual read at the
  // same strided address (the caller checked that the kernel takes the plan)
  const bool slice = out_stride != 0;
  const Tail plain = slice ? Tail::kSlice : Tail::kNone;
  p.out_stride = slice ? out_stride : c.cout;
  if (!zp_float) return launch_conv(c, p, s, plain);
  // the optimised kernels' zero padding: one-padding accumulators + a float correction. The
  // wgmma kernel does it in its epilogue; the others run unfused and a tail pass finishes.
  p.zp_float = 1;
  p.cin_pg = d.channels_in / d.groups;
  if (c.tc_ok && !slice) {
    const int rc = tc_launch(c, p, s);
    if (rc >= 0) return rc;
  }
  // run_slice_add: the strided residual is the output itself, whose old values the tail still
  // needs, so the convolution writes [M][cout] to the scratch and the tail reads it from there
  if (slice && residual != nullptr && scratch == nullptr)
    return fail("bconv2d: a strided residual with the zero-padding correction needs a scratch");
  lce::ConvKParams q = p;
  q.tap_popc = nullptr; q.residual = nullptr; q.packed_out = nullptr; q.res_stage = 0; q.zp_float = 0;
  if (scratch != nullptr) {
    q.out = scratch;
    q.out_stride = c.cout;
  }
  const bool tc_was = c.tc_ok;
  c.tc_ok = false;
  const int rc = launch_conv(c, q, s, plain);
  c.tc_ok = tc_was;
  if (rc) return rc;
  lce::ZpcTailParams z;
  z.out = static_cast<float*>(out_dev); z.mul = c.mul; z.tap_popc = c.tap_popc;
  z.src = static_cast<const float*>(q.out); z.src_stride = q.out_stride;
  z.residual = residual; z.packed_out = packed_out; z.M = p.M; z.out_stride = p.out_stride;
  z.H = p.H; z.W = p.W; z.OH = p.OH; z.OW = p.OW; z.KH = p.KH; z.KW = p.KW;
  z.sh = p.sh; z.sw = p.sw; z.dh = p.dh; z.dw = p.dw;
  z.cout = c.cout; z.cin_pg = p.cin_pg; z.cw_out = p.cw_out; z.residual_act = residual_act;
  lce::zpc_tail_kernel<<<grid_for(p.M * cdiv(c.cout, 32) * 32, 256), 256, 0, s>>>(z);
  return launch_check("zpc_tail_kernel");
}

int lce_b200_bconv2d_run(lce_b200_bconv2d* plan, const int32_t* in_dev, void* out_dev,
                         void* stream) {
  return bconv_run_impl(plan, in_dev, out_dev, nullptr, LCE_ACT_NONE, nullptr, nullptr, stream);
}

int lce_b200_bconv2d_run_fused(lce_b200_bconv2d* plan, const int32_t* in_dev,
                               const float* residual_dev, int add_activation, float* out_dev,
                               int32_t* packed_out_dev, void* stream) {
  if (plan->d.out_type != LCE_OUT_FLOAT)
    return fail("bconv2d_run_fused: only float-output plans can take a residual");
  if (packed_out_dev && !grouped_packs(plan->d, &plan->core))
    return fail("bconv2d_run_fused: packed output needs groups == 1, or channels_out / groups a "
                "multiple of 32 on the b1 mma.sync kernel");
  if (residual_dev && (reinterpret_cast<uintptr_t>(residual_dev) & 15u) != 0)
    return fail("bconv2d_run_fused: residual must be 16-byte aligned");
  return bconv_run_impl(plan, in_dev, out_dev, residual_dev, add_activation, packed_out_dev,
                        nullptr, stream);
}

int lce_b200_bconv2d_run_fused_chain(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                     const float* residual_dev, int add_activation,
                                     const lce_chain_desc* chain, float* out_dev,
                                     int32_t* packed_out_dev, void* stream) {
  if (plan->d.out_type != LCE_OUT_FLOAT)
    return fail("bconv2d_run_fused_chain: only float-output plans can take a chain");
  if (packed_out_dev && !grouped_packs(plan->d, &plan->core))
    return fail("bconv2d_run_fused_chain: packed output needs groups == 1, or channels_out / groups "
                "a multiple of 32 on the b1 mma.sync kernel");
  if (residual_dev && (reinterpret_cast<uintptr_t>(residual_dev) & 15u) != 0)
    return fail("bconv2d_run_fused_chain: residual must be 16-byte aligned");
  if (chain)
    for (const float* v : {chain->shift_in, chain->alpha, chain->shift_out, chain->sign_shift})
      if (v && !is_device_ptr(v)) return fail("bconv2d_run_fused_chain: chain vectors must be device memory");
  return bconv_run_impl(plan, in_dev, out_dev, residual_dev, add_activation, packed_out_dev, chain,
                        stream);
}

int lce_b200_bconv2d_run_fused_gate(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                    const lce_gate_desc* gate, const float* residual_dev,
                                    int add_activation, float* out_dev, int32_t* packed_out_dev,
                                    void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (d.out_type != LCE_OUT_FLOAT)
    return fail("bconv2d_run_fused_gate: only float-output plans can take a gate");
  if (packed_out_dev && d.groups != 1)
    return fail("bconv2d_run_fused_gate: packed output needs groups == 1");
  if (!gate || !gate->gate) return fail("bconv2d_run_fused_gate: the gate tensor is required");
  if (add_activation < LCE_ACT_NONE || add_activation > LCE_ACT_RELU6)
    return fail("bconv2d_run_fused_gate: unknown ADD activation %d", add_activation);
  if (residual_dev && !aligned16(residual_dev))
    return fail("bconv2d_run_fused_gate: residual must be 16-byte aligned");
  if ((reinterpret_cast<uintptr_t>(gate->gate) & 7u) != 0)
    return fail("bconv2d_run_fused_gate: the gate must be 8-byte aligned");
  for (const float* v : {gate->gate, gate->alpha, gate->sign_scale, gate->sign_shift})
    if (v && !is_device_ptr(v)) return fail("bconv2d_run_fused_gate: gate vectors must be device memory");
  // the epilogue reads the shortcut and the gate of rows other CTAs write: out must not alias them
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t o1 = o0 + bconv_out_bytes(plan);
  auto overlaps = [&](const void* v, size_t bytes) {
    const uintptr_t v0 = reinterpret_cast<uintptr_t>(v);
    return v != nullptr && v0 < o1 && o0 < v0 + bytes;
  };
  if (overlaps(residual_dev, bconv_out_bytes(plan)))
    return fail("bconv2d_run_fused_gate: output must not overlap the residual");
  if (overlaps(gate->gate, static_cast<size_t>(d.batch) * d.channels_out * sizeof(float)))
    return fail("bconv2d_run_fused_gate: output must not overlap the gate");
  return bconv_run_impl(plan, in_dev, out_dev, residual_dev, add_activation, packed_out_dev,
                        nullptr, stream, gate);
}

int lce_b200_bconv2d_run_fused_scale(lce_b200_bconv2d* plan, const int32_t* in_dev,
                                     const lce_scale_desc* scale, const float* residual_dev,
                                     int add_activation, float* out_dev, int32_t* packed_out_dev,
                                     void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (d.out_type != LCE_OUT_FLOAT)
    return fail("bconv2d_run_fused_scale: only float-output plans can take a scale");
  if (packed_out_dev && d.groups != 1)
    return fail("bconv2d_run_fused_scale: packed output needs groups == 1");
  if (!scale || !scale->scale) return fail("bconv2d_run_fused_scale: the scale tensor is required");
  if (add_activation < LCE_ACT_NONE || add_activation > LCE_ACT_RELU6)
    return fail("bconv2d_run_fused_scale: unknown ADD activation %d", add_activation);
  if (residual_dev && !aligned16(residual_dev))
    return fail("bconv2d_run_fused_scale: residual must be 16-byte aligned");
  if ((reinterpret_cast<uintptr_t>(scale->scale) & 7u) != 0)
    return fail("bconv2d_run_fused_scale: the scale must be 8-byte aligned");
  for (const float* v : {scale->scale, scale->sign_scale, scale->sign_shift})
    if (v && !is_device_ptr(v)) return fail("bconv2d_run_fused_scale: scale vectors must be device memory");
  // the epilogue reads the shortcut and the scale rows other CTAs may write: out must not alias them
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t o1 = o0 + bconv_out_bytes(plan);
  auto overlaps = [&](const void* v, size_t bytes) {
    const uintptr_t v0 = reinterpret_cast<uintptr_t>(v);
    return v != nullptr && v0 < o1 && o0 < v0 + bytes;
  };
  if (overlaps(residual_dev, bconv_out_bytes(plan)))
    return fail("bconv2d_run_fused_scale: output must not overlap the residual");
  if (overlaps(scale->scale, static_cast<size_t>(plan->out_h) * plan->out_w * d.channels_out * sizeof(float)))
    return fail("bconv2d_run_fused_scale: output must not overlap the scale");
  const lce_gate_desc gate{scale->scale, nullptr, scale->sign_scale, scale->sign_shift};
  return bconv_run_impl(plan, in_dev, out_dev, residual_dev, add_activation, packed_out_dev,
                        nullptr, stream, &gate, 0, nullptr, /*gate_per_position=*/true);
}

int lce_b200_bconv2d_run_slice(lce_b200_bconv2d* plan, const int32_t* in_dev, float* out_dev,
                               int64_t out_pixel_stride, void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (const char* why = slice_refusal(d, &plan->core))
    return fail("bconv2d_run_slice: the plan needs %s", why);
  if (out_pixel_stride < d.channels_out || out_pixel_stride % 4 != 0)
    return fail("bconv2d_run_slice: the output pixel stride %lld must be a multiple of 4 and at "
                "least channels_out %d", static_cast<long long>(out_pixel_stride), d.channels_out);
  if (!aligned16(out_dev)) return fail("bconv2d_run_slice: output must be 16-byte aligned");
  const long long px = static_cast<long long>(d.batch) * plan->out_h * plan->out_w;
  if (px == 0) return 0;
  // the output's span, first float of pixel 0 to the last of pixel px - 1, against the packed input
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t o1 = o0 + (static_cast<uintptr_t>(px - 1) * out_pixel_stride + d.channels_out) * 4;
  const uintptr_t i0 = reinterpret_cast<uintptr_t>(in_dev);
  const uintptr_t i1 = i0 + static_cast<uintptr_t>(d.batch) * d.in_h * d.in_w * cdiv(d.channels_in, 32) * 4;
  if (o0 < i1 && i0 < o1) return fail("bconv2d_run_slice: output must not overlap the input");
  return bconv_run_impl(plan, in_dev, out_dev, nullptr, LCE_ACT_NONE, nullptr, nullptr, stream,
                        nullptr, out_pixel_stride);
}

int lce_b200_bconv2d_run_slice_add(lce_b200_bconv2d* plan, const int32_t* in_dev, float* io_dev,
                                   int64_t io_pixel_stride, float* scratch_dev, void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (const char* why = slice_refusal(d, &plan->core))
    return fail("bconv2d_run_slice_add: the plan needs %s", why);
  if (io_pixel_stride < d.channels_out || io_pixel_stride % 4 != 0)
    return fail("bconv2d_run_slice_add: the pixel stride %lld must be a multiple of 4 and at "
                "least channels_out %d", static_cast<long long>(io_pixel_stride), d.channels_out);
  if (!aligned16(io_dev)) return fail("bconv2d_run_slice_add: io must be 16-byte aligned");
  const long long px = static_cast<long long>(d.batch) * plan->out_h * plan->out_w;
  const bool corr = plan->core.tap_popc != nullptr && plan->zp_mode == LCE_ZERO_PADDING_CORRECTION;
  if (corr && scratch_dev == nullptr)
    return fail("bconv2d_run_slice_add: a zero-padding CORRECTION plan needs the scratch "
                "([pixels, channels_out] floats)");
  if (corr && !aligned16(scratch_dev)) return fail("bconv2d_run_slice_add: scratch must be 16-byte aligned");
  if (px == 0) return 0;
  // the spans: io from the first float of pixel 0 to the last of pixel px - 1, the packed input,
  // the scratch
  auto span = [](const void* p, uintptr_t bytes) {
    return std::make_pair(reinterpret_cast<uintptr_t>(p), reinterpret_cast<uintptr_t>(p) + bytes);
  };
  auto overlap = [](std::pair<uintptr_t, uintptr_t> a, std::pair<uintptr_t, uintptr_t> b) {
    return a.first < b.second && b.first < a.second;
  };
  const auto io = span(io_dev, (static_cast<uintptr_t>(px - 1) * io_pixel_stride + d.channels_out) * 4);
  const auto in = span(in_dev, static_cast<uintptr_t>(d.batch) * d.in_h * d.in_w * cdiv(d.channels_in, 32) * 4);
  if (overlap(io, in)) return fail("bconv2d_run_slice_add: io must not overlap the input");
  if (corr) {
    const auto sc = span(scratch_dev, static_cast<uintptr_t>(px) * d.channels_out * 4);
    if (overlap(sc, io) || overlap(sc, in))
      return fail("bconv2d_run_slice_add: scratch must not overlap io or the input");
  }
  return bconv_run_impl(plan, in_dev, io_dev, io_dev, LCE_ACT_NONE, nullptr, nullptr, stream, nullptr,
                        io_pixel_stride, corr ? scratch_dev : nullptr);
}

int lce_b200_bconv2d_run_fused_shuffle(lce_b200_bconv2d* plan, const int32_t* in_dev, int s_h, int s_w,
                                       const float* bias_dev, int activation, const float* skip_dev,
                                       int add_activation, float* out_dev, int32_t* packed_out_dev,
                                       void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (const char* why = shuffle_refusal(d, s_h, s_w, &plan->core))
    return fail("bconv2d_run_fused_shuffle: the plan needs %s", why);
  for (int a : {activation, add_activation})
    if (a < LCE_ACT_NONE || a > LCE_ACT_RELU6) return fail("bconv2d_run_fused_shuffle: unknown activation %d", a);
  if (!aligned16(out_dev) || (skip_dev && !aligned16(skip_dev)) ||
      (bias_dev && (reinterpret_cast<uintptr_t>(bias_dev) & 7u) != 0))
    return fail("bconv2d_run_fused_shuffle: out and skip must be 16-byte aligned, bias 8-byte aligned");
  if (bias_dev && !is_device_ptr(bias_dev)) return fail("bconv2d_run_fused_shuffle: bias must be device memory");
  const long long px = static_cast<long long>(d.batch) * plan->out_h * plan->out_w;
  if (px >= (1LL << 31) - lce::kIBM) return fail("bconv2d_run_fused_shuffle: too many input pixels (%lld)", px);
  if (px == 0) return 0;
  // the epilogue reads the skip and the input other CTAs' rows may land on: out must not alias them
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t o1 = o0 + bconv_out_bytes(plan);   // px * s_h * s_w * C floats
  auto overlaps = [&](const void* v, size_t bytes) {
    const uintptr_t v0 = reinterpret_cast<uintptr_t>(v);
    return v != nullptr && v0 < o1 && o0 < v0 + bytes;
  };
  if (overlaps(skip_dev, bconv_out_bytes(plan)) ||
      overlaps(in_dev, static_cast<size_t>(px) * cdiv(d.channels_in, 32) * 4))
    return fail("bconv2d_run_fused_shuffle: out must not overlap the skip or the input");
  const lce::ConvKParams shuf = [&] {
    lce::ConvKParams q;
    memset(&q, 0, sizeof(q));
    q.shuf_sh = s_h; q.shuf_sw = s_w; q.shuf_c = d.channels_out / (s_h * s_w);
    q.shuf_act = activation; q.shuf_bias = bias_dev; q.shuf_k = d.channels_in;
    return q;
  }();
  return bconv_run_impl(plan, in_dev, out_dev, skip_dev, add_activation, packed_out_dev, nullptr, stream, nullptr,
                        0, nullptr, false, &shuf);
}

// host-internal (Graph::FuseBinaryTransposeConvs): lce_b200_bconv2d_run_fused_shuffle takes an s_h x s_w
// shuffle of a plan created now from *d; no device needed
int lce_b200_internal_shuffle_takes(const lce_bconv2d_desc* d, int s_h, int s_w) {
  return shuffle_refusal(*d, s_h, s_w, nullptr) == nullptr;
}

// What keeps a plan off lce_b200_bconv2d_run_fused_fc, or nullptr: the shuffle store's plan with s_h =
// s_w = 1 (channels_out % 64 == 0, the b1 mma.sync kernel) on a 1 x 1 input, so that its rows are the
// dense layer's rows.
static const char* fc_refusal(const lce_bconv2d_desc& d, const GemmCore* c) {
  if (d.in_h != 1 || d.in_w != 1) return "in_h = in_w = 1 (one row per image)";
  return shuffle_refusal(d, 1, 1, c);
}

int lce_b200_bconv2d_run_fused_fc(lce_b200_bconv2d* plan, const int32_t* in_dev, const float* alpha_dev,
                                  const float* bias_dev, int activation, const float* scale_dev,
                                  const float* shift_dev, int bn_activation, float* out_dev,
                                  int32_t* packed_out_dev, void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (const char* why = fc_refusal(d, &plan->core)) return fail("bconv2d_run_fused_fc: the plan needs %s", why);
  for (int a : {activation, bn_activation})
    if (a < LCE_ACT_NONE || a > LCE_ACT_RELU6) return fail("bconv2d_run_fused_fc: unknown activation %d", a);
  if (!aligned16(out_dev)) return fail("bconv2d_run_fused_fc: out must be 16-byte aligned");
  for (const float* v : {alpha_dev, bias_dev, scale_dev, shift_dev}) {
    if (v && (reinterpret_cast<uintptr_t>(v) & 7u) != 0)
      return fail("bconv2d_run_fused_fc: alpha, bias, scale and shift must be 8-byte aligned");
    if (v && !is_device_ptr(v)) return fail("bconv2d_run_fused_fc: alpha, bias, scale and shift must be device memory");
  }
  const long long rows = d.batch;
  if (rows >= (1LL << 31) - lce::kIBM) return fail("bconv2d_run_fused_fc: too many rows (%lld)", rows);
  if (rows == 0) return 0;
  // other CTAs read the input rows this CTA's store may land on
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t o1 = o0 + bconv_out_bytes(plan);   // rows * N floats
  const size_t in_bytes = static_cast<size_t>(rows) * cdiv(d.channels_in, 32) * 4;
  const size_t pk_bytes = static_cast<size_t>(rows) * (d.channels_out / 32) * 4;
  auto overlap = [](const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a != nullptr && b != nullptr && a0 < b0 + nb && b0 < a0 + na;
  };
  if (overlap(in_dev, in_bytes, out_dev, o1 - o0) || overlap(packed_out_dev, pk_bytes, out_dev, o1 - o0) ||
      overlap(packed_out_dev, pk_bytes, in_dev, in_bytes))
    return fail("bconv2d_run_fused_fc: out, packed_out and the input must not overlap");
  const lce::ConvKParams fc = [&] {
    lce::ConvKParams q;
    memset(&q, 0, sizeof(q));
    q.shuf_sh = 1; q.shuf_sw = 1; q.shuf_c = d.channels_out; q.shuf_k = d.channels_in;
    q.shuf_act = activation; q.shuf_bias = bias_dev; q.shuf_alpha = alpha_dev;
    q.shuf_scale = scale_dev; q.shuf_shift = shift_dev; q.shuf_act2 = bn_activation;
    return q;
  }();
  return bconv_run_impl(plan, in_dev, out_dev, nullptr, LCE_ACT_NONE, packed_out_dev, nullptr, stream, nullptr, 0,
                        nullptr, false, &fc);
}

// host-internal (Graph::FuseBinaryFullyConnected): lce_b200_bconv2d_run_fused_fc takes a plan created
// now from *d; no device needed
int lce_b200_internal_fc_takes(const lce_bconv2d_desc* d) { return fc_refusal(*d, nullptr) == nullptr; }

// The keys of lce_b200_bconv2d_run_fused_fc_max as floats (max_key_value), one thread per (image,
// column), and each 32 columns' signs packed by a ballot (N % 32 == 0): keys [B][N], out [B][N] or
// null, packed [B][N / 32] or null.
__global__ void __launch_bounds__(256) fc_max_finalize_kernel(const unsigned long long* __restrict__ keys,
                                                              long long total, float* __restrict__ out,
                                                              int32_t* __restrict__ packed) {
  // total % 32 == 0: every warp is whole
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    const float v = lce::max_key_value(keys[i]);
    if (out) out[i] = v;
    const unsigned bits = __ballot_sync(0xffffffffu, v < 0.0f);
    if (packed && (threadIdx.x & 31) == 0) packed[i / 32] = static_cast<int32_t>(bits);
  }
}

static const char* fc_max_refusal(const lce_bconv2d_desc& d, int points, const GemmCore* c) {
  if (points <= 0 || d.batch % points != 0) return "batch rows a whole number of images of `points` rows";
  return fc_refusal(d, c);
}

int lce_b200_bconv2d_run_fused_fc_max(lce_b200_bconv2d* plan, const int32_t* in_dev, const float* alpha_dev,
                                      const float* bias_dev, int activation, const float* scale_dev,
                                      const float* shift_dev, int bn_activation, int points, void* keys_dev,
                                      float* max_out_dev, int32_t* packed_out_dev, void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  if (const char* why = fc_max_refusal(d, points, &plan->core))
    return fail("bconv2d_run_fused_fc_max: the plan needs %s", why);
  for (int a : {activation, bn_activation})
    if (a < LCE_ACT_NONE || a > LCE_ACT_RELU6) return fail("bconv2d_run_fused_fc_max: unknown activation %d", a);
  if (!aligned16(keys_dev)) return fail("bconv2d_run_fused_fc_max: keys must be 16-byte aligned");
  if (!max_out_dev && !packed_out_dev) return fail("bconv2d_run_fused_fc_max: max_out and packed_out are both null");
  for (const float* v : {alpha_dev, bias_dev, scale_dev, shift_dev}) {
    if (v && (reinterpret_cast<uintptr_t>(v) & 7u) != 0)
      return fail("bconv2d_run_fused_fc_max: alpha, bias, scale and shift must be 8-byte aligned");
    if (v && !is_device_ptr(v))
      return fail("bconv2d_run_fused_fc_max: alpha, bias, scale and shift must be device memory");
  }
  const long long rows = d.batch;
  if (rows >= (1LL << 31) - lce::kIBM) return fail("bconv2d_run_fused_fc_max: too many rows (%lld)", rows);
  if (rows == 0) return 0;
  const int n = d.channels_out;
  const long long images = rows / points, total = images * n;
  const size_t in_bytes = static_cast<size_t>(rows) * cdiv(d.channels_in, 32) * 4;
  const size_t key_bytes = static_cast<size_t>(total) * 8, out_bytes = static_cast<size_t>(total) * 4;
  const size_t pk_bytes = static_cast<size_t>(total / 32) * 4;
  auto overlap = [](const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a != nullptr && b != nullptr && a0 < b0 + nb && b0 < a0 + na;
  };
  if (overlap(keys_dev, key_bytes, in_dev, in_bytes) || overlap(keys_dev, key_bytes, max_out_dev, out_bytes) ||
      overlap(keys_dev, key_bytes, packed_out_dev, pk_bytes) || overlap(max_out_dev, out_bytes, packed_out_dev, pk_bytes))
    return fail("bconv2d_run_fused_fc_max: keys, max_out and packed_out must not overlap each other or the input");
  cudaStream_t s = as_stream(stream);
  // every key starts below every value's: replays and reused memory give the same bits
  CUDA_OK(cudaMemsetAsync(keys_dev, 0, key_bytes, s));
  const lce::ConvKParams fc = [&] {
    lce::ConvKParams q;
    memset(&q, 0, sizeof(q));
    q.shuf_sh = 1; q.shuf_sw = 1; q.shuf_c = n; q.shuf_k = d.channels_in;
    q.shuf_act = activation; q.shuf_bias = bias_dev; q.shuf_alpha = alpha_dev;
    q.shuf_scale = scale_dev; q.shuf_shift = shift_dev; q.shuf_act2 = bn_activation;
    q.max_keys = static_cast<unsigned long long*>(keys_dev);
    q.fd_pts = lce::make_fastdiv(static_cast<uint32_t>(points));
    return q;
  }();
  // keys_dev stands in for the output: the instance stores nothing there but reads its alignment
  const int rc = bconv_run_impl(plan, in_dev, keys_dev, nullptr, LCE_ACT_NONE, nullptr, nullptr, stream, nullptr, 0,
                                nullptr, false, &fc);
  if (rc) return rc;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, 148LL * 16));
  fc_max_finalize_kernel<<<grid, 256, 0, s>>>(static_cast<const unsigned long long*>(keys_dev), total, max_out_dev,
                                              packed_out_dev);
  return launch_check("fc_max_finalize_kernel");
}

// host-internal (Graph::FuseBinaryFcMax): lce_b200_bconv2d_run_fused_fc_max takes a plan created now
// from *d with images of `points` rows; no device needed
int lce_b200_internal_fc_max_takes(const lce_bconv2d_desc* d, int points) {
  return fc_max_refusal(*d, points, nullptr) == nullptr;
}

// Whether lce_b200_bconv2d_run_slice will take a plan created now from *d
// (Graph::FuseDenseBlocks asks before it rewrites the graph).
int lce_b200_internal_slice_takes(const lce_bconv2d_desc* d) {
  return slice_refusal(*d, nullptr) == nullptr;
}

// host-internal (Graph::FuseResidualBlocks, BconvPrepare): run_fused / run_fused_chain take
// packed output for a plan created now from *d; no device needed
int lce_b200_internal_grouped_packs(const lce_bconv2d_desc* d) {
  return grouped_packs(*d, nullptr);
}

// host-internal (Graph::FuseBinaryBases): lce_b200_bconv2d_bases_create would take M * N terms of
// this descriptor; no device needed
int lce_b200_internal_bases_takes(const lce_bconv2d_desc* d, int m_bases, int n_planes) {
  return bases_refusal(*d, m_bases, n_planes) == nullptr;
}

int lce_b200_bconv2d_run_fused_pair(lce_b200_bconv2d* plan1, lce_b200_bconv2d* plan2,
                                    const int32_t* in_dev, const float* residual_dev,
                                    int act1, int act2, float* out_dev, int32_t* packed_out_dev,
                                    void* stream) {
  if (!plan1 || !plan2 || !in_dev || !residual_dev || !out_dev)
    return fail("bconv2d_run_fused_pair: plans, input, residual and output are required");
  for (const lce_b200_bconv2d* pl : {plan1, plan2}) {
    if (const char* why = pair_layer_refusal(pl->d))
      return fail("bconv2d_run_fused_pair: each layer needs %s", why);
    if (pl->core.pair_wt == nullptr && (!pl->core.imma_b1 || pl->core.wt_nat == nullptr))
      return fail("bconv2d_run_fused_pair: each plan needs the b1 mma.sync weight fragments");
  }
  const lce_bconv2d_desc& d = plan1->d;
  const lce_bconv2d_desc& d2 = plan2->d;
  if (d2.channels_in != d.channels_out || d2.batch != d.batch || d2.in_h != d.in_h ||
      d2.in_w != d.in_w)
    return fail("bconv2d_run_fused_pair: the second layer must take the first one's output shape");
  for (int a : {act1, act2})
    if (a < LCE_ACT_NONE || a > LCE_ACT_RELU6)
      return fail("bconv2d_run_fused_pair: unknown ADD activation %d", a);
  const int C = d.channels_out, CW = C / 32;
  if ((reinterpret_cast<uintptr_t>(in_dev) & (4u * CW - 1)) != 0)
    return fail("bconv2d_run_fused_pair: input pointer must be %d-byte aligned", 4 * CW);
  if (!aligned16(residual_dev) || !aligned16(out_dev))
    return fail("bconv2d_run_fused_pair: residual and output must be 16-byte aligned");
  const long long px = static_cast<long long>(d.batch) * d.in_h * d.in_w;
  if (px == 0) return 0;
  // a CTA reads the shortcut of its neighbours' tiles: writing x2 over x0 would race
  const uintptr_t r0 = reinterpret_cast<uintptr_t>(residual_dev), o0 = reinterpret_cast<uintptr_t>(out_dev);
  const uintptr_t bytes = static_cast<uintptr_t>(px) * C * 4;
  if (r0 < o0 + bytes && o0 < r0 + bytes)
    return fail("bconv2d_run_fused_pair: output must not overlap the residual");
  lce::PairParams p;
  memset(&p, 0, sizeof(p));
  p.in = in_dev; p.residual = residual_dev; p.out = out_dev; p.packed_out = packed_out_dev;
  const lce_b200_bconv2d* plans[2] = {plan1, plan2};
  for (int k = 0; k < 2; ++k) {
    const GemmCore& c = plans[k]->core;
    p.wt[k] = reinterpret_cast<const uint2*>(c.pair_wt != nullptr ? c.pair_wt : c.wt_nat);
    p.wpop[k] = c.wpop; p.mul[k] = c.mul; p.bias[k] = c.bias;
    p.clamp_min[k] = c.clamp_min; p.clamp_max[k] = c.clamp_max;
  }
  p.act[0] = act1; p.act[1] = act2;
  p.H = d.in_h; p.W = d.in_w;
  int th, tw;
  pair_tile(C, &th, &tw);
  p.tiles_x = cdiv(d.in_w, tw);
  p.tiles_per_img = p.tiles_x * cdiv(d.in_h, th);
  const long long grid = static_cast<long long>(d.batch) * p.tiles_per_img;
  if (grid > INT_MAX) return fail("bconv2d_run_fused_pair: too many tiles");
  cudaStream_t s = as_stream(stream);
  if (CW == 1) return launch_pair<1>(p, static_cast<int>(grid), s);
  if (CW == 2) return launch_pair<2>(p, static_cast<int>(grid), s);
  return launch_pair<4>(p, static_cast<int>(grid), s);
}

// Whether Graph::FuseResidualPairs should pair two such layers at this image size: the pair kernel
// takes them and at least half of its tiles' pixels are the image's. Measured on an H100 80GB
// HBM3, batch 256 (tools/pair_bench.py), pair time over two run_fused calls: whole tiles 0.65 -
// 0.77 (56x56x64, 28x28x128, 42x42x64, 14x14x64 and x128); 22x22x64 (62 % used) 0.80, 32x32x64
// (58 %) 0.95, 11x11x128 (62 %) 0.97, 7x7x128 (50 %) 0.88; 16x16x64 and 8x8x128 (33 %) 1.26 and
// 1.73: there the ring recompute and the empty tile area cost more than x1's round trip saves.
// The 32-channel instance follows the same rule with the 64-channel tile; it is measured at
// 56x56 only (QuickNetSmall), not at partial tiles.
int lce_b200_internal_pair_pays_off(const lce_bconv2d_desc* d) {
  if (pair_layer_refusal(*d) != nullptr || d->in_h < 1 || d->in_w < 1) return 0;
  int th, tw;
  pair_tile(d->channels_out, &th, &tw);
  const long long tiled = static_cast<long long>(cdiv(d->in_h, th)) * th * cdiv(d->in_w, tw) * tw;
  return 2LL * d->in_h * d->in_w >= tiled;
}

int lce_b200_bconv2d_run_f32(lce_b200_bconv2d* plan, const float* in_dev, void* out_dev,
                             void* stream) {
  const lce_bconv2d_desc& d = plan->d;
  const int cw = cdiv(d.channels_in, 32);
  const size_t rows = static_cast<size_t>(d.batch) * d.in_h * d.in_w;
  const size_t words = rows * cw;
  if (words > plan->packed_scratch_words) {
    cudaFree(plan->packed_scratch);
    plan->packed_scratch = nullptr;
    plan->packed_scratch_words = 0;
    CUDA_OK(cudaMalloc(&plan->packed_scratch, words * 4 + 16));
    plan->packed_scratch_words = words;
  }
  if (lce_b200_quantize(LCE_T_FLOAT, in_dev, static_cast<int64_t>(rows), d.channels_in, 0,
                        plan->packed_scratch, stream))
    return 1;
  return lce_b200_bconv2d_run(plan, plan->packed_scratch, out_dev, stream);
}

int lce_b200_bconv2d_run_host(lce_b200_bconv2d* plan, const int32_t* in_host, void* out_host) {
  const lce_bconv2d_desc& d = plan->d;
  const size_t in_bytes =
      static_cast<size_t>(d.batch) * d.in_h * d.in_w * cdiv(d.channels_in, 32) * 4;
  const size_t out_bytes = bconv_out_bytes(plan);
  if (in_bytes > plan->h2d_bytes) {
    cudaFree(plan->h2d_in);
    plan->h2d_in = nullptr; plan->h2d_bytes = 0;
    CUDA_OK(cudaMalloc(&plan->h2d_in, in_bytes + 16));
    plan->h2d_bytes = in_bytes;
  }
  if (out_bytes > plan->d2h_bytes) {
    cudaFree(plan->d2h_out);
    plan->d2h_out = nullptr; plan->d2h_bytes = 0;
    CUDA_OK(cudaMalloc(&plan->d2h_out, out_bytes + 16));
    plan->d2h_bytes = out_bytes;
  }
  if (in_bytes) CUDA_OK(cudaMemcpyAsync(plan->h2d_in, in_host, in_bytes, cudaMemcpyHostToDevice, 0));
  if (lce_b200_bconv2d_run(plan, static_cast<const int32_t*>(plan->h2d_in), plan->d2h_out,
                           nullptr))
    return 1;
  if (out_bytes)
    CUDA_OK(cudaMemcpyAsync(out_host, plan->d2h_out, out_bytes, cudaMemcpyDeviceToHost, 0));
  CUDA_OK(cudaStreamSynchronize(0));
  return 0;
}

void lce_b200_bconv2d_destroy(lce_b200_bconv2d* plan) {
  if (!plan) return;
  plan->core.release();
  cudaFree(plan->packed_scratch);
  cudaFree(plan->h2d_in);
  cudaFree(plan->d2h_out);
  delete plan;
}

// ------------------------- ABC-Net binary bases -------------------------- //
struct lce_b200_bconv2d_bases {
  int M = 0, N = 0;
  lce_b200_bconv2d* geo = nullptr;   // term (0, 0)'s plan: shape, padding, clamp, K layout
  int32_t* wt = nullptr;             // [tile][M][n_slices][8][32] b1 fragments
  int32_t* wpop = nullptr;           // [M][ldc]
  float* tmul = nullptr;             // [M * N][ldc]
  float* tbias = nullptr;
  int ldc = 0, chunk_slices = 0, chunks = 1, reuse = 1;
  size_t smem = 0;
  unsigned w_bytes = 0;
  ~lce_b200_bconv2d_bases() {
    lce_b200_bconv2d_destroy(geo);
    cudaFree(wt); cudaFree(wpop); cudaFree(tmul); cudaFree(tbias);
  }
};

int lce_b200_bconv2d_bases_create(int m_bases, int n_planes, const lce_bconv2d_desc* terms,
                                  const int32_t* const* filters, const float* const* post_mul,
                                  const float* const* post_bias, lce_b200_bconv2d_bases** out_plan) {
  *out_plan = nullptr;
  if (lce_b200_device_count() < 1) return fail("no CUDA device: this library has no CPU path");
  if (!terms || !filters || !post_mul || !post_bias) return fail("bconv2d_bases: null argument");
  const lce_bconv2d_desc& d = terms[0];
  int oh, ow, ph, pw;
  if (lce_b200_bconv2d_out_shape(&d, &oh, &ow, &ph, &pw)) return 1;
  if (const char* why = bases_refusal(d, m_bases, n_planes))
    return fail("bconv2d_bases: the terms must be %s", why);
  const int T = m_bases * n_planes;
  for (int t = 1; t < T; ++t)
    if (memcmp(&terms[t], &d, sizeof(d)) != 0)
      return fail("bconv2d_bases: term %d's descriptor differs from term 0's", t);
  for (int t = 0; t < T; ++t)
    if (!filters[t] || !post_mul[t] || !post_bias[t]) return fail("bconv2d_bases: term %d lacks a constant", t);
  const int cout = d.channels_out;
  const int Kw = d.filter_h * d.filter_w * (d.channels_in / 32);
  const size_t fwords = static_cast<size_t>(cout) * Kw;
  // term (n, m) must convolve with base m's filter
  {
    std::vector<int32_t> f0(fwords), fn(fwords);
    for (int m = 0; m < m_bases; ++m) {
      if (to_host(filters[m], fwords * 4, f0.data())) return 1;
      for (int n = 1; n < n_planes; ++n) {
        if (to_host(filters[n * m_bases + m], fwords * 4, fn.data())) return 1;
        if (f0 != fn) return fail("bconv2d_bases: term (%d, %d) does not share base %d's filter", n, m, m);
      }
    }
  }
  auto* plan = new lce_b200_bconv2d_bases();
  plan->M = m_bases; plan->N = n_planes;
  plan->ldc = cout + kChanPad;
  const int n_slices = cdiv(Kw, 8);
  const size_t tile_bytes = static_cast<size_t>(n_slices) * (8 * 32 * 8);
  const int tiles = cout / lce::kBN;
  plan->w_bytes = static_cast<unsigned>(tile_bytes * m_bases);
  bases_staging(n_slices, m_bases, &plan->chunk_slices, &plan->chunks, &plan->reuse, &plan->smem);
  auto cleanup = [&](int rc) {
    delete plan;
    return rc;
  };
  if (cudaMalloc(&plan->wt, static_cast<size_t>(tiles) * plan->w_bytes) != cudaSuccess ||
      cudaMalloc(&plan->wpop, static_cast<size_t>(m_bases) * plan->ldc * 4) != cudaSuccess ||
      cudaMemset(plan->wpop, 0, static_cast<size_t>(m_bases) * plan->ldc * 4) != cudaSuccess)
    return cleanup(fail("bconv2d_bases: out of device memory"));
  // each base's plan packs its fragments and popcounts; the tiles are interleaved base by base
  for (int m = 0; m < m_bases; ++m) {
    lce_b200_bconv2d* b = nullptr;
    if (lce_b200_bconv2d_create(&d, filters[m], post_mul[m], post_bias[m], nullptr, &b)) return cleanup(1);
    const GemmCore& c = b->core;
    if (c.wt_nat == nullptr || !c.imma_b1) {
      lce_b200_bconv2d_destroy(b);
      return cleanup(fail("bconv2d_bases: no b1 weight fragments"));
    }
    const bool ok =
        cudaMemcpy2D(reinterpret_cast<unsigned char*>(plan->wt) + m * tile_bytes, plan->w_bytes, c.wt_nat,
                     tile_bytes, tile_bytes, tiles, cudaMemcpyDeviceToDevice) == cudaSuccess &&
        cudaMemcpy(plan->wpop + static_cast<size_t>(m) * plan->ldc, c.wpop, static_cast<size_t>(cout) * 4,
                   cudaMemcpyDeviceToDevice) == cudaSuccess;
    if (m == 0) plan->geo = b;
    else lce_b200_bconv2d_destroy(b);
    if (!ok) return cleanup(fail("bconv2d_bases: weight copy failed"));
  }
  std::vector<float> fm(static_cast<size_t>(T) * plan->ldc, 0.f), fb(fm.size(), 0.f);
  for (int t = 0; t < T; ++t)
    if (fold_output_transform(d, post_mul[t], post_bias[t], fm.data() + static_cast<size_t>(t) * plan->ldc,
                              fb.data() + static_cast<size_t>(t) * plan->ldc))
      return cleanup(1);
  void *dm = nullptr, *db = nullptr;
  const int rc = to_device(fm.data(), fm.size() * 4, fm.size() * 4, &dm);
  plan->tmul = static_cast<float*>(dm);
  if (rc || to_device(fb.data(), fb.size() * 4, fb.size() * 4, &db)) return cleanup(1);
  plan->tbias = static_cast<float*>(db);
  *out_plan = plan;
  return 0;
}

int lce_b200_bconv2d_bases_set_input_shape(lce_b200_bconv2d_bases* plan, int batch, int in_h, int in_w) {
  return lce_b200_bconv2d_set_input_shape(plan->geo, batch, in_h, in_w);
}

int lce_b200_bconv2d_bases_get_desc(const lce_b200_bconv2d_bases* plan, lce_bconv2d_desc* d, int* out_h,
                                    int* out_w) {
  return lce_b200_bconv2d_get_desc(plan->geo, d, out_h, out_w);
}

int lce_b200_bconv2d_bases_run(lce_b200_bconv2d_bases* plan, const int32_t* const* planes_dev,
                               const float* bn_scale_dev, const float* bn_shift_dev, int bn_activation,
                               const float* residual_dev, int add_activation, float* out_dev, int n_next,
                               const float* next_shifts, int32_t* const* next_planes_dev, void* stream) {
  const lce_bconv2d_desc& d = plan->geo->d;
  const GemmCore& c = plan->geo->core;
  if (!planes_dev) return fail("bconv2d_bases_run: the input planes are required");
  if (!bn_scale_dev || !bn_shift_dev || !is_device_ptr(bn_scale_dev) || !is_device_ptr(bn_shift_dev))
    return fail("bconv2d_bases_run: the BatchNorm vectors must be device memory");
  for (int a : {bn_activation, add_activation})
    if (a < LCE_ACT_NONE || a > LCE_ACT_RELU6) return fail("bconv2d_bases_run: unknown activation %d", a);
  if (n_next < 0 || n_next > lce::kMaxBases) return fail("bconv2d_bases_run: 0 to 8 next planes");
  if (n_next > 0 && (!next_shifts || !next_planes_dev)) return fail("bconv2d_bases_run: next shifts and planes required");
  if (residual_dev && !aligned16(residual_dev)) return fail("bconv2d_bases_run: residual must be 16-byte aligned");
  if (out_dev && !aligned16(out_dev)) return fail("bconv2d_bases_run: output must be 16-byte aligned");
  const long long M = static_cast<long long>(d.batch) * plan->geo->out_h * plan->geo->out_w;
  const size_t in_bytes = static_cast<size_t>(d.batch) * d.in_h * d.in_w * (d.channels_in / 32) * 4;
  const size_t out_bytes = static_cast<size_t>(M) * d.channels_out * 4;
  const size_t pk_bytes = static_cast<size_t>(M) * (d.channels_out / 32) * 4;
  auto overlaps = [](const void* a, size_t an, const void* b, size_t bn) {
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
    return a && b && a0 < b0 + bn && b0 < a0 + an;
  };
  // CTAs gather neighbouring pixels of the planes and read the shortcut: the outputs alias neither
  for (int n = 0; n < plan->N; ++n) {
    if (!planes_dev[n]) return fail("bconv2d_bases_run: input plane %d is NULL", n);
    if ((reinterpret_cast<uintptr_t>(planes_dev[n]) & (4u * c.V - 1)) != 0)
      return fail("bconv2d_bases_run: input planes must be %d-byte aligned", 4 * c.V);
    if (overlaps(out_dev, out_bytes, planes_dev[n], in_bytes))
      return fail("bconv2d_bases_run: the output overlaps an input plane");
    for (int k = 0; k < n_next; ++k)
      if (overlaps(next_planes_dev[k], pk_bytes, planes_dev[n], in_bytes))
        return fail("bconv2d_bases_run: a next plane overlaps an input plane");
  }
  for (int k = 0; k < n_next; ++k) {
    if (!next_planes_dev[k] || (reinterpret_cast<uintptr_t>(next_planes_dev[k]) & 7u) != 0)
      return fail("bconv2d_bases_run: next planes must be 8-byte aligned");
    if (overlaps(next_planes_dev[k], pk_bytes, residual_dev, out_bytes))
      return fail("bconv2d_bases_run: a next plane overlaps the residual");
  }
  if (overlaps(out_dev, out_bytes, residual_dev, out_bytes))
    return fail("bconv2d_bases_run: output must not overlap the residual");
  lce::BasesParams bp;
  memset(&bp, 0, sizeof(bp));
  lce::ConvKParams& p = bp.p;
  p.wt = plan->wt; p.out = out_dev; p.residual = residual_dev; p.residual_act = add_activation;
  p.M = M;
  p.H = d.in_h; p.W = d.in_w;
  p.Cw_total = d.channels_in / 32; p.Cw_pg = c.Cw_pg; p.CwV = c.Cw_pg / c.V;
  p.KH = d.filter_h; p.KW = d.filter_w;
  p.sh = d.stride_h; p.sw = d.stride_w; p.dh = d.dilation_h; p.dw = d.dilation_w;
  p.ph = plan->geo->pad_h; p.pw = plan->geo->pad_w; p.OH = plan->geo->out_h; p.OW = plan->geo->out_w;
  p.cout = c.cout; p.cout_pg = c.cout; p.tiles_per_group = c.tiles_per_group;
  p.Kv = c.Kv; p.Kc_v = plan->chunk_slices * 8 / c.V; p.n_chunks = plan->chunks;
  p.clamp_min = c.clamp_min; p.clamp_max = c.clamp_max;
  p.cw_out = d.channels_out / 32;
  p.fd_ohw = lce::make_fastdiv(static_cast<uint32_t>(p.OH) * p.OW);
  p.fd_ow = lce::make_fastdiv(p.OW);
  p.fd_cwv = lce::make_fastdiv(p.CwV);
  p.fd_kw = lce::make_fastdiv(p.KW);
  p.fd_tpg = lce::make_fastdiv(p.tiles_per_group);
  p.img_words = static_cast<long long>(p.H) * p.W * p.Cw_total;
  for (int n = 0; n < plan->N; ++n) bp.planes[n] = planes_dev[n];
  bp.tmul = plan->tmul; bp.tbias = plan->tbias; bp.wpop = plan->wpop;
  bp.ldc = plan->ldc; bp.n_bases = plan->M; bp.n_planes = plan->N; bp.reuse = plan->reuse;
  bp.bn_scale = bn_scale_dev; bp.bn_shift = bn_shift_dev; bp.bn_act = bn_activation;
  bp.n_next = n_next;
  for (int k = 0; k < n_next; ++k) {
    bp.next_shift[k] = next_shifts[k];
    bp.next_planes[k] = next_planes_dev[k];
  }
  bp.w_bytes = plan->w_bytes;
  if (M == 0) return 0;
  const long long m_tiles = (M + lce::kIBM - 1) / lce::kIBM;
  if (m_tiles > INT_MAX) return fail("bconv2d_bases_run: too many output pixels");
  if (p.img_words >= (1LL << 31)) return fail("bconv2d_bases_run: input image too large (>= 2^31 packed words)");
  cudaStream_t s = as_stream(stream);
  const dim3 grid(static_cast<unsigned>(m_tiles), static_cast<unsigned>(c.tiles_per_group));
  switch (c.V) {
    case 4: return launch_bases<4>(bp, grid, plan->smem, s);
    case 2: return launch_bases<2>(bp, grid, plan->smem, s);
    default: return launch_bases<1>(bp, grid, plan->smem, s);
  }
}

void lce_b200_bconv2d_bases_destroy(lce_b200_bconv2d_bases* plan) { delete plan; }

// --------------------------------- BGEMM --------------------------------- //
int lce_b200_bgemm_create(int N, int Kw, const int32_t* W, const lce_bgemm_epilogue* ep,
                          lce_b200_bgemm** out_plan) {
  *out_plan = nullptr;
  if (lce_b200_device_count() < 1) return fail("no CUDA device: this library has no CPU path");
  if (N < 1 || Kw < 1 || !W || !ep) return fail("bgemm: bad arguments");
  if (ep->out_type < LCE_OUT_FLOAT || ep->out_type > LCE_OUT_RAW_ACC)
    return fail("bgemm: unsupported output type %d", ep->out_type);
  auto* plan = new lce_b200_bgemm();
  plan->N = N; plan->Kw = Kw;
  GemmCore& c = plan->core;
  c.groups = 1; c.cout = N; c.cout_pg = N; c.Cw_pg = Kw; c.taps = 1;
  c.out_type = ep->out_type;
  c.clamp_min = ep->clamp_min; c.clamp_max = ep->clamp_max;
  int rc = build_core_weights(&c, W, false);
  const size_t padded = static_cast<size_t>(N) + kChanPad;
  if (!rc && (ep->out_type == LCE_OUT_FLOAT || ep->out_type == LCE_OUT_INT8)) {
    if (!ep->multiplier || !ep->bias) rc = fail("bgemm: multiplier/bias missing");
    void *dm = nullptr, *db = nullptr;
    rc = rc || to_device(ep->multiplier, N * 4, padded * 4, &dm) ||
         to_device(ep->bias, N * 4, padded * 4, &db);
    c.mul = static_cast<float*>(dm);
    c.bias = static_cast<float*>(db);
  } else if (!rc && ep->out_type == LCE_OUT_BITPACKED) {
    if (!ep->thresholds) rc = fail("bgemm: thresholds missing");
    void* dt = nullptr;
    rc = rc || to_device(ep->thresholds, N * 4, padded * 4, &dt);
    c.thr = static_cast<int32_t*>(dt);
  }
  if (rc) {
    c.release();
    delete plan;
    return 1;
  }
  *out_plan = plan;
  return 0;
}

int lce_b200_bgemm_run(lce_b200_bgemm* plan, int64_t M, const int32_t* A_dev, void* out_dev,
                       void* stream) {
  GemmCore& c = plan->core;
  if (M < 0) return fail("bgemm: negative M");
  if (M == 0) return 0;
  if (M > INT_MAX) return fail("bgemm: M too large");
  lce::ConvKParams p;
  memset(&p, 0, sizeof(p));
  p.in = A_dev; p.wt = c.wt; p.out = out_dev;
  p.mul = c.mul; p.bias = c.bias; p.thr = c.thr; p.tap_popc = nullptr;
  p.M = M;
  p.H = 1; p.W = 1;  // every row of A is its own 1 x 1 "image": offsets stay 32-bit
  p.Cw_total = plan->Kw; p.Cw_pg = plan->Kw; p.CwV = plan->Kw / c.V;
  p.KH = p.KW = 1; p.sh = p.sw = p.dh = p.dw = 1; p.ph = p.pw = 0;
  p.OH = 1; p.OW = 1;
  p.cout = c.cout; p.cout_pg = c.cout_pg; p.tiles_per_group = c.tiles_per_group;
  p.Kv = c.Kv; p.Kc_v = c.Kc_v; p.n_chunks = c.n_chunks;
  p.clamp_min = c.clamp_min; p.clamp_max = c.clamp_max;
  p.cw_out = cdiv(c.cout, 32);
  if (c.out_type == LCE_OUT_INT8)
    p.vec_store = (c.cout % 8 == 0 && (reinterpret_cast<uintptr_t>(out_dev) & 7u) == 0);
  else
    p.vec_store = (c.cout % 4 == 0 && aligned16(out_dev));
  p.bp_fast = 1;
  if ((reinterpret_cast<uintptr_t>(A_dev) & (4u * c.V - 1)) != 0)
    return fail("bgemm: A must be %d-byte aligned", 4 * c.V);
  return launch_conv(c, p, as_stream(stream));
}

void lce_b200_bgemm_destroy(lce_b200_bgemm* plan) {
  if (!plan) return;
  plan->core.release();
  delete plan;
}

}  // extern "C"
