// Tensor-core linear layer for the bf16 tier (wgmma + TMA), the dense GEMMs of the path that
// are not the fused depth step:
//   W_i initialise (chemprop/nn/message_passing/mixins.py:8-9, 22-23)   K = d_v+d_e -> h
//   W_o finalize   (chemprop/nn/message_passing/base.py:180-182)        K = d_v+h   -> h
//   dX = dY . W    (autograd mirror of base.py:135-141, 180-182)        K = h       -> h
//
//   C[r, 0:N] = act( A[r, 0:K] . W^T + bias )        A, C bf16 row-major; W pre-packed bf16
//
// Persistent kernel, one CTA per SM, work item = (128-row tile, output columns [152 j, 152 j + 152)):
//   warp 0      TMA producer: per 64-wide k slab one A box (128 rows x 64, SWIZZLE_128B) + the item's rows of the W slab
//               (pre-packed shared-memory image, cp.async.bulk) into a 4-stage ring
//   warps 4-11  two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: wgmma m64n152k16 with the f32
//               accumulator in registers, then the epilogue from registers: +bias (+residual) -> act -> bf16 -> global
// HBM bytes per tile: read 128 x K x 2, write 128 x N x 2; W comes from L2.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dmpnn {
namespace lintc {

using namespace dmpnn::tc;

constexpr int kTileM = 128;
constexpr int kNT = 152;                          // output columns per work item (the wgmma N)
constexpr int kSlabBytes = kTileM * 128;          // A stage: 128 rows x 64 bf16
constexpr int kMaxN = 304;
constexpr int kMaxK = 448;                        // 7 k slabs (CGR dims: d_v + h = 406)
constexpr int kWSlabBytes = kNT * 128;            // W stage: up to 152 rows x 64 bf16 = 19456
constexpr int kStageBytes = kSlabBytes + kWSlabBytes;   // 35840 (multiple of 1024)
constexpr int kStages = 4;
constexpr int kThreads = 384;                     // producer warpgroup + 2 consumer warpgroups
constexpr int kConsumers = 256;

constexpr int kOffStage = 0;
constexpr int kOffBar = kStages * kStageBytes;
constexpr int kOffBias = kOffBar + 16 * 8;
constexpr int kSmemBytes = kOffBias + 320 * 4;
constexpr int kSmemAlloc = kSmemBytes + 1024;
static_assert(kStageBytes % 1024 == 0 && kSlabBytes % 1024 == 0, "SWIZZLE_128B buffers need 1024-byte alignment");
static_assert(kSmemAlloc <= 232448, "exceeds shared memory");

enum { B_FULL = 0, B_EMPTY = 4 };

struct Params {
  const uint8_t* Wpk;
  const float* bias;
  const __nv_bfloat16* res;   // optional residual rows (bf16, row stride ldres), added before the activation
  int64_t ldres;
  __nv_bfloat16* C;
  int64_t ldc;
  int64_t R;
  int K, N, Npad, nslab, ksteps_last, n_tiles, n_nt;
  float act_param;
};

template <int ACT, bool HAS_BIAS>
__global__ void __launch_bounds__(kThreads, 1)
k_linear_tc(const __grid_constant__ CUtensorMap tmapA, Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sStage = sbase + kOffStage, sBar = sbase + kOffBar;
  float* s_bias = reinterpret_cast<float*>(smem + kOffBias);
  const int warp = threadIdx.x >> 5;
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };
  const int n_items = p.n_tiles * p.n_nt;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar(B_FULL + i), 1);
      mbar_init(bar(B_EMPTY + i), kConsumers);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 320; i += kThreads) s_bias[i] = (HAS_BIAS && i < p.N) ? p.bias[i] : 0.f;
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer =====================
    uint32_t ks = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int t = item / p.n_nt, n0 = (item - t * p.n_nt) * kNT;
      const uint32_t wbytes = (uint32_t)min(kNT, p.Npad - n0) * 128u;
      for (int s = 0; s < p.nslab; ++s, ++ks) {
        const uint32_t st = ks % kStages, use = ks / kStages;
        mbar_wait(bar(B_EMPTY + st), (use & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(bar(B_FULL + st), kSlabBytes + wbytes);
          tma_load_2d(sStage + st * kStageBytes, &tmapA, bar(B_FULL + st), s * 64, t * kTileM);
          bulk_load(sStage + st * kStageBytes + kSlabBytes, p.Wpk + (size_t)s * p.Npad * 128 + (size_t)n0 * 128, wbytes,
                    bar(B_FULL + st));
        }
        __syncwarp();
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====================
    // W rows past the item's last column may hold stale data of an earlier stage: they only reach accumulator columns
    // that the epilogue never stores.
    const int wg = (warp - 4) >> 2;
    const int tt = threadIdx.x - 128 - wg * 128;
    const int rl = wg * 64 + acc_row0(tt), cl = acc_col0(tt);
    uint32_t ks = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int t = item / p.n_nt, n0 = (item - t * p.n_nt) * kNT;
      float acc[76];
#pragma unroll
      for (int i = 0; i < 76; ++i) acc[i] = 0.f;
      for (int s = 0; s < p.nslab; ++s, ++ks) {
        const uint32_t st = ks % kStages, use = ks / kStages;
        mbar_wait(bar(B_FULL + st), use & 1);
        const int nk = (s == p.nslab - 1) ? p.ksteps_last : 4;
        const uint64_t adesc = desc_sw128(sStage + st * kStageBytes + (uint32_t)wg * 8192u);
        const uint64_t bdesc = desc_sw128(sStage + st * kStageBytes + kSlabBytes);
        wgmma_fence();
        for (int kk = 0; kk < nk; ++kk) wgmma_bf16_n152(acc, adesc + (uint64_t)(2 * kk), bdesc + (uint64_t)(2 * kk), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
        mbar_arrive(bar(B_EMPTY + st));
      }
      // epilogue: rows rl, rl + 8 of the tile; columns n0 + 8 b + cl + {0, 1}
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t grow = (int64_t)t * kTileM + rl + 8 * h;
        if (grow >= p.R) continue;
        __nv_bfloat16* crow = p.C + grow * p.ldc;
        const __nv_bfloat16* rrow = p.res != nullptr ? p.res + grow * p.ldres : nullptr;
#pragma unroll
        for (int b = 0; b < kNT / 8; ++b) {
          const int n = n0 + 8 * b + cl;
          if (n >= p.Npad) continue;
          float z0 = acc[4 * b + 2 * h], z1 = acc[4 * b + 2 * h + 1];
          if (rrow != nullptr) {
            const uint32_t rw = __ldg(reinterpret_cast<const unsigned int*>(rrow + n));
            z0 += bf_lo(rw); z1 += bf_hi(rw);
          }
          if constexpr (HAS_BIAS) { z0 += s_bias[n]; z1 += s_bias[n + 1]; }
          uint32_t o;
          if constexpr (ACT == DMPNN_ACT_RELU) o = act_word<ACT>(pack_bf2(z0, z1), 0.f);
          else o = pack_bf2(act_t<ACT>(p.act_param, z0), act_t<ACT>(p.act_param, z1));
          *reinterpret_cast<uint32_t*>(crow + n) = o;
        }
      }
    }
  }
}

// ---- weight packing: (optionally transposed) W -> per-k-slab [Npad x 128 B] SWIZZLE_128B images ----
struct PackGeom {
  int N, K, Npad, Kpad, nslab;
};
__host__ __device__ inline PackGeom pack_geom(int64_t N, int64_t K) {
  PackGeom g;
  g.N = (int)N; g.K = (int)K;
  g.Npad = (int)((N + 15) / 16 * 16);
  g.Kpad = (int)((K + 15) / 16 * 16);
  g.nslab = (g.Kpad + 63) / 64;
  return g;
}
// B[n][k] = transpose ? W[k][n] : W[n][k]   (W row-major with row stride ldw)
__global__ void k_pack_weight_tc(const float* __restrict__ W, int64_t ldw, int transpose, PackGeom g,
                                 __nv_bfloat16* __restrict__ out) {
  const int n = blockIdx.x;  // 0 .. Npad-1
  for (int k = threadIdx.x; k < g.nslab * 64; k += blockDim.x) {
    const int s = k >> 6, kl = k & 63;
    const size_t off = (size_t)s * g.Npad * 128 + (size_t)(n >> 3) * 1024 + (n & 7) * 128 + (((kl >> 3) ^ (n & 7)) << 4) + (kl & 7) * 2;
    float v = 0.f;
    if (n < g.N && k < g.K) v = transpose ? W[(int64_t)k * ldw + n] : W[(int64_t)n * ldw + k];
    out[off >> 1] = __float2bfloat16_rn(v);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}
static bool encode_map(EncodeTiledFn enc, CUtensorMap* tmap, const void* base, int64_t cols, int64_t rows, int64_t ld) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)kTileM};
  cuuint32_t estr[2] = {1, 1};
  return enc(tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int ACT, bool HAS_BIAS>
static cudaError_t launch_variant(int grid, cudaStream_t st, const CUtensorMap& mA, const Params& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_linear_tc<ACT, HAS_BIAS>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  k_linear_tc<ACT, HAS_BIAS><<<grid, kThreads, kSmemAlloc, st>>>(mA, p);
  return cudaSuccess;
}

}  // namespace lintc
}  // namespace dmpnn

using namespace dmpnn;
using namespace dmpnn::lintc;

extern "C" int dmpnn_pack_weight_tc_bytes(int64_t N, int64_t K, size_t* bytes) {
  DMPNN_CHECK_ARG(bytes && N > 0 && K > 0 && N <= kMaxN && K <= kMaxK, "pack_weight_tc: need 0 < N <= %d, 0 < K <= %d", kMaxN, kMaxK);
  PackGeom g = pack_geom(N, K);
  *bytes = (size_t)g.nslab * g.Npad * 128;
  return 0;
}

extern "C" int dmpnn_pack_weight_tc(const float* W, int64_t ldw, int64_t N, int64_t K, int transpose, void* Wpk,
                                    void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(W && Wpk && N > 0 && K > 0 && N <= kMaxN && K <= kMaxK, "pack_weight_tc: bad args");
  PackGeom g = pack_geom(N, K);
  k_pack_weight_tc<<<g.Npad, 128, 0, st>>>(W, ldw, transpose, g, (__nv_bfloat16*)Wpk);
  DMPNN_CHECK_LAUNCH("pack_weight_tc", 1);
  return 0;
}

extern "C" int dmpnn_linear_tc_bf16(const void* A, int64_t lda, int64_t R, int64_t K, const void* Wpk, int64_t N,
                                    const float* bias, const void* res, int64_t ldres, int act, float act_param,
                                    void* Cout, int64_t ldc, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && K > 0 && K <= kMaxK && N > 0 && N <= kMaxN, "linear_tc: unsupported sizes K=%lld N=%lld",
                  (long long)K, (long long)N);
  if (R == 0) return 0;
  DMPNN_CHECK_ARG(A && Wpk && Cout, "linear_tc: null pointer");
  PackGeom g = pack_geom(N, K);
  DMPNN_CHECK_ARG(lda >= K && lda % 8 == 0 && ldc >= g.Npad && ldc % 8 == 0, "linear_tc: lda/ldc must be multiples of 8 and ldc >= %d", g.Npad);
  DMPNN_CHECK_ARG((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(Cout) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(Wpk) & 15) == 0, "linear_tc: buffers must be 16-byte aligned");
  DMPNN_CHECK_ARG(act >= DMPNN_ACT_NONE && act <= DMPNN_ACT_ELU, "linear_tc: bad activation %d", act);
  DMPNN_CHECK_ARG(res == nullptr || (ldres >= g.Npad && ldres % 8 == 0 && (reinterpret_cast<uintptr_t>(res) & 15) == 0 && res != Cout),
                  "linear_tc: residual needs ldres >= %d, a multiple of 8, 16-byte alignment, and may not alias C", g.Npad);
  EncodeTiledFn enc = get_encode_fn();
  DMPNN_CHECK_ARG(enc != nullptr, "linear_tc: cuTensorMapEncodeTiled not available from the driver");
  CUtensorMap mA;
  // A columns beyond K are zero-filled by TMA (the tensor's inner extent is exactly K)
  DMPNN_CHECK_ARG(encode_map(enc, &mA, A, K, R, lda), "linear_tc: cuTensorMapEncodeTiled failed");
  Params p;
  p.Wpk = (const uint8_t*)Wpk;
  p.bias = bias;
  p.res = (const __nv_bfloat16*)res;
  p.ldres = ldres;
  p.C = (__nv_bfloat16*)Cout;
  p.ldc = ldc;
  p.R = R;
  p.K = (int)K;
  p.N = (int)N;
  p.Npad = g.Npad;
  p.nslab = g.nslab;
  p.ksteps_last = (g.Kpad - 64 * (g.nslab - 1)) / 16;
  p.n_tiles = (int)((R + kTileM - 1) / kTileM);
  p.n_nt = (g.Npad + kNT - 1) / kNT;
  p.act_param = act_param;
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  const int items = p.n_tiles * p.n_nt;
  const int grid = items < sm_count ? items : sm_count;
  cudaError_t e = cudaErrorInvalidValue;
#define DMPNN_LAUNCH_ACT(A_)                                                                                   \
  case A_:                                                                                                     \
    e = bias ? launch_variant<A_, true>(grid, st, mA, p) : launch_variant<A_, false>(grid, st, mA, p); \
    break;
  switch (act) {
    DMPNN_LAUNCH_ACT(DMPNN_ACT_NONE)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_RELU)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_LEAKYRELU)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_TANH)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_ELU)
  }
#undef DMPNN_LAUNCH_ACT
  DMPNN_CHECK_ARG(e == cudaSuccess, "linear_tc: cannot configure %d B dynamic smem: %s", kSmemAlloc, cudaGetErrorString(e));
  DMPNN_CHECK_LAUNCH("linear_tc", 1);
  return 0;
}
