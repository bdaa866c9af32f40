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
//
// Epilogue variants (template EPI; the pipeline above is shared by all of them):
//   kEpiBf16    C = act(acc + bias + res), bf16 store                              (dmpnn_linear_tc_bf16)
//   kEpiF32     C = act(acc + bias), f32 store of columns [0, N)                   (per-atom / per-edge read-outs)
//   kEpiMirror  C[out_row[r]] = (acc + res[res_row[r]]) * tau'(Y[out_row[r]]), bf16 store: the gradient of a read-out
//               that enters a depth loop -- GEMM, row scatter, residual gather and tau' in one pass
// The last two are reached through dmpnn_linear_tc_rows_bf16.
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
enum { kEpiBf16 = 0, kEpiF32 = 1, kEpiMirror = 2 };

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
  // kEpiF32 / kEpiMirror only
  float* Cf;                  // f32 output (kEpiF32)
  const __nv_bfloat16* Y;     // tau' source rows (kEpiMirror), row stride ldy
  int64_t ldy;
  const int32_t* out_row;     // nullable: output / Y row of A row r (identity when null)
  const int32_t* res_row;     // nullable: residual row of A row r (identity when null)
  int from_preact;            // Y holds the pre-activation instead of the activation output
  int f32_v4;                 // kEpiF32: Cf and ldc keep every row 16-byte aligned (whole runs as float4 stores)
};

template <int ACT, bool HAS_BIAS, int EPI = kEpiBf16>
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
      // epilogue: rows rl, rl + 8 of the tile.  The packed W image permutes the columns of every work item (tc::acc_out_col):
      // per 32-column group G, this thread's accumulator blocks 4 G, 4 G + 1, ... hold the run of output columns
      // n0 + acc_out_col(32 G + cl, nc) + [0, run): 8 in a full group, 4 in a 16-column tail, 2 in an 8-column tail
      // (acc_run_cols).  A 16-column tail followed by an 8-column one (nc = 152 = 4 * 32 + 16 + 8, nc = 56 = 32 + 16 + 8) adds
      // a second run of 2 from block 4 G + 2.  Word w of a run (columns n, n + 1) comes from accumulator block b0 + w.
      const int nc = min(kNT, p.Npad - n0);   // columns of this item: all < Npad
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t grow = (int64_t)t * kTileM + rl + 8 * h;
        if (grow >= p.R) continue;
        __nv_bfloat16* crow = nullptr;
        float* cfrow = nullptr;
        const __nv_bfloat16* yrow = nullptr;
        const __nv_bfloat16* rrow = nullptr;
        if constexpr (EPI == kEpiF32) {
          cfrow = p.Cf + grow * p.ldc;
        } else if constexpr (EPI == kEpiMirror) {
          const int64_t q = p.out_row != nullptr ? (int64_t)__ldg(p.out_row + grow) : grow;
          const int64_t s = p.res_row != nullptr ? (int64_t)__ldg(p.res_row + grow) : grow;
          crow = p.C + q * p.ldc;
          yrow = p.Y + q * p.ldy;
          rrow = p.res != nullptr ? p.res + s * p.ldres : nullptr;
        } else {
          crow = p.C + grow * p.ldc;
          rrow = p.res != nullptr ? p.res + grow * p.ldres : nullptr;
        }
#pragma unroll
        for (int G = 0; G < (kNT + 31) / 32; ++G) {
          const int run0 = acc_run_cols(32 * G + cl, nc);
#pragma unroll
          for (int part = 0; part < 2; ++part) {
            const int b0 = 4 * G + 2 * part;     // first accumulator block of the run
            if (b0 >= kNT / 8) break;
            const int j = 32 * G + 16 * part + cl;
            const int run = part == 0 ? run0 : (run0 == 4 ? acc_run_cols(j, nc) : 0);
            if (run == 0) continue;
            const int nw = run >> 1;             // bf16x2 words of the run
            const int n = n0 + acc_out_col(j, nc);
            uint32_t rw[4] = {0u, 0u, 0u, 0u}, yw[4] = {0u, 0u, 0u, 0u}, o[4] = {0u, 0u, 0u, 0u};
            float zf[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (EPI != kEpiF32 && rrow != nullptr) ld_run(rrow + n, nw, rw);
            if (EPI == kEpiMirror && n < p.N) ld_run(yrow + n, nw, yw);
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              const int b = b0 + w;
              if (b >= kNT / 8 || w >= nw) break;
              const int nn = n + 2 * w;
              float z0 = acc[4 * b + 2 * h], z1 = acc[4 * b + 2 * h + 1];
              if constexpr (EPI == kEpiF32) {
                if constexpr (HAS_BIAS) { z0 += s_bias[nn]; z1 += s_bias[nn + 1]; }
                zf[2 * w] = act_t<ACT>(p.act_param, z0);
                zf[2 * w + 1] = act_t<ACT>(p.act_param, z1);
              } else if constexpr (EPI == kEpiMirror) {
                if (nn < p.N) {                    // columns [N, pad16(N)) are written as zeros
                  if (rrow != nullptr) { z0 += bf_lo(rw[w]); z1 += bf_hi(rw[w]); }
                  if (p.from_preact) {
                    z0 *= act_grad_from_pre(ACT, p.act_param, bf_lo(yw[w]));
                    z1 *= act_grad_from_pre(ACT, p.act_param, bf_hi(yw[w]));
                  } else {
                    z0 *= act_grad_from_out(ACT, p.act_param, bf_lo(yw[w]));
                    z1 *= act_grad_from_out(ACT, p.act_param, bf_hi(yw[w]));
                  }
                  o[w] = pack_bf2(z0, nn + 1 < p.N ? z1 : 0.f);
                }
              } else {
                if (rrow != nullptr) { z0 += bf_lo(rw[w]); z1 += bf_hi(rw[w]); }
                if constexpr (HAS_BIAS) { z0 += s_bias[nn]; z1 += s_bias[nn + 1]; }
                if constexpr (ACT == DMPNN_ACT_RELU) o[w] = act_word<ACT>(pack_bf2(z0, z1), 0.f);
                else o[w] = pack_bf2(act_t<ACT>(p.act_param, z0), act_t<ACT>(p.act_param, z1));
              }
            }
            if constexpr (EPI == kEpiF32) {
              // f32 columns [0, N) only: whole 16-byte stores where the run lies below N and the rows are 16-byte aligned
              if (p.f32_v4 && n + run <= p.N && nw >= 2) {
                float4* dst = reinterpret_cast<float4*>(cfrow + n);
                dst[0] = make_float4(zf[0], zf[1], zf[2], zf[3]);
                if (nw == 4) dst[1] = make_float4(zf[4], zf[5], zf[6], zf[7]);
              } else {
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                  const int nn = n + 2 * w;
                  if (w >= nw || nn >= p.N) break;
                  if (nn + 1 < p.N) *reinterpret_cast<float2*>(cfrow + nn) = make_float2(zf[2 * w], zf[2 * w + 1]);
                  else cfrow[nn] = zf[2 * w];
                }
              }
            } else {
              st_run(crow + n, nw, o);
            }
          }
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
// B[n][k] = transpose ? W[k][n] : W[n][k]   (W row-major with row stride ldw).  Inside each 152-row work item, image row
// 152 i + j holds B row 152 i + acc_out_col(j, nc_i) (tc_common.cuh), so that the epilogue's fragments are column runs.
__global__ void k_pack_weight_tc(const float* __restrict__ W, int64_t ldw, int transpose, PackGeom g,
                                 __nv_bfloat16* __restrict__ out) {
  const int r = blockIdx.x;  // image row, 0 .. Npad-1
  const int n0 = r / kNT * kNT;
  const int n = n0 + acc_out_col(r - n0, min(kNT, g.Npad - n0));   // the B row (output column) it holds; zero at n >= N
  for (int k = threadIdx.x; k < g.nslab * 64; k += blockDim.x) {
    const int s = k >> 6, kl = k & 63;
    const size_t off = (size_t)s * g.Npad * 128 + (size_t)(r >> 3) * 1024 + (r & 7) * 128 + (((kl >> 3) ^ (r & 7)) << 4) + (kl & 7) * 2;
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

template <int ACT, bool HAS_BIAS, int EPI = kEpiBf16>
static cudaError_t launch_variant(int grid, cudaStream_t st, const CUtensorMap& mA, const Params& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_linear_tc<ACT, HAS_BIAS, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  k_linear_tc<ACT, HAS_BIAS, EPI><<<grid, kThreads, kSmemAlloc, st>>>(mA, p);
  return cudaSuccess;
}

static int sm_count_cached() {
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  return sm_count;
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
  p.Cf = nullptr;
  p.Y = nullptr;
  p.out_row = p.res_row = nullptr;
  p.from_preact = p.f32_v4 = 0;
  const int items = p.n_tiles * p.n_nt;
  const int sms = sm_count_cached();
  const int grid = items < sms ? items : sms;
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

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int dmpnn_linear_tc_rows_bf16(const void* A, int64_t lda, int64_t R, int64_t K, const void* Wpk, int64_t N,
                                         const float* bias, int act, float act_param, const void* Y, int64_t ldy,
                                         int from_preact, const int32_t* out_row, const void* res, int64_t ldres,
                                         const int32_t* res_row, void* Cout, int out_dtype, int64_t ldc, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && K > 0 && K <= kMaxK && N > 0 && N <= kMaxN, "linear_tc_rows: unsupported sizes K=%lld N=%lld",
                  (long long)K, (long long)N);
  DMPNN_CHECK_ARG(act >= DMPNN_ACT_NONE && act <= DMPNN_ACT_ELU, "linear_tc_rows: bad activation %d", act);
  DMPNN_CHECK_ARG(out_dtype == DMPNN_F32 || out_dtype == DMPNN_BF16, "linear_tc_rows: bad output dtype %d", out_dtype);
  if (R == 0) return 0;
  DMPNN_CHECK_ARG(A && Wpk && Cout, "linear_tc_rows: null pointer");
  PackGeom g = pack_geom(N, K);
  DMPNN_CHECK_ARG(lda >= K && lda % 8 == 0 && al16(A) && al16(Wpk), "linear_tc_rows: lda must be >= K and a multiple of 8, "
                  "A and Wpk 16-byte aligned");
  const bool mirror = Y != nullptr;
  if (mirror) {
    DMPNN_CHECK_ARG(bias == nullptr && out_dtype == DMPNN_BF16, "linear_tc_rows: the mirror mode (Y given) takes no bias and "
                    "stores bf16");
    DMPNN_CHECK_ARG(ldy >= g.Npad && ldy % 8 == 0 && al16(Y), "linear_tc_rows: Y needs ldy >= %d, a multiple of 8, 16-byte "
                    "alignment", g.Npad);
    DMPNN_CHECK_ARG(res == nullptr || (ldres >= g.Npad && ldres % 8 == 0 && al16(res) && res != Cout),
                    "linear_tc_rows: residual needs ldres >= %d, a multiple of 8, 16-byte alignment, and may not alias C", g.Npad);
    DMPNN_CHECK_ARG(res != nullptr || res_row == nullptr, "linear_tc_rows: res_row without a residual");
    DMPNN_CHECK_ARG(Y != Cout && A != Cout, "linear_tc_rows: C may not alias A or Y");
  } else {
    DMPNN_CHECK_ARG(out_row == nullptr && res == nullptr && res_row == nullptr && from_preact == 0,
                    "linear_tc_rows: row maps, residual and from_preact belong to the mirror mode (Y given)");
  }
  if (out_dtype == DMPNN_BF16) {
    DMPNN_CHECK_ARG(ldc >= g.Npad && ldc % 8 == 0 && al16(Cout), "linear_tc_rows: bf16 C needs ldc >= %d, a multiple of 8, "
                    "16-byte alignment", g.Npad);
  } else {
    DMPNN_CHECK_ARG(ldc >= N && ldc % 2 == 0 && (reinterpret_cast<uintptr_t>(Cout) & 7) == 0,
                    "linear_tc_rows: f32 C needs ldc >= N, even, and 8-byte alignment");
  }
  EncodeTiledFn enc = get_encode_fn();
  DMPNN_CHECK_ARG(enc != nullptr, "linear_tc_rows: cuTensorMapEncodeTiled not available from the driver");
  CUtensorMap mA;
  DMPNN_CHECK_ARG(encode_map(enc, &mA, A, K, R, lda), "linear_tc_rows: cuTensorMapEncodeTiled failed");
  Params p;
  p.Wpk = (const uint8_t*)Wpk;
  p.bias = bias;
  p.res = (const __nv_bfloat16*)res;
  p.ldres = ldres;
  p.C = out_dtype == DMPNN_BF16 ? (__nv_bfloat16*)Cout : nullptr;
  p.Cf = out_dtype == DMPNN_F32 ? (float*)Cout : nullptr;
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
  p.Y = (const __nv_bfloat16*)Y;
  p.ldy = ldy;
  p.out_row = out_row;
  p.res_row = res_row;
  p.from_preact = from_preact ? 1 : 0;
  p.f32_v4 = out_dtype == DMPNN_F32 && (reinterpret_cast<uintptr_t>(Cout) & 15) == 0 && ldc % 4 == 0;
  const int items = p.n_tiles * p.n_nt;
  const int sms = sm_count_cached();
  const int grid = items < sms ? items : sms;
  cudaError_t e = cudaErrorInvalidValue;
#define DMPNN_LAUNCH_ACT(A_)                                                                                    \
  case A_:                                                                                                      \
    if (mirror) e = launch_variant<A_, false, kEpiMirror>(grid, st, mA, p);                                     \
    else if (out_dtype == DMPNN_F32)                                                                            \
      e = bias ? launch_variant<A_, true, kEpiF32>(grid, st, mA, p) : launch_variant<A_, false, kEpiF32>(grid, st, mA, p); \
    else e = bias ? launch_variant<A_, true>(grid, st, mA, p) : launch_variant<A_, false>(grid, st, mA, p);     \
    break;
  switch (act) {
    DMPNN_LAUNCH_ACT(DMPNN_ACT_NONE)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_RELU)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_LEAKYRELU)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_TANH)
    DMPNN_LAUNCH_ACT(DMPNN_ACT_ELU)
  }
#undef DMPNN_LAUNCH_ACT
  DMPNN_CHECK_ARG(e == cudaSuccess, "linear_tc_rows: cannot configure %d B dynamic smem: %s", kSmemAlloc, cudaGetErrorString(e));
  DMPNN_CHECK_LAUNCH("linear_tc_rows", 1);
  return 0;
}
