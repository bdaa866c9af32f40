// Tensor-core weight gradient of the bf16 tier:  dW[n, k] (+)= sum_r dY[r, n] * X[r, k]
// (autograd mirror of the nn.Linear layers W_i / W_h / W_o: base.py:135-141, 180-182, mixins.py:8-9).
//
// The contraction runs over ROWS, so both operands are used "MN-major": a TMA box of 64 rows x 64
// columns (SWIZZLE_128B) of the row-major dY / X matrices is exactly the canonical MN-major SW128 atom
// stack (row r = K index at 128-byte pitch, 64 contiguous columns = MN index); the tensor core transposes them.
//
//   CTA (mt, kt, slot): output rows n in [128*mt, 128*mt+128), columns k in [192*kt, 192*kt+192); loops over 64-row
//   blocks slot, slot+S, ...
//     warp 0      TMA producer: 2 dY boxes per term + up to 3 X boxes per 64-row stage, 3-stage ring
//     warps 4-11  two consumer warpgroups (output rows [0, 64) / [64, 128) of the tile): wgmma m64n64k16 with
//                 transposed operands, D[64 x 192] (registers, fp32) += dY_blk^T . X_blk; after the last block the
//                 accumulator is written as f32 partial[cta][128][Kpad] to global memory
//   a second kernel adds the partials of each mt in fixed order (deterministic) into dW.
// Up to three dY TERMS may share one launch (dW = sum_t dY_t^T X): the X boxes of a stage are loaded once and every term
// accumulates into the same registers -- the W_i gradient of the bf16 mirror, whose dH_0 is a sum of per-step terms that
// is never formed (engine.bond_backward_tc), reads X_0 once instead of once per term.
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dmpnn {
namespace wgtc {

using namespace dmpnn::tc;

constexpr int kRowsPerStage = 64;
constexpr int kBoxBytes = kRowsPerStage * 128;    // 64 rows x 64 bf16 = 8 KB
constexpr int kMaxXBoxes = 7;                     // K <= 448
constexpr int kKT = 192;                          // output columns per CTA
constexpr int kXBoxesPerTile = kKT / 64;
constexpr int kStageBytes = (2 * 3 + kXBoxesPerTile) * kBoxBytes;   // 72 KB (three terms)
constexpr int kStages = 3;
constexpr int kThreads = 384;
constexpr int kConsumers = 256;
constexpr int kOffBar = kStages * kStageBytes;    // 221184
constexpr int kSmemBytes = kOffBar + 8 * 8;
constexpr int kSmemAlloc = kSmemBytes + 1024;
static_assert(kSmemAlloc <= 232448, "exceeds shared memory");

enum { B_FULL = 0, B_EMPTY = 3 };

struct Params {
  float* partial;       // [gridDim.x][128][Kpad]
  int64_t R;
  int N, Kx, Kpad, nxb, n_mt, slots, n_blocks, n_terms;
};

__global__ void __launch_bounds__(kThreads, 1)
k_wgrad_tc(const __grid_constant__ CUtensorMap tmapY, const __grid_constant__ CUtensorMap tmapY1,
           const __grid_constant__ CUtensorMap tmapY2, const __grid_constant__ CUtensorMap tmapX, Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sBar = sbase + kOffBar;
  const int warp = threadIdx.x >> 5;
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };
  const int mt = blockIdx.x % p.n_mt, slot = blockIdx.x / p.n_mt;
  const int kt = blockIdx.y;
  const int kw = min(kKT, p.Kpad - kt * kKT);        // accumulator columns of this CTA (multiple of 16)
  const int nxb = (kw + 63) / 64;                    // X boxes per stage

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar(B_FULL + i), 1);
      mbar_init(bar(B_EMPTY + i), kConsumers);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int nt = p.n_terms;
  const uint32_t stage_tx = (uint32_t)(2 * nt + nxb) * kBoxBytes;
  const uint32_t x_off = (uint32_t)(2 * nt) * kBoxBytes;      // a stage = [2 boxes per term | X boxes]

  if (warp == 0) {
    uint32_t ks = 0;
    for (int blk = slot; blk < p.n_blocks; blk += p.slots, ++ks) {
      const uint32_t st = ks % kStages, use = ks / kStages;
      mbar_wait(bar(B_EMPTY + st), (use & 1) ^ 1);
      if (elect_one()) {
        const uint32_t base = sbase + st * kStageBytes;
        mbar_expect_tx(bar(B_FULL + st), stage_tx);
        for (int t = 0; t < nt; ++t) {
          const CUtensorMap* my = t == 0 ? &tmapY : (t == 1 ? &tmapY1 : &tmapY2);
          tma_load_2d(base + (2 * t) * kBoxBytes, my, bar(B_FULL + st), mt * 128, blk * kRowsPerStage);
          tma_load_2d(base + (2 * t + 1) * kBoxBytes, my, bar(B_FULL + st), mt * 128 + 64, blk * kRowsPerStage);
        }
        for (int xb = 0; xb < nxb; ++xb)
          tma_load_2d(base + x_off + xb * kBoxBytes, &tmapX, bar(B_FULL + st), kt * kKT + xb * 64, blk * kRowsPerStage);
      }
      __syncwarp();
    }
  } else if (warp >= 4) {
    const int wg = (warp - 4) >> 2;
    const int tt = threadIdx.x - 128 - wg * 128;
    float acc[kXBoxesPerTile][32];
#pragma unroll
    for (int b = 0; b < kXBoxesPerTile; ++b)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[b][i] = 0.f;
    uint32_t ks = 0;
    for (int blk = slot; blk < p.n_blocks; blk += p.slots, ++ks) {
      const uint32_t st = ks % kStages, use = ks / kStages;
      mbar_wait(bar(B_FULL + st), use & 1);
      const uint32_t base = sbase + st * kStageBytes;
      wgmma_fence();
      for (int t = 0; t < nt; ++t)
#pragma unroll
        for (int kk = 0; kk < kRowsPerStage / 16; ++kk) {
          const uint64_t adesc = desc_mn_sw128(base + (2 * t + wg) * kBoxBytes + kk * 2048, kBoxBytes);
#pragma unroll
          for (int b = 0; b < kXBoxesPerTile; ++b)
            if (b < nxb) wgmma_bf16_n64_mn(acc[b], adesc, desc_mn_sw128(base + x_off + b * kBoxBytes + kk * 2048, kBoxBytes), 1u);
        }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int b = 0; b < kXBoxesPerTile; ++b) acc_fence(acc[b]);
      mbar_arrive(bar(B_EMPTY + st));
    }
    // drain: rows 64 wg + acc_row0 (+8), columns 64 b + 8 j + acc_col0 (+1); zeros when this CTA had no block
    const int rl = wg * 64 + acc_row0(tt), cl = acc_col0(tt);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float* out = p.partial + ((size_t)blockIdx.x * 128 + rl + 8 * h) * p.Kpad + kt * kKT;
#pragma unroll
      for (int b = 0; b < kXBoxesPerTile; ++b)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 64 * b + 8 * j + cl;
          if (c < kw) *reinterpret_cast<float2*>(out + c) = make_float2(acc[b][4 * j + 2 * h], acc[b][4 * j + 2 * h + 1]);
        }
    }
  }
}

// dW[n, k] (+)= sum_slot partial[slot * n_mt + n/128][n % 128][k]
// block = 128 k lanes x 4 slot groups: group g sums slots g, g+4, ... (independent loads, four in flight per thread), the four
// group sums are combined in a fixed order through shared memory -- deterministic, and the ~50 serial loads per output of
// the one-thread-per-output version (9-27 us per call, six calls per step) become ~12.
__global__ void __launch_bounds__(512) k_wgrad_reduce(const float* __restrict__ partial, int slots, int n_mt, int Kpad, int N, int Kx,
                                                      float* __restrict__ dW, int64_t lddw, int accumulate) {
  __shared__ float part[4][128];
  const int n = blockIdx.x;
  const int mt = n >> 7, nl = n & 127;
  const int kx = threadIdx.x & 127, g = threadIdx.x >> 7;
  const int k = blockIdx.y * 128 + kx;
  float s0 = 0.f, s1 = 0.f;
  if (k < Kx) {
    const float* src = partial + ((size_t)mt * 128 + nl) * Kpad + k;
    const size_t step = (size_t)n_mt * 128 * Kpad;
    int sl = g;
    for (; sl + 4 < slots; sl += 8) {
      s0 += src[(size_t)sl * step];
      s1 += src[(size_t)(sl + 4) * step];
    }
    if (sl < slots) s0 += src[(size_t)sl * step];
  }
  part[g][kx] = s0 + s1;
  __syncthreads();
  if (g == 0 && k < Kx) {
    const float t = (part[0][kx] + part[1][kx]) + (part[2][kx] + part[3][kx]);
    float* o = dW + (int64_t)n * lddw + k;
    *o = accumulate ? (*o + t) : t;
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
  cuuint32_t box[2] = {64, (cuuint32_t)kRowsPerStage};
  cuuint32_t estr[2] = {1, 1};
  return enc(tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Geom {
  int Kpad, nxb, n_mt, n_kt, slots, grid;
};
static Geom geom(int64_t N, int64_t Kx) {
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (sm_count <= 0) sm_count = 132;
  }
  Geom g;
  g.Kpad = (int)((Kx + 15) / 16 * 16);
  g.nxb = (g.Kpad + 63) / 64;
  g.n_mt = (int)((N + 127) / 128);
  g.n_kt = (g.Kpad + kKT - 1) / kKT;
  g.slots = sm_count / (g.n_mt * g.n_kt);
  if (g.slots < 1) g.slots = 1;
  g.grid = g.slots * g.n_mt;
  return g;
}

}  // namespace wgtc
}  // namespace dmpnn

using namespace dmpnn;
using namespace dmpnn::wgtc;

extern "C" int dmpnn_wgrad_tc_workspace_bytes(int64_t N, int64_t Kx, size_t* bytes) {
  DMPNN_CHECK_ARG(bytes && N > 0 && N <= 384 && Kx > 0 && Kx <= 64 * kMaxXBoxes, "wgrad_tc: need 0 < N <= 384, 0 < K <= 448");
  Geom g = geom(N, Kx);
  *bytes = (size_t)g.grid * 128 * g.Kpad * sizeof(float);
  return 0;
}

extern "C" int dmpnn_wgrad_tc_multi_bf16(const void* const* dYs, int n_terms, int64_t lddy, const void* X, int64_t ldx, int64_t R,
                                         int64_t N, int64_t Kx, float* dW, int64_t lddw, int accumulate, void* workspace,
                                         void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && N <= 384 && Kx > 0 && Kx <= 64 * kMaxXBoxes, "wgrad_tc: unsupported sizes N=%lld K=%lld",
                  (long long)N, (long long)Kx);
  DMPNN_CHECK_ARG(dW && workspace && dYs, "wgrad_tc: null pointer");
  Geom g = geom(N, Kx);
  DMPNN_CHECK_ARG(n_terms >= 1 && n_terms <= 3 && 2 * n_terms + g.nxb <= 2 + kMaxXBoxes,
                  "wgrad_tc: %d terms x K=%lld do not fit a stage (2 * terms + ceil(K / 64) <= 9)", n_terms, (long long)Kx);
  DMPNN_CHECK_ARG(lddy % 8 == 0 && ldx % 8 == 0 && lddy >= N && ldx >= Kx, "wgrad_tc: lddy/ldx must be multiples of 8");
  for (int t = 0; t < n_terms; ++t)
    DMPNN_CHECK_ARG(R == 0 || (dYs[t] && (reinterpret_cast<uintptr_t>(dYs[t]) & 15) == 0), "wgrad_tc: dY operands must be 16-byte aligned");
  DMPNN_CHECK_ARG(R == 0 || (X && (reinterpret_cast<uintptr_t>(X) & 15) == 0), "wgrad_tc: operands must be 16-byte aligned");
  if (R > 0) {
    EncodeTiledFn enc = get_encode_fn();
    DMPNN_CHECK_ARG(enc != nullptr, "wgrad_tc: cuTensorMapEncodeTiled not available from the driver");
    CUtensorMap mY[3], mX;
    for (int t = 0; t < 3; ++t)
      DMPNN_CHECK_ARG(encode_map(enc, &mY[t], dYs[t < n_terms ? t : 0], N, R, lddy), "wgrad_tc: cuTensorMapEncodeTiled failed");
    DMPNN_CHECK_ARG(encode_map(enc, &mX, X, Kx, R, ldx), "wgrad_tc: cuTensorMapEncodeTiled failed");
    Params p;
    p.partial = (float*)workspace;
    p.R = R;
    p.N = (int)N;
    p.Kx = (int)Kx;
    p.Kpad = g.Kpad;
    p.nxb = g.nxb;
    p.n_mt = g.n_mt;
    p.slots = g.slots;
    p.n_blocks = (int)((R + kRowsPerStage - 1) / kRowsPerStage);
    p.n_terms = n_terms;
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(k_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
      DMPNN_CHECK_ARG(e == cudaSuccess, "wgrad_tc: cannot configure %d B dynamic smem: %s", kSmemAlloc, cudaGetErrorString(e));
      attr_set = true;
    }
    k_wgrad_tc<<<dim3((unsigned)g.grid, (unsigned)g.n_kt), kThreads, kSmemAlloc, st>>>(mY[0], mY[1], mY[2], mX, p);
  } else {
    cudaMemsetAsync(workspace, 0, (size_t)g.grid * 128 * g.Kpad * sizeof(float), st);
  }
  k_wgrad_reduce<<<dim3((unsigned)N, (unsigned)((Kx + 127) / 128)), 512, 0, st>>>((const float*)workspace, g.slots, g.n_mt, g.Kpad, (int)N, (int)Kx, dW, lddw, accumulate);
  DMPNN_CHECK_LAUNCH("wgrad_tc", 2);
  return 0;
}

extern "C" int dmpnn_wgrad_tc_bf16(const void* dY, int64_t lddy, const void* X, int64_t ldx, int64_t R, int64_t N,
                                   int64_t Kx, float* dW, int64_t lddw, int accumulate, void* workspace,
                                   void* stream_) {
  DMPNN_CHECK_ARG(R == 0 || dY, "wgrad_tc: null operand");
  const void* terms[1] = {dY};
  return dmpnn_wgrad_tc_multi_bf16(terms, 1, lddy, X, ldx, R, N, Kx, dW, lddw, accumulate, workspace, stream_);
}
