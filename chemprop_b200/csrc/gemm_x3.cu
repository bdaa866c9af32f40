// fp32-accurate tensor-core GEMMs for the fp32 tier (BASELINE config 3: h = 600, depth 6, fp32): every product is
// evaluated as THREE tf32 wgmma passes on an error-free split of both operands,
//
//     x = x_hi + x_lo,   x_hi = rna_tf32(x),  x_lo = rna_tf32(x - x_hi)   (x - x_hi is exact in f32)
//     a . b  ~=  a_lo . b_hi + a_hi . b_lo + a_hi . b_hi                  (the a_lo . b_lo term, 2^-22 relative, is dropped)
//
// with f32 accumulation in registers: 2^-21-class relative error per product instead of tf32's 2^-11, i.e. the
// accuracy of an f32 FMA chain (the reference's ATen sgemm), at tensor-core speed.  SURVEY.md section 7, hard part 2.
//
//   dmpnn_linear_x3   C[r, 0:N] = act(A[r, 0:K] . W^T + bias + res[r, 0:N])        A, C, res f32 row-major
//        replaces chemprop/nn/message_passing/base.py:135-141 (W_h), :180-182 (W_o) and the dX GEMMs of their autograd
//   dmpnn_wgrad_x3    dW[n, k] (+)= sum_r dY[r, n] X[r, k]                          autograd of the same nn.Linear layers
//
// k_linear_x3 -- persistent, one CTA per SM, work item = (128-row tile, 128-column pass over N):
//   warps 0-3    A producers, thread = tile row: 128-byte row segment of the slab by LDG.128 (optionally through a row
//                index), split into hi / lo in registers, written as K-major SWIZZLE_128B operand tiles (generic proxy ->
//                fence.proxy.async); thread 0 also lands the pre-split, pre-swizzled {W_hi, W_lo} blocks of the 32-wide
//                k slab (cp.async.bulk)
//   warps 4-11   two consumer warpgroups (tile rows [0, 64) / [64, 128)): per stage 4 k steps x 3 products of
//                wgmma m64n128k8 (tf32), then the epilogue from registers: + bias + residual -> act -> f32 rows to global
//
// k_wgrad_x3 -- CTA (n tile of 128, k tile of 128, row slot): D[128 x 128] (registers) += dY_blk^T . X_blk over 32-row
// blocks.  tf32 wgmma reads K-major operands only, so the producers write both operands transposed (rows = n or k,
// 32 contraction rows per 128-byte line, K-major SWIZZLE_128B); partial sums per CTA, fixed-order reduce (deterministic).
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dmpnn {
namespace x3 {

using namespace dmpnn::tc;

// ------------------------------------------------------------------------------------------------------------------
// shared pieces
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rna_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}
// x -> (hi, lo), both exactly representable in tf32; hi + lo == x up to 2^-22 |x|
__device__ __forceinline__ void split1(float x, uint32_t& hi, uint32_t& lo) {
  hi = rna_tf32(x);
  lo = rna_tf32(__fsub_rn(x, __uint_as_float(hi)));
}
__device__ __forceinline__ void split4(const float4 v, uint4& hi, uint4& lo) {
  split1(v.x, hi.x, lo.x);
  split1(v.y, hi.y, lo.y);
  split1(v.z, hi.z, lo.z);
  split1(v.w, hi.w, lo.w);
}
// ------------------------------------------------------------------------------------------------------------------
// linear
// ------------------------------------------------------------------------------------------------------------------
namespace lin {
constexpr int kTileM = 128;
constexpr int kNP = 128;                      // output columns per pass
constexpr int kABytes = kTileM * 128;         // one tile x one 32-wide k slab x one of {hi, lo}: 16 KB
constexpr int kWBytes = kNP * 128;            // one of {W_hi, W_lo} of a k slab: 16 KB
constexpr int kOffAhi = 0, kOffAlo = kABytes, kOffW = 2 * kABytes;
constexpr int kStageBytes = 2 * kABytes + 2 * kWBytes;   // 64 KB
constexpr int kStages = 3;
constexpr int kThreads = 384;
constexpr int kProducerWarps = 4;
constexpr int kConsumers = 256;
constexpr int kOffBar = kStages * kStageBytes;
constexpr int kSmemBytes = kOffBar + 8 * 8;
constexpr int kSmemAlloc = kSmemBytes + 1024;
static_assert(kStageBytes % 1024 == 0, "SWIZZLE_128B operand tiles need 1024-byte alignment");
static_assert(kSmemAlloc <= 232448, "exceeds shared memory");

enum { B_FULL = 0, B_EMPTY = 3 };

struct Params {
  const float* A;
  const int32_t* idx;      // optional row gather: A row of output row r is idx[r]
  int64_t lda;
  const uint8_t* Wpk;
  const float* bias;
  const float* res;
  int64_t ldres;
  float* C;
  int64_t ldc;
  int64_t R;
  int K, N, Npad, ldc_pad, nslab, n_pass, n_tiles;
  int act;
  float act_param;
};

__global__ void __launch_bounds__(kThreads, 1) k_linear_x3(Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sBar = sbase + kOffBar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };
  const int n_items = p.n_tiles * p.n_pass;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar(B_FULL + i), 1 + kProducerWarps);   // W loader's expect_tx arrive + one arrive per producer warp
      mbar_init(bar(B_EMPTY + i), kConsumers);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < kProducerWarps) {
    // ===================== A producers (thread = tile row) + W loader (thread 0) =====================
    const int r = threadIdx.x;
    uint32_t ks = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int t = item / p.n_pass, ps = item - t * p.n_pass;
      const int64_t grow = (int64_t)t * kTileM + r;
      const bool rv = grow < p.R;
      const float* arow = nullptr;
      if (rv) arow = p.A + (p.idx ? (int64_t)__ldg(p.idx + grow) : grow) * p.lda;
      for (int s = 0; s < p.nslab; ++s, ++ks) {
        // the row segment of this slab: 8 x 16 B, all loads in flight before the stage is waited for
        float4 x[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int k0 = s * 32 + c * 4;
          x[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rv && k0 < p.K) x[c] = __ldg(reinterpret_cast<const float4*>(arow + k0));   // K % 4 == 0
        }
        const uint32_t st = ks % kStages, use = ks / kStages;
        mbar_wait(bar(B_EMPTY + st), (use & 1) ^ 1);
        const uint32_t stg = sbase + st * kStageBytes;
        if (threadIdx.x == 0) {
          mbar_expect_tx(bar(B_FULL + st), 2 * kWBytes);
          bulk_load(stg + kOffW, p.Wpk + ((size_t)ps * p.nslab + s) * (2 * kWBytes), 2 * kWBytes, bar(B_FULL + st));
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          uint4 hi, lo;
          split4(x[c], hi, lo);
          const uint32_t off = sw128_off(r, c);
          sts128(stg + kOffAhi + off, hi);
          sts128(stg + kOffAlo + off, lo);
        }
        fence_proxy_async();                        // generic-proxy writes -> visible to the tensor core's async proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(B_FULL + st));
      }
    }
  } else {
    // ===================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====================
    const int wg = (warp - 4) >> 2;
    const int tt = threadIdx.x - 128 - wg * 128;
    const int rl = wg * 64 + acc_row0(tt), cl = acc_col0(tt);
    uint32_t ks = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const int t = item / p.n_pass, ps = item - t * p.n_pass;
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
      for (int s = 0; s < p.nslab; ++s, ++ks) {
        const uint32_t st = ks % kStages, use = ks / kStages;
        mbar_wait(bar(B_FULL + st), use & 1);
        const uint32_t stg = sbase + st * kStageBytes;
        const uint64_t bhi = desc_sw128(stg + kOffW), blo = desc_sw128(stg + kOffW + kWBytes);
        const uint64_t ahi = desc_sw128(stg + kOffAhi + (uint32_t)wg * 8192u), alo = desc_sw128(stg + kOffAlo + (uint32_t)wg * 8192u);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {            // k step = 8 tf32 = 32 B of every operand row
          const uint64_t o = (uint64_t)(2 * kk);
          wgmma_tf32_n128(acc, alo + o, bhi + o, 1u);
          wgmma_tf32_n128(acc, ahi + o, blo + o, 1u);
          wgmma_tf32_n128(acc, ahi + o, bhi + o, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        acc_fence(acc);
        mbar_arrive(bar(B_EMPTY + st));
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t grow = (int64_t)t * kTileM + rl + 8 * h;
        if (grow >= p.R) continue;
        float* crow = p.C + grow * p.ldc;
        const float* rrow = p.res ? p.res + grow * p.ldres : nullptr;
#pragma unroll
        for (int b = 0; b < kNP / 8; ++b) {
          const int n = ps * kNP + 8 * b + cl;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (n + e >= p.ldc_pad) continue;
            float o = 0.f;
            if (n + e < p.N) {
              float z = acc[4 * b + 2 * h + e];
              if (rrow != nullptr) z += __ldg(rrow + n + e);
              if (p.bias != nullptr) z += __ldg(p.bias + n + e);
              o = act_apply(p.act, p.act_param, z);
            }
            crow[n + e] = o;
          }
        }
      }
    }
  }
}

// W (f32, N x K row-major, or its transpose) -> per (pass, slab): {hi block, lo block}, each 128 rows x 128 B, K-major
// SWIZZLE_128B; rows >= N and columns >= K are zero
struct PackGeom {
  int N, K, Npad, nslab, n_pass;
};
__host__ __device__ inline PackGeom pack_geom(int64_t N, int64_t K) {
  PackGeom g;
  g.N = (int)N; g.K = (int)K;
  g.Npad = (int)((N + 15) / 16 * 16);
  g.nslab = (int)((K + 31) / 32);
  g.n_pass = (g.Npad + kNP - 1) / kNP;
  return g;
}
__global__ void k_pack_weight_x3(const float* __restrict__ W, int64_t ldw, int transpose, PackGeom g, uint8_t* __restrict__ out) {
  const int n = blockIdx.x;                 // 0 .. n_pass * 128 - 1
  const int ps = n / kNP, nl = n % kNP;
  for (int k = threadIdx.x; k < g.nslab * 32; k += blockDim.x) {
    const int s = k >> 5, kl = k & 31;
    float v = 0.f;
    if (n < g.N && k < g.K) v = transpose ? W[(int64_t)k * ldw + n] : W[(int64_t)n * ldw + k];
    uint32_t hi, lo;
    split1(v, hi, lo);
    const size_t blk = ((size_t)ps * g.nslab + s) * (2 * kWBytes);
    const size_t off = (size_t)(nl >> 3) * 1024 + (nl & 7) * 128 + (((kl >> 2) ^ (nl & 7)) << 4) + (kl & 3) * 4;
    *reinterpret_cast<uint32_t*>(out + blk + off) = hi;
    *reinterpret_cast<uint32_t*>(out + blk + kWBytes + off) = lo;
  }
}
}  // namespace lin

// ------------------------------------------------------------------------------------------------------------------
// weight gradient
// ------------------------------------------------------------------------------------------------------------------
namespace wg {
constexpr int kRows = 32;                      // contraction rows per stage
constexpr int kMT = 128, kKT = 128;            // output tile: n x k
constexpr int kOpBytes = 128 * 128;            // one operand (128 rows of n or k x 32 contraction rows) x one of {hi, lo}
constexpr int kOffAhi = 0, kOffAlo = kOpBytes, kOffBhi = 2 * kOpBytes, kOffBlo = 3 * kOpBytes;
constexpr int kStageBytes = 4 * kOpBytes;      // 64 KB
constexpr int kStages = 3;
constexpr int kThreads = 384;
constexpr int kProducerWarps = 4;
constexpr int kConsumers = 256;
constexpr int kOffBar = kStages * kStageBytes;
constexpr int kSmemBytes = kOffBar + 8 * 8;
constexpr int kSmemAlloc = kSmemBytes + 1024;
static_assert(kSmemAlloc <= 232448, "exceeds shared memory");
enum { B_FULL = 0, B_EMPTY = 3 };

struct Params {
  const float* dY;
  const float* X;
  int64_t lddy, ldx, R;
  float* partial;            // [grid][128][128]
  int N, K, n_mt, n_kt, slots, n_blocks;
};

__global__ void __launch_bounds__(kThreads, 1) k_wgrad_x3(Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sBar = sbase + kOffBar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };
  const int tile = blockIdx.x % (p.n_mt * p.n_kt), slot = blockIdx.x / (p.n_mt * p.n_kt);
  const int mt = tile % p.n_mt, kt = tile / p.n_mt;
  const int n_base = mt * kMT, k_base = kt * kKT;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(bar(B_FULL + i), kProducerWarps);
      mbar_init(bar(B_EMPTY + i), kConsumers);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < kProducerWarps) {
    // producers: 32 rows x (128 dY columns + 128 X columns) = 2048 16-byte chunks per stage, 16 per thread.  A warp takes
    // one 4-column chunk of all 32 rows, so the transposed 4-byte shared-memory stores of a warp fill one 128-byte line
    // (K-major: line = output row n or k, 32 contraction rows) without bank conflicts.
    const int tid = threadIdx.x;
    uint32_t ks = 0;
    for (int blk = slot; blk < p.n_blocks; blk += p.slots, ++ks) {
      float4 x[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int q = tid + 128 * i;
        const int rr = q & 31, cc = q >> 5;
        const int64_t grow = (int64_t)blk * kRows + rr;
        x[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (grow < p.R) {
          if (cc < 32) {
            const int n = n_base + cc * 4;
            if (n < p.N) x[i] = __ldg(reinterpret_cast<const float4*>(p.dY + grow * p.lddy + n));     // N % 4 == 0
          } else {
            const int k = k_base + (cc - 32) * 4;
            if (k < p.K) x[i] = __ldg(reinterpret_cast<const float4*>(p.X + grow * p.ldx + k));        // K % 4 == 0
          }
        }
      }
      const uint32_t st = ks % kStages, use = ks / kStages;
      mbar_wait(bar(B_EMPTY + st), (use & 1) ^ 1);
      const uint32_t stg = sbase + st * kStageBytes;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int q = tid + 128 * i;
        const int rr = q & 31, cc = q >> 5;
        uint4 hi, lo;
        split4(x[i], hi, lo);
        const uint32_t hw[4] = {hi.x, hi.y, hi.z, hi.w}, lw[4] = {lo.x, lo.y, lo.z, lo.w};
        const uint32_t ohi = cc < 32 ? kOffAhi : kOffBhi, olo = cc < 32 ? kOffAlo : kOffBlo;
        const int m0 = (cc & 31) * 4;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int m = m0 + e;
          const uint32_t off = (uint32_t)((m >> 3) * 1024 + (m & 7) * 128 + (((rr >> 2) ^ (m & 7)) << 4) + (rr & 3) * 4);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + ohi + off), "r"(hw[e]) : "memory");
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg + olo + off), "r"(lw[e]) : "memory");
        }
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_FULL + st));
    }
  } else {
    const int wg = (warp - 4) >> 2;
    const int tt = threadIdx.x - 128 - wg * 128;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    uint32_t ks = 0;
    for (int blk = slot; blk < p.n_blocks; blk += p.slots, ++ks) {
      const uint32_t st = ks % kStages, use = ks / kStages;
      mbar_wait(bar(B_FULL + st), use & 1);
      const uint32_t stg = sbase + st * kStageBytes;
      const uint64_t ahi = desc_sw128(stg + kOffAhi + (uint32_t)wg * 8192u), alo = desc_sw128(stg + kOffAlo + (uint32_t)wg * 8192u);
      const uint64_t bhi = desc_sw128(stg + kOffBhi), blo = desc_sw128(stg + kOffBlo);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kRows / 8; ++kk) {        // k step = 8 contraction rows = 32 B of every operand line
        const uint64_t o = (uint64_t)(2 * kk);
        wgmma_tf32_n128(acc, alo + o, bhi + o, 1u);
        wgmma_tf32_n128(acc, ahi + o, blo + o, 1u);
        wgmma_tf32_n128(acc, ahi + o, bhi + o, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc);
      mbar_arrive(bar(B_EMPTY + st));
    }
    // drain: zeros when this CTA had no block (acc stays 0)
    const int rl = wg * 64 + acc_row0(tt), cl = acc_col0(tt);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float* out = p.partial + ((size_t)blockIdx.x * kMT + rl + 8 * h) * kKT;
#pragma unroll
      for (int b = 0; b < kKT / 8; ++b)
        *reinterpret_cast<float2*>(out + 8 * b + cl) = make_float2(acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]);
    }
  }
}

// dW[n, k] (+)= sum_slot partial[(slot * n_tiles + kt * n_mt + mt)][n % kMT][k % kKT]   (fixed order: deterministic)
__global__ void k_wgrad_x3_reduce(const float* __restrict__ partial, int slots, int n_mt, int n_kt, int N, int K,
                                  float* __restrict__ dW, int64_t lddw, int accumulate) {
  const int n = blockIdx.x;
  const int mt = n >> 7, nl = n & 127;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int kt = k / kKT, kl = k % kKT;
    float s = 0.f;
    for (int sl = 0; sl < slots; ++sl)
      s += partial[((size_t)(sl * n_mt * n_kt + kt * n_mt + mt) * kMT + nl) * kKT + kl];
    float* o = dW + (int64_t)n * lddw + k;
    *o = accumulate ? (*o + s) : s;
  }
}

struct Geom {
  int n_mt, n_kt, slots, n_blocks, grid;
};
static Geom geom(int64_t R, int64_t N, int64_t K) {
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (sm_count <= 0) sm_count = 132;
  }
  Geom g;
  g.n_mt = (int)((N + kMT - 1) / kMT);
  g.n_kt = (int)((K + kKT - 1) / kKT);
  const int64_t nb = (R + kRows - 1) / kRows;
  g.n_blocks = nb > 0x7fffffff ? 0x7fffffff : (int)nb;
  int slots = sm_count / (g.n_mt * g.n_kt);
  if (slots < 1) slots = 1;
  if (slots > g.n_blocks) slots = g.n_blocks > 0 ? g.n_blocks : 1;
  g.slots = slots;
  g.grid = g.n_mt * g.n_kt * slots;
  return g;
}
// the workspace must not depend on R (callers size it once): slots <= SM count / tiles
static size_t workspace_bytes(int64_t N, int64_t K) {
  Geom g = geom((int64_t)1 << 30, N, K);     // any R large enough to give every tile its full set of row slots
  return (size_t)g.grid * kMT * kKT * sizeof(float);
}
}  // namespace wg

}  // namespace x3
}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_pack_weight_x3_bytes(int64_t N, int64_t K, size_t* bytes) {
  DMPNN_CHECK_ARG(bytes && N > 0 && K > 0 && N <= 4096 && K <= 8192, "pack_weight_x3: need 0 < N <= 4096, 0 < K <= 8192");
  x3::lin::PackGeom g = x3::lin::pack_geom(N, K);
  *bytes = (size_t)g.n_pass * g.nslab * 2 * x3::lin::kWBytes;
  return 0;
}

extern "C" int dmpnn_pack_weight_x3(const float* W, int64_t ldw, int64_t N, int64_t K, int transpose, void* Wpk, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(W && Wpk && N > 0 && K > 0 && N <= 4096 && K <= 8192, "pack_weight_x3: bad args");
  x3::lin::PackGeom g = x3::lin::pack_geom(N, K);
  x3::lin::k_pack_weight_x3<<<g.n_pass * x3::lin::kNP, 128, 0, st>>>(W, ldw, transpose, g, (uint8_t*)Wpk);
  DMPNN_CHECK_LAUNCH("pack_weight_x3", 1);
  return 0;
}

extern "C" int dmpnn_linear_x3(const float* A, int64_t lda, const int32_t* row_idx, int64_t R, int64_t K, const void* Wpk,
                               int64_t N, const float* bias, const float* res, int64_t ldres, int act, float act_param,
                               float* Cout, int64_t ldc, int64_t ldc_pad, void* stream_) {
  using namespace x3::lin;
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && K > 0 && N > 0 && N <= 4096 && K <= 8192, "linear_x3: unsupported sizes K=%lld N=%lld", (long long)K, (long long)N);
  if (R == 0) return 0;
  DMPNN_CHECK_ARG(A && Wpk && Cout, "linear_x3: null pointer");
  DMPNN_CHECK_ARG(K % 4 == 0 && lda % 4 == 0 && lda >= K && (reinterpret_cast<uintptr_t>(A) & 15) == 0,
                  "linear_x3: A needs K %% 4 == 0, lda %% 4 == 0 and a 16-byte aligned base (K=%lld lda=%lld)", (long long)K, (long long)lda);
  DMPNN_CHECK_ARG(ldc % 4 == 0 && ldc >= N && ldc_pad >= N && ldc_pad <= ldc && (reinterpret_cast<uintptr_t>(Cout) & 15) == 0,
                  "linear_x3: C needs ldc %% 4 == 0, N <= ldc_pad <= ldc and a 16-byte aligned base");
  DMPNN_CHECK_ARG(res == nullptr || (ldres % 4 == 0 && ldres >= N && (reinterpret_cast<uintptr_t>(res) & 15) == 0 && res != Cout),
                  "linear_x3: residual needs ldres %% 4 == 0, 16-byte alignment, and may not alias C");
  DMPNN_CHECK_ARG((reinterpret_cast<uintptr_t>(Wpk) & 15) == 0, "linear_x3: packed weight must be 16-byte aligned");
  DMPNN_CHECK_ARG(act >= DMPNN_ACT_NONE && act <= DMPNN_ACT_ELU, "linear_x3: bad activation %d", act);
  PackGeom g = pack_geom(N, K);
  Params p;
  p.A = A; p.idx = row_idx; p.lda = lda;
  p.Wpk = (const uint8_t*)Wpk;
  p.bias = bias; p.res = res; p.ldres = ldres;
  p.C = Cout; p.ldc = ldc; p.R = R;
  p.K = (int)K; p.N = (int)N; p.Npad = g.Npad;
  p.ldc_pad = (int)ldc_pad;
  p.nslab = g.nslab; p.n_pass = g.n_pass;
  p.n_tiles = (int)((R + kTileM - 1) / kTileM);
  p.act = act; p.act_param = act_param;
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_linear_x3, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
    DMPNN_CHECK_ARG(e == cudaSuccess, "linear_x3: cannot configure %d B dynamic smem: %s", kSmemAlloc, cudaGetErrorString(e));
    attr_set = true;
  }
  const int items = p.n_tiles * p.n_pass;
  const int grid = items < sm_count ? items : sm_count;
  k_linear_x3<<<grid, kThreads, kSmemAlloc, st>>>(p);
  DMPNN_CHECK_LAUNCH("linear_x3", 1);
  return 0;
}

extern "C" int dmpnn_wgrad_x3_workspace_bytes(int64_t N, int64_t K, size_t* bytes) {
  DMPNN_CHECK_ARG(bytes && N > 0 && K > 0 && N <= 4096 && K <= 8192, "wgrad_x3_workspace_bytes: bad args");
  *bytes = x3::wg::workspace_bytes(N, K) + 256;
  return 0;
}

extern "C" int dmpnn_wgrad_x3(const float* dY, int64_t lddy, const float* X, int64_t ldx, int64_t R, int64_t N, int64_t K,
                              float* dW, int64_t lddw, int accumulate, void* workspace, void* stream_) {
  using namespace x3::wg;
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && K > 0 && N <= 4096 && K <= 8192, "wgrad_x3: unsupported sizes N=%lld K=%lld", (long long)N, (long long)K);
  DMPNN_CHECK_ARG(dW && workspace && lddw >= K, "wgrad_x3: null pointer / lddw");
  DMPNN_CHECK_ARG(R == 0 || (dY && X), "wgrad_x3: null operand");
  DMPNN_CHECK_ARG(N % 4 == 0 && K % 4 == 0 && lddy % 4 == 0 && ldx % 4 == 0 && lddy >= N && ldx >= K &&
                      (reinterpret_cast<uintptr_t>(dY) & 15) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0,
                  "wgrad_x3: N, K, lddy, ldx must be multiples of 4 and the operands 16-byte aligned");
  if (R == 0) {
    if (!accumulate) cudaMemset2DAsync(dW, (size_t)lddw * 4, 0, (size_t)K * 4, (size_t)N, st);
    return 0;
  }
  Geom g = geom(R, N, K);
  Params p;
  p.dY = dY; p.X = X; p.lddy = lddy; p.ldx = ldx; p.R = R;
  p.partial = (float*)workspace;
  p.N = (int)N; p.K = (int)K;
  p.n_mt = g.n_mt; p.n_kt = g.n_kt; p.slots = g.slots; p.n_blocks = g.n_blocks;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_wgrad_x3, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
    DMPNN_CHECK_ARG(e == cudaSuccess, "wgrad_x3: cannot configure %d B dynamic smem: %s", kSmemAlloc, cudaGetErrorString(e));
    attr_set = true;
  }
  k_wgrad_x3<<<g.grid, kThreads, kSmemAlloc, st>>>(p);
  k_wgrad_x3_reduce<<<(unsigned)N, 256, 0, st>>>(p.partial, g.slots, g.n_mt, g.n_kt, (int)N, (int)K, dW, lddw, accumulate);
  DMPNN_CHECK_LAUNCH("wgrad_x3", 2);
  return 0;
}
