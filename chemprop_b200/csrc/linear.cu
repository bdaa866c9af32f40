// fp32-accurate fused linear layers (SIMT, f32 accumulate) -- the <=1e-5 parity tier and the
// generic fallback of the engine.  Covers W_i (mixins.py:8-9,22-23), W_h (base.py:135-141),
// W_o (base.py:180-182) of the reference and the GEMMs of their autograd mirror.
//
// The A operand is never materialised: rows are assembled on the fly from up to two sources
// with optional int32 row gathers, i.e. torch.cat([V[src], E], 1) (mixins.py:9) and
// torch.cat((V, M), 1) (base.py:180) become address arithmetic inside the tile loader.
#include "common.cuh"

namespace dmpnn {

struct ASrc {
  const void* X1; const void* X2;
  const int32_t* idx1; const int32_t* idx2;
  int64_t ld1, ld2;
  int K1, K2;
};

// load 8 consecutive k of row `r` (already index-resolved base pointers) as floats
template <typename T1, typename T2>
__device__ __forceinline__ void load_a8(const T1* p1, const T2* p2, int K1, int K, int k, float (&v)[8]) {
  // fast paths: whole chunk inside one source and 16B aligned
  if (k + 8 <= K1) {
    const T1* p = p1 + k;
    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
      if constexpr (sizeof(T1) == 4) {
        float4 a = *reinterpret_cast<const float4*>(p);
        float4 b = *reinterpret_cast<const float4*>(p + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
        uint4 u = *reinterpret_cast<const uint4*>(p);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
      }
      return;
    }
  } else if (k >= K1 && k + 8 <= K) {
    const T2* p = p2 + (k - K1);
    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
      if constexpr (sizeof(T2) == 4) {
        float4 a = *reinterpret_cast<const float4*>(p);
        float4 b = *reinterpret_cast<const float4*>(p + 4);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
      } else {
        uint4 u = *reinterpret_cast<const uint4*>(p);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
      }
      return;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int kk = k + i;
    float x = 0.f;
    if (kk < K1) x = ld_as_float(p1 + kk);
    else if (kk < K) x = ld_as_float(p2 + (kk - K1));
    v[i] = x;
  }
}

constexpr int BM = 128, BN = 64, BK = 16;

template <typename T1, typename T2, typename TR, typename TC>
__global__ void __launch_bounds__(256)
k_linear_fwd(ASrc a, const float* __restrict__ W, int64_t ldw, const float* __restrict__ bias,
             const TR* __restrict__ Rres, int64_t ldr, int act, float act_param,
             TC* __restrict__ C, int64_t ldc, int ldc_pad, int64_t R, int N) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Ws[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int K1 = a.K1, K = a.K1 + a.K2;

  // A loader mapping: thread -> (row = tid/2, 8 k's at (tid&1)*8)
  const int a_row = tid >> 1, a_k = (tid & 1) * 8;
  const int64_t gr = row0 + a_row;
  const T1* p1 = nullptr;
  const T2* p2 = nullptr;
  const bool row_ok = gr < R;
  if (row_ok) {
    int64_t r1 = a.idx1 ? (int64_t)a.idx1[gr] : gr;
    p1 = reinterpret_cast<const T1*>(a.X1) + r1 * a.ld1;
    if (a.K2 > 0) {
      int64_t r2 = a.idx2 ? (int64_t)a.idx2[gr] : gr;
      p2 = reinterpret_cast<const T2*>(a.X2) + r2 * a.ld2;
    }
  }
  // W loader mapping: thread -> (n = tid/4, 4 k's at (tid&3)*4)
  const int w_n = tid >> 2, w_k = (tid & 3) * 4;
  const int gn = n0 + w_n;
  const float* wp = (gn < N) ? W + (int64_t)gn * ldw : nullptr;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    float av[8];
    if (row_ok) load_a8<T1, T2>(p1, p2, K1, K, k0 + a_k, av);
    else {
#pragma unroll
      for (int i = 0; i < 8; ++i) av[i] = 0.f;
    }
    float wv[4] = {0.f, 0.f, 0.f, 0.f};
    if (wp) {
      const float* q = wp + k0 + w_k;
      if (k0 + w_k + 4 <= K && (reinterpret_cast<uintptr_t>(q) & 15) == 0) {
        float4 t = *reinterpret_cast<const float4*>(q);
        wv[0] = t.x; wv[1] = t.y; wv[2] = t.z; wv[3] = t.w;
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) if (k0 + w_k + i < K) wv[i] = q[i];
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) As[a_k + i][a_row] = av[i];
#pragma unroll
    for (int i = 0; i < 4; ++i) Ws[w_k + i][w_n] = wv[i];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      float4 w = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
      float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float wr[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(ar[i], wr[j], acc[i][j]);
    }
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int64_t r = row0 + ty * 8 + i;
    if (r >= R) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n < N) {
        float z = acc[i][j];
        if (bias) z += bias[n];
        if (Rres) z += ld_as_float(Rres + r * ldr + n);
        st_from_float(C + r * ldc + n, act_apply(act, act_param, z));
      } else if (n < ldc_pad) {
        st_from_float(C + r * ldc + n, 0.f);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// weight gradient: partial[s][n][k] = sum_{r in split s} dY[r,n] * A[r,k]
constexpr int WN = 64, WK = 64, WR = 16;

template <typename TY, typename T1, typename T2>
__global__ void __launch_bounds__(256)
k_wgrad_partial(const TY* __restrict__ dY, int64_t lddy, ASrc a, float* __restrict__ part,
                int64_t R, int N, int64_t rows_per_split) {
  __shared__ __align__(16) float Ys[WR][WN + 4];
  __shared__ __align__(16) float As[WR][WK + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;  // tx -> k group, ty -> n group
  const int n0 = blockIdx.x * WN, k0 = blockIdx.y * WK;
  const int K1 = a.K1, K = a.K1 + a.K2;
  const int64_t r_begin = (int64_t)blockIdx.z * rows_per_split;
  const int64_t r_end = min(R, r_begin + rows_per_split);
  const int lr = tid >> 4, lc = (tid & 15) * 4;  // loader: row lr, 4 consecutive columns at lc

  // Two-level sum: a WR-row block is accumulated from zero (fmaf chain of 16 terms), the block sums are added with
  // Kahan compensation.  A plain chain over the ~1000 rows of a split has an error of ~sqrt(rows) ulps of sum|terms|,
  // which on weight gradients with heavy cancellation (reference config 1, all 500 molecules: |dW_o| up to 63, an
  // element of 0.96) exceeded the fp32 tier's 1e-4 relative bound; this keeps it at a few ulps of sum|terms|.
  float tot[4][4], comp[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { tot[i][j] = 0.f; comp[i][j] = 0.f; }

  for (int64_t rb = r_begin; rb < r_end; rb += WR) {
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    const int64_t r = rb + lr;
    float yv[4] = {0.f, 0.f, 0.f, 0.f}, av[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < r_end) {
      const TY* yp = dY + r * lddy + n0 + lc;
#pragma unroll
      for (int i = 0; i < 4; ++i) if (n0 + lc + i < N) yv[i] = ld_as_float(yp + i);
      int64_t r1 = a.idx1 ? (int64_t)a.idx1[r] : r;
      const T1* p1 = reinterpret_cast<const T1*>(a.X1) + r1 * a.ld1;
      const T2* p2 = nullptr;
      if (a.K2 > 0) {
        int64_t r2 = a.idx2 ? (int64_t)a.idx2[r] : r;
        p2 = reinterpret_cast<const T2*>(a.X2) + r2 * a.ld2;
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int kk = k0 + lc + i;
        if (kk < K1) av[i] = ld_as_float(p1 + kk);
        else if (kk < K) av[i] = ld_as_float(p2 + (kk - K1));
      }
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&Ys[lr][lc]) = make_float4(yv[0], yv[1], yv[2], yv[3]);
    *reinterpret_cast<float4*>(&As[lr][lc]) = make_float4(av[0], av[1], av[2], av[3]);
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < WR; ++rr) {
      float4 y = *reinterpret_cast<const float4*>(&Ys[rr][ty * 4]);
      float4 x = *reinterpret_cast<const float4*>(&As[rr][tx * 4]);
      float yr[4] = {y.x, y.y, y.z, y.w}, xr[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(yr[i], xr[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {                 // Kahan: tot += acc, rounding error carried in comp
        const float y = __fsub_rn(acc[i][j], comp[i][j]);
        const float t = __fadd_rn(tot[i][j], y);
        comp[i][j] = __fsub_rn(__fsub_rn(t, tot[i][j]), y);
        tot[i][j] = t;
      }
  }
  float* P = part + (int64_t)blockIdx.z * N * K;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int n = n0 + ty * 4 + i;
    if (n >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = k0 + tx * 4 + j;
      if (k < K) P[(int64_t)n * K + k] = tot[i][j];
    }
  }
}

template <typename TY>
__global__ void k_colsum_partial(const TY* __restrict__ dY, int64_t lddy, float* __restrict__ part,
                                 int64_t R, int N, int64_t rows_per_split) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const int64_t r_begin = (int64_t)blockIdx.y * rows_per_split;
  const int64_t r_end = min(R, r_begin + rows_per_split);
  float s = 0.f, c = 0.f;                           // Kahan (see k_wgrad_partial)
  for (int64_t r = r_begin; r < r_end; ++r) {
    const float y = __fsub_rn(ld_as_float(dY + r * lddy + n), c);
    const float t = __fadd_rn(s, y);
    c = __fsub_rn(__fsub_rn(t, s), y);
    s = t;
  }
  part[(int64_t)blockIdx.y * N + n] = s;
}

// column sums with 4-wide loads: block = 8 warps striding over the rows of its split, lanes over
// column quads; per-block partial reduced through shared memory (fixed order: deterministic)
template <typename TY>
__global__ void __launch_bounds__(256)
k_colsum_partial_v4(const TY* __restrict__ dY, int64_t lddy, float* __restrict__ part, int64_t R, int N,
                    int64_t rows_per_split) {
  extern __shared__ float s_part[];   // [8][Npad4]
  const int Q = N / 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r_begin = (int64_t)blockIdx.x * rows_per_split;
  const int64_t r_end = min(R, r_begin + rows_per_split);
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (q < Q) {
      int64_t r = r_begin + warp;
      for (; r + 56 < r_end; r += 64) {      // 8 independent row loads in flight per lane
        float v[8][4];
#pragma unroll
        for (int u = 0; u < 8; ++u) ld4(dY + (r + 8 * u) * lddy + 4 * q, v[u]);
#pragma unroll
        for (int u = 0; u < 8; ++u) { acc[0] += v[u][0]; acc[1] += v[u][1]; acc[2] += v[u][2]; acc[3] += v[u][3]; }
      }
      for (; r < r_end; r += 8) {
        float v[4];
        ld4(dY + r * lddy + 4 * q, v);
        acc[0] += v[0]; acc[1] += v[1]; acc[2] += v[2]; acc[3] += v[3];
      }
    }
    if (q < Q) {
#pragma unroll
      for (int i = 0; i < 4; ++i) s_part[warp * N + 4 * q + i] = acc[i];
    }
  }
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_part[w * N + n];
    part[(int64_t)blockIdx.x * N + n] = s;
  }
}

__global__ void k_reduce_splits(const float* __restrict__ part, int S, int64_t count, float* __restrict__ out,
                                int64_t inner, int64_t ld_out, int accumulate) {
  // out[(i / inner) * ld_out + i % inner] (+)= sum_s part[s*count + i]
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.f, c = 0.f;                           // Kahan over the splits (fixed order: deterministic)
  for (int k = 0; k < S; ++k) {
    const float y = __fsub_rn(part[(int64_t)k * count + i], c);
    const float t = __fadd_rn(s, y);
    c = __fsub_rn(__fsub_rn(t, s), y);
    s = t;
  }
  float* o = out + (i / inner) * ld_out + (i % inner);
  *o = accumulate ? (*o + s) : s;
}

static int wgrad_splits(int64_t R) {
  int64_t s = (R + 1023) / 1024;
  if (s < 1) s = 1;
  if (s > 296) s = 296;
  return (int)s;
}

}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_linear_fwd(const void* X1, int x1_dtype, int64_t ld1, const int32_t* idx1, int64_t K1,
                                const void* X2, int x2_dtype, int64_t ld2, const int32_t* idx2, int64_t K2,
                                const float* W, int64_t ldw, const float* bias, const void* Rres, int r_dtype,
                                int64_t ldr, int act, float act_param, void* C, int c_dtype, int64_t ldc,
                                int64_t ldc_pad, int64_t R, int64_t N, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && K1 > 0 && K2 >= 0, "linear_fwd: bad sizes R=%lld N=%lld K1=%lld K2=%lld",
                  (long long)R, (long long)N, (long long)K1, (long long)K2);
  if (R == 0) return 0;
  DMPNN_CHECK_ARG(X1 && W && C, "linear_fwd: null pointer");
  DMPNN_CHECK_ARG(K2 == 0 || X2, "linear_fwd: X2 null with K2>0");
  DMPNN_CHECK_ARG(ldc >= N && ldc_pad <= ldc, "linear_fwd: ldc/ldc_pad too small");
  if (K2 == 0) { x2_dtype = x1_dtype; }
  if (!Rres) r_dtype = c_dtype;
  ASrc a{X1, X2, idx1, idx2, ld1, ld2, (int)K1, (int)K2};
  int64_t ncols = ldc_pad > N ? ldc_pad : N;
  dim3 grid(ceil_div_i64(R, BM), ceil_div_i64(ncols, BN));
  DMPNN_DISPATCH_DTYPE(x1_dtype, T1,
    DMPNN_DISPATCH_DTYPE(x2_dtype, T2,
      DMPNN_DISPATCH_DTYPE(r_dtype, TR,
        DMPNN_DISPATCH_DTYPE(c_dtype, TC,
          k_linear_fwd<T1, T2, TR, TC><<<grid, 256, 0, st>>>(a, W, ldw, bias, (const TR*)Rres, ldr, act,
                                                             act_param, (TC*)C, ldc, (int)ldc_pad, R, (int)N);
        ))))
  DMPNN_CHECK_LAUNCH("linear_fwd", 1);
  return 0;
}

extern "C" int dmpnn_linear_wgrad_workspace_bytes(int64_t R, int64_t N, int64_t K, size_t* bytes) {
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && K > 0 && bytes, "wgrad_workspace_bytes: bad args");
  int S = wgrad_splits(R);
  *bytes = sizeof(float) * ((size_t)S * N * K + (size_t)S * N) + 256;
  return 0;
}

extern "C" int dmpnn_linear_wgrad(const void* dY, int dy_dtype, int64_t lddy, const void* X1, int x1_dtype,
                                  int64_t ld1, const int32_t* idx1, int64_t K1, const void* X2, int x2_dtype,
                                  int64_t ld2, const int32_t* idx2, int64_t K2, float* dW, int64_t lddw,
                                  float* dbias, int accumulate, int64_t R, int64_t N, void* workspace,
                                  void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && K1 > 0 && K2 >= 0, "linear_wgrad: bad sizes");
  DMPNN_CHECK_ARG(dW && workspace, "linear_wgrad: null pointer");
  DMPNN_CHECK_ARG(R == 0 || (dY && X1), "linear_wgrad: null operand");
  DMPNN_CHECK_ARG(R == 0 || K2 == 0 || X2, "linear_wgrad: X2 null with K2>0");
  const int64_t K = K1 + K2;
  if (K2 == 0) x2_dtype = x1_dtype;
  const int S = wgrad_splits(R);
  const int64_t rps = ((R + S - 1) / S + WR - 1) / WR * WR;
  float* part = (float*)workspace;
  float* bpart = part + (size_t)S * N * K;
  ASrc a{X1, X2, idx1, idx2, ld1, ld2, (int)K1, (int)K2};
  dim3 grid(ceil_div_i64(N, WN), ceil_div_i64(K, WK), S);
  DMPNN_DISPATCH_DTYPE(dy_dtype, TY,
    DMPNN_DISPATCH_DTYPE(x1_dtype, T1,
      DMPNN_DISPATCH_DTYPE(x2_dtype, T2,
        k_wgrad_partial<TY, T1, T2><<<grid, 256, 0, st>>>((const TY*)dY, lddy, a, part, R, (int)N, rps > 0 ? rps : WR);
      )))
  k_reduce_splits<<<ceil_div_i64(N * K, 256), 256, 0, st>>>(part, S, N * K, dW, K, lddw, accumulate);
  if (dbias) {
    dim3 g2(ceil_div_i64(N, 128), S);
    DMPNN_DISPATCH_DTYPE(dy_dtype, TY,
      k_colsum_partial<TY><<<g2, 128, 0, st>>>((const TY*)dY, lddy, bpart, R, (int)N, rps > 0 ? rps : WR);
    )
    k_reduce_splits<<<ceil_div_i64(N, 256), 256, 0, st>>>(bpart, S, N, dbias, N, N, accumulate);
  }
  DMPNN_CHECK_LAUNCH("linear_wgrad", dbias ? 4 : 2);
  return 0;
}

extern "C" int dmpnn_column_sum(const void* Y, int y_dtype, int64_t ldy, int64_t R, int64_t N, float* out, int accumulate,
                                void* workspace, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(R >= 0 && N > 0 && out && workspace, "column_sum: bad args");
  DMPNN_CHECK_ARG(R == 0 || Y, "column_sum: null operand");
  const int S = wgrad_splits(R);
  const int64_t rps = ((R + S - 1) / S + WR - 1) / WR * WR;
  float* bpart = (float*)workspace;
  // the 4-wide kernel keeps 8 partial rows of N floats in shared memory; it runs while they fit the 48 KB a launch gets
  // without opting in (N <= 1536), wider rows take the column-per-thread kernel
  DMPNN_DISPATCH_DTYPE(y_dtype, TY,
    if (N % 4 == 0 && 8 * N * sizeof(float) <= 48 * 1024 && vec4_ok<TY>(Y, ldy)) {
      k_colsum_partial_v4<TY><<<S, 256, 8 * N * sizeof(float), st>>>((const TY*)Y, ldy, bpart, R, (int)N, rps > 0 ? rps : WR);
    } else {
      dim3 g2(ceil_div_i64(N, 128), S);
      k_colsum_partial<TY><<<g2, 128, 0, st>>>((const TY*)Y, ldy, bpart, R, (int)N, rps > 0 ? rps : WR);
    }
  )
  k_reduce_splits<<<ceil_div_i64(N, 256), 256, 0, st>>>(bpart, S, N, out, N, N, accumulate);
  DMPNN_CHECK_LAUNCH("column_sum", 2);
  return 0;
}
