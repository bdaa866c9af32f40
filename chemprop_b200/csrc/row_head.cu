// Atom- and bond-level heads (chemprop/models/mol_atom_bond.py:237-339): the kernels that differ from the molecule-level
// head because they run over V atom rows or E directed-edge rows instead of b molecules.
//
//   dmpnn_edge_pair_mean(_bwd)   the bond predictor's average over each reverse-edge pair, (P[::2] + P[1::2]) / 2
//                                (mol_atom_bond.py:140-151), with chemprop's edge order checked on the device
//   dmpnn_regression_loss_rows   dmpnn_regression_loss (MSE / MAE / RMSE, bounded or not) spread over the whole grid
//   dmpnn_bce_loss_rows          dmpnn_bce_loss spread over the whole grid
//   dmpnn_ce_loss_rows           dmpnn_ce_loss spread over the whole grid
//   dmpnn_pinball_loss_rows      PointQuantileLoss (chemprop/nn/metrics.py:264-288) over the whole grid, at every level: it
//                                has no single-block twin, molecules run it too
//
// The _rows criteria keep their single-block twins' arguments, conventions and outputs.  Their reduction is two-phase: each
// CTA of the first launch sums a fixed contiguous chunk of the (row, task) terms into one partial in the workspace; each CTA
// of the second launch sums every partial in the same fixed order (so all of them hold the same totals), CTA 0 writes the
// loss, and every CTA writes the gradient of its own chunk.  The grid size depends on the element count only: no float
// atomics, bitwise repeatable, no host synchronisation.
#include <math_constants.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "loss_terms.cuh"

namespace dmpnn {
namespace rowhead {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 1024;
constexpr int64_t kMinChunk = 2048;      // elements per CTA at least: below that the second launch's partial sum dominates

enum RowLoss { kMse = 0, kMae = 1, kRmse = 2, kBce = 3, kCe = 4, kPinball = 5 };

struct Args {
  const float* P;
  int64_t ldp;
  const float* Y;
  int64_t ldy;
  const float* w;
  const float* tw;
  const uint8_t* lt;
  const uint8_t* gt;
  int64_t ldm;
  int64_t B;
  int T;
  int C;
  float* loss;
  float* dP;
  int64_t lddp;
  float alpha;                           // kPinball's quantile
};

// fixed-order block sum of (l, n): lanes by a shuffle tree, then the warp partials in order; every thread gets the totals
__device__ __forceinline__ void block_sum(float& l, long long& n) {
  __shared__ float s_l[kThreads / 32];
  __shared__ long long s_n[kThreads / 32];
  __shared__ float t_l;
  __shared__ long long t_n;
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_down_sync(0xffffffffu, l, o);
    n += __shfl_down_sync(0xffffffffu, n, o);
  }
  if ((threadIdx.x & 31) == 0) { s_l[threadIdx.x >> 5] = l; s_n[threadIdx.x >> 5] = n; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f;
    long long b = 0;
    for (int k = 0; k < kThreads / 32; ++k) { a += s_l[k]; b += s_n[k]; }
    t_l = a;
    t_n = b;
  }
  __syncthreads();
  l = t_l;
  n = t_n;
}

// the term of element (b, t), from the per-element functions the single-block kernels use (loss_terms.cuh)
template <int L>
__device__ __forceinline__ float term(const Args& a, int64_t b, int t, float y) {
  const float ww = (a.w ? a.w[b] : 1.f) * (a.tw ? a.tw[t] : 1.f);
  if (L == kCe) {
    const float* p = a.P + b * a.ldp + (int64_t)t * a.C;
    const int k = class_of(y, a.C);
    float mx = p[0];
    for (int c = 1; c < a.C; ++c) mx = fmaxf(mx, p[c]);
    float s = 0.f;
    for (int c = 0; c < a.C; ++c) s += expf(p[c] - mx);
    return ww * (k >= 0 ? logf(s) + mx - p[k] : CUDART_NAN_F);
  }
  const float p = a.P[b * a.ldp + t];
  if (L == kBce) return ww * bce_with_logits(p, y);
  if (L == kPinball) {
    float g;
    return ww * pinball_term(p, y, a.alpha, &g);
  }
  const float e = reg_residual(p, y, a.lt, a.gt, b * a.ldm + t);
  if (L == kMae) return ww * fabsf(e);
  return ww * e * e;
}

// phase 1: CTA k sums the terms of elements [k * chunk, (k + 1) * chunk) into part_l[k], part_n[k]
template <int L>
__global__ void __launch_bounds__(kThreads)
k_row_loss_partials(Args a, int64_t chunk, float* __restrict__ part_l, long long* __restrict__ part_n) {
  const int64_t n = a.B * (int64_t)a.T;
  const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
  float l = 0.f;
  long long c = 0;
  for (int64_t i = lo + threadIdx.x; i < hi; i += kThreads) {
    const int64_t b = i / a.T;
    const int t = (int)(i - b * a.T);
    const float y = a.Y[b * a.ldy + t];
    if (!isfinite(y)) continue;
    l += term<L>(a, b, t, y);
    ++c;
  }
  block_sum(l, c);
  if (threadIdx.x == 0) {
    part_l[blockIdx.x] = l;
    part_n[blockIdx.x] = c;
  }
}

// phase 2: every CTA sums the G partials in one fixed order (identical totals in every CTA); CTA 0 writes the loss, and CTA k
// writes dP over phase 1's chunk k
template <int L>
__global__ void __launch_bounds__(kThreads)
k_row_loss_finish(Args a, int64_t chunk, int G, const float* __restrict__ part_l, const long long* __restrict__ part_n) {
  float l = 0.f;
  long long c = 0;
  for (int k = threadIdx.x; k < G; k += kThreads) { l += part_l[k]; c += part_n[k]; }
  block_sum(l, c);
  const float mse = c > 0 ? l / (float)c : 0.f;
  const float value = L == kRmse ? sqrtf(mse) : mse;
  if (blockIdx.x == 0 && threadIdx.x == 0) a.loss[0] = value;
  if (a.dP == nullptr) return;
  const float inv_n = c > 0 ? 1.f / (float)c : 0.f;
  const float rmse_scale = L == kRmse ? (value > 0.f ? 0.5f / value : 0.f) : 1.f;
  const int64_t n = a.B * (int64_t)a.T;
  const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
  for (int64_t i = lo + threadIdx.x; i < hi; i += kThreads) {
    const int64_t b = i / a.T;
    const int t = (int)(i - b * a.T);
    const float y = a.Y[b * a.ldy + t];
    const bool m = isfinite(y);
    const float ww = (a.w ? a.w[b] : 1.f) * (a.tw ? a.tw[t] : 1.f);
    if (L == kCe) {
      const float* p = a.P + b * a.ldp + (int64_t)t * a.C;
      float* d = a.dP + b * a.lddp + (int64_t)t * a.C;
      if (!m) {
        for (int k = 0; k < a.C; ++k) d[k] = 0.f;
        continue;
      }
      const int k = class_of(y, a.C);
      const float scale = ww * inv_n;
      float mx = p[0];
      for (int q = 1; q < a.C; ++q) mx = fmaxf(mx, p[q]);
      float s = 0.f;
      for (int q = 0; q < a.C; ++q) s += expf(p[q] - mx);
      const float inv_s = 1.f / s;
      for (int q = 0; q < a.C; ++q)
        d[q] = k >= 0 ? (expf(p[q] - mx) * inv_s - (q == k ? 1.f : 0.f)) * scale : CUDART_NAN_F;
      continue;
    }
    float g = 0.f;
    if (m) {
      const float p = a.P[b * a.ldp + t];
      if (L == kBce) {
        g = (sigmoid_stable(p) - y) * ww * inv_n;
      } else if (L == kPinball) {
        pinball_term(p, y, a.alpha, &g);
        g *= ww * inv_n;
      } else {
        const float e = reg_residual(p, y, a.lt, a.gt, b * a.ldm + t);
        if (L == kMae) g = ww * (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f)) * inv_n;
        else g = 2.f * ww * e * inv_n;
        if (L == kRmse) g *= rmse_scale;
      }
    }
    a.dP[b * a.lddp + t] = g;
  }
}

// out[i, c] = (P[2i, c] + P[2i + 1, c]) / 2 where rev[2i] == 2i + 1, NaN otherwise
__global__ void __launch_bounds__(kThreads)
k_edge_pair_mean(const float* __restrict__ P, int64_t ldp, const int32_t* __restrict__ rev, int64_t pairs, int C,
                 float* __restrict__ out, int64_t ldo) {
  const int64_t n = pairs * C;
  for (int64_t k = blockIdx.x * (int64_t)kThreads + threadIdx.x; k < n; k += (int64_t)gridDim.x * kThreads) {
    const int64_t i = k / C;
    const int c = (int)(k - i * C);
    const bool ok = rev[2 * i] == 2 * i + 1;
    out[i * ldo + c] = ok ? (P[2 * i * ldp + c] + P[(2 * i + 1) * ldp + c]) * 0.5f : CUDART_NAN_F;
  }
}

__global__ void __launch_bounds__(kThreads)
k_edge_pair_mean_bwd(const float* __restrict__ G, int64_t ldg, int64_t pairs, int C, float* __restrict__ dP, int64_t lddp) {
  const int64_t n = pairs * C;
  for (int64_t k = blockIdx.x * (int64_t)kThreads + threadIdx.x; k < n; k += (int64_t)gridDim.x * kThreads) {
    const int64_t i = k / C;
    const int c = (int)(k - i * C);
    const float g = G[i * ldg + c] * 0.5f;
    dP[2 * i * lddp + c] = g;
    dP[(2 * i + 1) * lddp + c] = g;
  }
}

static int loss_blocks(int64_t n) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(kMaxBlocks, (n + kMinChunk - 1) / kMinChunk));
}

static size_t workspace_bytes(int64_t n) {
  return (size_t)loss_blocks(n) * (sizeof(long long) + sizeof(float));
}

static unsigned elementwise_blocks(int64_t n) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, 132 * 16));
}

template <int L>
static int row_loss(const char* name, const Args& a, void* workspace, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  const int64_t n = a.B * (int64_t)a.T;
  const int G = loss_blocks(n);
  const int64_t chunk = std::max<int64_t>(1, (n + G - 1) / G);
  long long* part_n = (long long*)workspace;
  float* part_l = (float*)(part_n + G);
  k_row_loss_partials<L><<<(unsigned)G, kThreads, 0, st>>>(a, chunk, part_l, part_n);
  k_row_loss_finish<L><<<a.dP ? (unsigned)G : 1u, kThreads, 0, st>>>(a, chunk, G, part_l, part_n);
  DMPNN_CHECK_LAUNCH(name, 2);
  return 0;
}

}  // namespace rowhead
}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_edge_pair_mean(const float* P, int64_t ldp, const int32_t* rev, int64_t E, int64_t C, float* out,
                                    int64_t ldo, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(E >= 0 && E % 2 == 0 && C > 0 && C <= INT32_MAX && (E == 0 || (P && rev && out)),
                  "edge_pair_mean: bad args (E must be even)");
  DMPNN_CHECK_ARG(ldp >= C && ldo >= C, "edge_pair_mean: row strides too small");
  if (E == 0) return 0;
  const int64_t pairs = E / 2;
  rowhead::k_edge_pair_mean<<<rowhead::elementwise_blocks(pairs * C), rowhead::kThreads, 0, st>>>(P, ldp, rev, pairs, (int)C,
                                                                                                  out, ldo);
  DMPNN_CHECK_LAUNCH("edge_pair_mean", 1);
  return 0;
}

extern "C" int dmpnn_edge_pair_mean_bwd(const float* G, int64_t ldg, int64_t E, int64_t C, float* dP, int64_t lddp,
                                        void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(E >= 0 && E % 2 == 0 && C > 0 && C <= INT32_MAX && (E == 0 || (G && dP)),
                  "edge_pair_mean_bwd: bad args (E must be even)");
  DMPNN_CHECK_ARG(ldg >= C && lddp >= C, "edge_pair_mean_bwd: row strides too small");
  if (E == 0) return 0;
  const int64_t pairs = E / 2;
  rowhead::k_edge_pair_mean_bwd<<<rowhead::elementwise_blocks(pairs * C), rowhead::kThreads, 0, st>>>(G, ldg, pairs, (int)C,
                                                                                                      dP, lddp);
  DMPNN_CHECK_LAUNCH("edge_pair_mean_bwd", 1);
  return 0;
}

extern "C" int dmpnn_regression_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && bytes, "regression_loss_rows_workspace_bytes: bad args");
  *bytes = rowhead::workspace_bytes(B * T);
  return 0;
}

extern "C" int dmpnn_bce_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && bytes, "bce_loss_rows_workspace_bytes: bad args");
  *bytes = rowhead::workspace_bytes(B * T);
  return 0;
}

extern "C" int dmpnn_ce_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && bytes, "ce_loss_rows_workspace_bytes: bad args");
  *bytes = rowhead::workspace_bytes(B * T);
  return 0;
}

extern "C" int dmpnn_pinball_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && bytes, "pinball_loss_rows_workspace_bytes: bad args");
  *bytes = rowhead::workspace_bytes(B * T);
  return 0;
}

extern "C" int dmpnn_regression_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                          const float* task_weights, const uint8_t* lt_mask, const uint8_t* gt_mask,
                                          int64_t ldm, int64_t B, int64_t T, int kind, float* loss, float* dP, int64_t lddp,
                                          void* workspace, void* stream) {
  DMPNN_CHECK_ARG(kind >= rowhead::kMse && kind <= rowhead::kRmse, "regression_loss_rows: unknown kind");
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && loss && workspace && (B == 0 || (P && Y)),
                  "regression_loss_rows: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T) && ((!lt_mask && !gt_mask) || ldm >= T),
                  "regression_loss_rows: row strides too small");
  const rowhead::Args a{P, ldp, Y, ldy, weights, task_weights, lt_mask, gt_mask, ldm, B, (int)T, 1, loss, dP, lddp};
  if (kind == rowhead::kMae) return rowhead::row_loss<rowhead::kMae>("regression_loss_rows", a, workspace, stream);
  if (kind == rowhead::kRmse) return rowhead::row_loss<rowhead::kRmse>("regression_loss_rows", a, workspace, stream);
  return rowhead::row_loss<rowhead::kMse>("regression_loss_rows", a, workspace, stream);
}

extern "C" int dmpnn_bce_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                   const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                                   void* workspace, void* stream) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && loss && workspace && (B == 0 || (P && Y)), "bce_loss_rows: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "bce_loss_rows: row strides too small");
  const rowhead::Args a{P, ldp, Y, ldy, weights, task_weights, nullptr, nullptr, 0, B, (int)T, 1, loss, dP, lddp};
  return rowhead::row_loss<rowhead::kBce>("bce_loss_rows", a, workspace, stream);
}

extern "C" int dmpnn_ce_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                  const float* task_weights, int64_t B, int64_t T, int64_t C, float* loss, float* dP,
                                  int64_t lddp, void* workspace, void* stream) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && C > 0 && T * C <= INT32_MAX && loss && workspace && (B == 0 || (P && Y)),
                  "ce_loss_rows: bad args");
  DMPNN_CHECK_ARG(ldp >= T * C && ldy >= T && (dP == nullptr || lddp >= T * C), "ce_loss_rows: row strides too small");
  const rowhead::Args a{P, ldp, Y, ldy, weights, task_weights, nullptr, nullptr, 0, B, (int)T, (int)C, loss, dP, lddp};
  return rowhead::row_loss<rowhead::kCe>("ce_loss_rows", a, workspace, stream);
}

extern "C" int dmpnn_pinball_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                       const float* task_weights, int64_t B, int64_t T, float alpha, float* loss, float* dP,
                                       int64_t lddp, void* workspace, void* stream) {
  DMPNN_CHECK_ARG(std::isfinite(alpha), "pinball_loss_rows: alpha must be finite");
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && loss && workspace && (B == 0 || (P && Y)),
                  "pinball_loss_rows: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "pinball_loss_rows: row strides too small");
  const rowhead::Args a{P, ldp, Y, ldy, weights, task_weights, nullptr, nullptr, 0, B, (int)T, 1, loss, dP, lddp, alpha};
  return rowhead::row_loss<rowhead::kPinball>("pinball_loss_rows", a, workspace, stream);
}
