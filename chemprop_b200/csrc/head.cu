// Molecule-level head of the training step (SURVEY.md section 8f-2): what follows the aggregation in
// chemprop/models/model.py:126-161 -- BatchNorm1d over the b x d fingerprints, the FFN (chemprop/nn/ffn.py:38-61; its
// GEMMs run on dmpnn_linear_fwd / dmpnn_linear_x3) and the masked, weighted MSE criterion (chemprop/nn/metrics.py:78-123,
// 139-141).  b x d is tiny next to the E x h work of the encoder: these kernels exist so that the WHOLE step is
// libdmpnn launches with no host round trip (and therefore capturable in one CUDA graph), not for their own speed.
//
//   dmpnn_bn_train_fwd   batch statistics (biased variance, two-pass, fixed summation order) + normalisation + affine, one
//                        launch; updates running_mean / running_var (momentum, unbiased variance) like nn.BatchNorm1d
//   dmpnn_bn_bwd         dX, dgamma, dbeta from the saved x_hat / invstd
//   dmpnn_mse_loss       loss = sum(w_b * tw_t * mask * (p - y)^2) / sum(mask) and dLoss/dp, NaN targets masked, one launch
//   dmpnn_bce_loss       the same reduction of binary_cross_entropy_with_logits (chemprop's BCELoss, metrics.py:291-294)
//   dmpnn_ce_loss        the same reduction of cross_entropy over groups of C logits (CrossEntropyLoss, metrics.py:297-303)
//   dmpnn_class_probs    eval-mode outputs of the classification predictors: sigmoid, or softmax per group of C columns
#include <math_constants.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace dmpnn {
namespace head {

constexpr int kWarps = 8;          // block = 8 warps x 32 lanes; lane = column of the block's 32-column strip

// column strip [32 * blockIdx.x, +32); warps stride over the rows; fixed-order reductions (deterministic)
__global__ void __launch_bounds__(kWarps * 32)
k_bn_train_fwd(const float* __restrict__ X, int64_t ldx, int64_t B, int d, const float* __restrict__ gamma,
               const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean,
               float* __restrict__ running_var, float* __restrict__ Y, int64_t ldy, float* __restrict__ Xhat, int64_t ldh,
               float* __restrict__ save_mean, float* __restrict__ save_invstd) {
  __shared__ float red[kWarps][32];
  __shared__ float s_mean[32], s_inv[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * 32 + lane;
  const bool cv = c < d;
  // pass 1: mean
  float s = 0.f;
  for (int64_t r = warp; r < B; r += kWarps) s += cv ? X[r * ldx + c] : 0.f;
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[w][lane];
    s_mean[lane] = t / (float)B;
  }
  __syncthreads();
  const float mean = s_mean[lane];
  // pass 2: variance around the mean (the strip is L2-resident)
  float q = 0.f;
  for (int64_t r = warp; r < B; r += kWarps) {
    const float dlt = cv ? X[r * ldx + c] - mean : 0.f;
    q = fmaf(dlt, dlt, q);
  }
  __syncthreads();
  red[warp][lane] = q;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) t += red[w][lane];
    const float var = t / (float)B;                       // biased: what normalises the batch
    s_inv[lane] = rsqrtf(var + eps);
    if (cv) {
      save_mean[c] = mean;
      save_invstd[c] = s_inv[lane];
      if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      if (running_var) running_var[c] = (1.f - momentum) * running_var[c] + momentum * (B > 1 ? t / (float)(B - 1) : var);
    }
  }
  __syncthreads();
  const float inv = s_inv[lane];
  const float g = (cv && gamma) ? gamma[c] : 1.f, bt = (cv && beta) ? beta[c] : 0.f;
  for (int64_t r = warp; r < B; r += kWarps) {
    if (!cv) continue;
    const float xh = (X[r * ldx + c] - mean) * inv;
    Xhat[r * ldh + c] = xh;
    Y[r * ldy + c] = fmaf(xh, g, bt);
  }
}

__global__ void __launch_bounds__(kWarps * 32)
k_bn_bwd(const float* __restrict__ dY, int64_t lddy, const float* __restrict__ Xhat, int64_t ldh, int64_t B, int d,
         const float* __restrict__ gamma, const float* __restrict__ invstd, float* __restrict__ dX, int64_t lddx,
         float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float red1[kWarps][32], red2[kWarps][32];
  __shared__ float s_sdy[32], s_sdyx[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * 32 + lane;
  const bool cv = c < d;
  float a = 0.f, b = 0.f;
  for (int64_t r = warp; r < B; r += kWarps) {
    if (!cv) continue;
    const float g = dY[r * lddy + c];
    a += g;
    b = fmaf(g, Xhat[r * ldh + c], b);
  }
  red1[warp][lane] = a;
  red2[warp][lane] = b;
  __syncthreads();
  if (warp == 0) {
    float ta = 0.f, tb = 0.f;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) { ta += red1[w][lane]; tb += red2[w][lane]; }
    s_sdy[lane] = ta;
    s_sdyx[lane] = tb;
    if (cv) {
      if (dbeta) dbeta[c] = ta;
      if (dgamma) dgamma[c] = tb;
    }
  }
  __syncthreads();
  if (!cv) return;
  const float sdy = s_sdy[lane], sdyx = s_sdyx[lane];
  const float k = (gamma ? gamma[c] : 1.f) * invstd[c] / (float)B;
  for (int64_t r = warp; r < B; r += kWarps)
    dX[r * lddx + c] = k * ((float)B * dY[r * lddy + c] - sdy - Xhat[r * ldh + c] * sdyx);
}

// one block: loss[0] = sum_{b,t} w_b tw_t m_bt (p - y)^2 / sum m,  dP = 2 w tw m (p - y) / sum m   (m = isfinite(y))
__global__ void __launch_bounds__(1024)
k_mse_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ w,
           const float* __restrict__ tw, int64_t B, int T, float* __restrict__ loss, float* __restrict__ dP, int64_t lddp) {
  __shared__ float s_l[32], s_n[32];
  __shared__ float s_tot[2];
  const int64_t n = B * (int64_t)T;
  float l = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float y = Y[b * ldy + t];
    if (isfinite(y)) {
      const float e = P[b * ldp + t] - y;
      l = fmaf((w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * e, e, l);
      cnt += 1.f;
    }
  }
  // fixed-order block reduction: lanes (shuffle tree), then the 32 warp partials in order
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_down_sync(0xffffffffu, l, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0) { s_l[threadIdx.x >> 5] = l; s_n[threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tn = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { tl += s_l[k]; tn += s_n[k]; }
    s_tot[0] = tl;
    s_tot[1] = tn;
    loss[0] = tn > 0.f ? tl / tn : 0.f;
  }
  __syncthreads();
  const float inv_n = s_tot[1] > 0.f ? 1.f / s_tot[1] : 0.f;
  if (dP != nullptr)
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t b = i / T;
      const int t = (int)(i - b * T);
      const float y = Y[b * ldy + t];
      dP[b * lddp + t] = isfinite(y) ? 2.f * (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * (P[b * ldp + t] - y) * inv_n : 0.f;
    }
}

// fixed-order sum of (l, cnt) over a block of up to 1024 threads; every thread gets {sum l, sum cnt}
__device__ __forceinline__ float2 block_sum2(float l, float cnt) {
  __shared__ float s_l[32], s_n[32];
  __shared__ float2 s_tot;
  for (int o = 16; o > 0; o >>= 1) {
    l += __shfl_down_sync(0xffffffffu, l, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0) { s_l[threadIdx.x >> 5] = l; s_n[threadIdx.x >> 5] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float tl = 0.f, tn = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { tl += s_l[k]; tn += s_n[k]; }
    s_tot = make_float2(tl, tn);
  }
  __syncthreads();
  return s_tot;
}

// binary_cross_entropy_with_logits as torch computes it: (1 - y) x + mx + log(e^{-mx} + e^{-x-mx}), mx = max(-x, 0)
__device__ __forceinline__ float bce_with_logits(float x, float y) {
  const float mx = fmaxf(-x, 0.f);
  return (1.f - y) * x + mx + logf(expf(-mx) + expf(-x - mx));
}

__device__ __forceinline__ float sigmoid_stable(float x) {
  if (x >= 0.f) return 1.f / (1.f + expf(-x));
  const float e = expf(x);
  return e / (1.f + e);
}

// one block: loss[0] = sum_{b,t} w_b tw_t m_bt bce(p, y) / sum m,  dP = (sigmoid(p) - y) w tw m / sum m   (m = isfinite(y))
__global__ void __launch_bounds__(1024)
k_bce_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ w,
           const float* __restrict__ tw, int64_t B, int T, float* __restrict__ loss, float* __restrict__ dP, int64_t lddp) {
  const int64_t n = B * (int64_t)T;
  float l = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float y = Y[b * ldy + t];
    if (isfinite(y)) {
      l = fmaf((w ? w[b] : 1.f) * (tw ? tw[t] : 1.f), bce_with_logits(P[b * ldp + t], y), l);
      cnt += 1.f;
    }
  }
  const float2 tot = block_sum2(l, cnt);
  if (threadIdx.x == 0) loss[0] = tot.y > 0.f ? tot.x / tot.y : 0.f;
  const float inv_n = tot.y > 0.f ? 1.f / tot.y : 0.f;
  if (dP != nullptr)
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t b = i / T;
      const int t = (int)(i - b * T);
      const float y = Y[b * ldy + t];
      dP[b * lddp + t] = isfinite(y)
          ? (sigmoid_stable(P[b * ldp + t]) - y) * (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * inv_n : 0.f;
    }
}

// class index of a finite label as torch's `.long()` truncates it; -1 when outside [0, C)
__device__ __forceinline__ int class_of(float y, int C) {
  const float k = truncf(y);
  return (k >= 0.f && k < (float)C) ? (int)k : -1;
}

// one block; row (b, t) = logits P[b, t*C : (t+1)*C].  loss[0] = sum w_b tw_t m_bt (lse(row) - row[label]) / sum m,
// dP row = (softmax(row) - onehot(label)) w tw m / sum m.  A finite label outside [0, C) makes its term and its dP row NaN.
__global__ void __launch_bounds__(1024)
k_ce_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ w,
          const float* __restrict__ tw, int64_t B, int T, int C, float* __restrict__ loss, float* __restrict__ dP,
          int64_t lddp) {
  const int64_t n = B * (int64_t)T;
  float l = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float y = Y[b * ldy + t];
    if (!isfinite(y)) continue;
    const float* p = P + b * ldp + (int64_t)t * C;
    const int k = class_of(y, C);
    float mx = p[0];
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, p[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(p[c] - mx);
    const float li = k >= 0 ? logf(s) + mx - p[k] : CUDART_NAN_F;
    l = fmaf((w ? w[b] : 1.f) * (tw ? tw[t] : 1.f), li, l);
    cnt += 1.f;
  }
  const float2 tot = block_sum2(l, cnt);
  if (threadIdx.x == 0) loss[0] = tot.y > 0.f ? tot.x / tot.y : 0.f;
  const float inv_n = tot.y > 0.f ? 1.f / tot.y : 0.f;
  if (dP != nullptr)
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t b = i / T;
      const int t = (int)(i - b * T);
      const float y = Y[b * ldy + t];
      const float* p = P + b * ldp + (int64_t)t * C;
      float* d = dP + b * lddp + (int64_t)t * C;
      if (!isfinite(y)) {
        for (int c = 0; c < C; ++c) d[c] = 0.f;
        continue;
      }
      const int k = class_of(y, C);
      const float scale = (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * inv_n;
      float mx = p[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, p[c]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(p[c] - mx);
      const float inv_s = 1.f / s;
      for (int c = 0; c < C; ++c)
        d[c] = k >= 0 ? (expf(p[c] - mx) * inv_s - (c == k ? 1.f : 0.f)) * scale : CUDART_NAN_F;
    }
}

// one thread per (b, t) group of C columns: sigmoid of every entry (softmax == 0) or the group's softmax
__global__ void __launch_bounds__(256)
k_class_probs(const float* __restrict__ P, int64_t ldp, int64_t B, int T, int C, int softmax, float* __restrict__ out,
              int64_t ldo) {
  const int64_t n = B * (int64_t)T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float* p = P + b * ldp + (int64_t)t * C;
    float* o = out + b * ldo + (int64_t)t * C;
    if (!softmax) {
      for (int c = 0; c < C; ++c) o[c] = sigmoid_stable(p[c]);
      continue;
    }
    float mx = p[0];
    for (int c = 1; c < C; ++c) mx = fmaxf(mx, p[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(p[c] - mx);
    const float inv_s = 1.f / s;
    for (int c = 0; c < C; ++c) o[c] = expf(p[c] - mx) * inv_s;
  }
}

}  // namespace head
}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_bn_train_fwd(const float* X, int64_t ldx, int64_t B, int64_t d, const float* gamma, const float* beta,
                                  float eps, float momentum, float* running_mean, float* running_var, float* Y, int64_t ldy,
                                  float* Xhat, int64_t ldh, float* save_mean, float* save_invstd, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B > 0 && d > 0 && X && Y && Xhat && save_mean && save_invstd, "bn_train_fwd: bad args (B must be >= 1)");
  DMPNN_CHECK_ARG(ldx >= d && ldy >= d && ldh >= d, "bn_train_fwd: row strides too small");
  head::k_bn_train_fwd<<<(unsigned)((d + 31) / 32), head::kWarps * 32, 0, st>>>(X, ldx, B, (int)d, gamma, beta, eps, momentum,
                                                                              running_mean, running_var, Y, ldy, Xhat, ldh,
                                                                              save_mean, save_invstd);
  DMPNN_CHECK_LAUNCH("bn_train_fwd", 1);
  return 0;
}

extern "C" int dmpnn_bn_bwd(const float* dY, int64_t lddy, const float* Xhat, int64_t ldh, int64_t B, int64_t d,
                            const float* gamma, const float* invstd, float* dX, int64_t lddx, float* dgamma, float* dbeta,
                            void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B > 0 && d > 0 && dY && Xhat && invstd && dX, "bn_bwd: bad args");
  DMPNN_CHECK_ARG(lddy >= d && ldh >= d && lddx >= d, "bn_bwd: row strides too small");
  head::k_bn_bwd<<<(unsigned)((d + 31) / 32), head::kWarps * 32, 0, st>>>(dY, lddy, Xhat, ldh, B, (int)d, gamma, invstd, dX, lddx,
                                                                        dgamma, dbeta);
  DMPNN_CHECK_LAUNCH("bn_bwd", 1);
  return 0;
}

extern "C" int dmpnn_mse_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                              const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                              void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && loss && (B == 0 || (P && Y)), "mse_loss: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "mse_loss: row strides too small");
  head::k_mse_loss<<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, B, (int)T, loss, dP, lddp);
  DMPNN_CHECK_LAUNCH("mse_loss", 1);
  return 0;
}

extern "C" int dmpnn_bce_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                              const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                              void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && loss && (B == 0 || (P && Y)), "bce_loss: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "bce_loss: row strides too small");
  head::k_bce_loss<<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, B, (int)T, loss, dP, lddp);
  DMPNN_CHECK_LAUNCH("bce_loss", 1);
  return 0;
}

extern "C" int dmpnn_ce_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                             const float* task_weights, int64_t B, int64_t T, int64_t C, float* loss, float* dP, int64_t lddp,
                             void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && C > 0 && T * C <= INT32_MAX && loss && (B == 0 || (P && Y)), "ce_loss: bad args");
  DMPNN_CHECK_ARG(ldp >= T * C && ldy >= T && (dP == nullptr || lddp >= T * C), "ce_loss: row strides too small");
  head::k_ce_loss<<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, B, (int)T, (int)C, loss, dP, lddp);
  DMPNN_CHECK_LAUNCH("ce_loss", 1);
  return 0;
}

extern "C" int dmpnn_class_probs(const float* P, int64_t ldp, int64_t B, int64_t T, int64_t C, int softmax, float* out,
                                 int64_t ldo, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && C > 0 && T * C <= INT32_MAX && (softmax == 0 || softmax == 1) &&
                      (B == 0 || (P && out)), "class_probs: bad args");
  DMPNN_CHECK_ARG(ldp >= T * C && ldo >= T * C, "class_probs: row strides too small");
  if (B == 0) return 0;
  const int64_t groups = B * T;
  const unsigned blocks = (unsigned)std::min<int64_t>((groups + 255) / 256, 1024);
  head::k_class_probs<<<blocks, 256, 0, st>>>(P, ldp, B, (int)T, (int)C, softmax, out, ldo);
  DMPNN_CHECK_LAUNCH("class_probs", 1);
  return 0;
}
