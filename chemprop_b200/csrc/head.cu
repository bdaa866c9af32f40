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
//   dmpnn_pred_transform(_bwd)  raw MLP output -> the output of the regression / MVE / evidential / quantile / Dirichlet
//                        predictors (softplus, + 1, eval-mode unscaling), and its mirror
//   dmpnn_mve_loss, dmpnn_evidential_loss, dmpnn_quantile_loss, dmpnn_dirichlet_loss
//                        the uncertainty criteria (metrics.py:202-257, 502-544, 588-613) under the same reduction, one launch
//   dmpnn_regression_loss  MSE / MAE / RMSE and their bounded variants (metrics.py:128-169); dmpnn_mse_loss is its MSE case
//   dmpnn_enrichment_loss  NLogProbEnrichment (metrics.py:616-692) on b x 1 predictions and b x 2 counts, one launch
//   dmpnn_spectral_transform(_bwd), dmpnn_sid_loss, dmpnn_wasserstein_loss
//                        SpectralFFN's output and the SID / Wasserstein criteria (predictors.py:342-376, metrics.py:547-585),
//                        one CTA per spectrum row
#include <float.h>
#include <math_constants.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "loss_terms.cuh"

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

enum RegLossKind { kMseLoss = 0, kMaeLoss = 1, kRmseLoss = 2 };

// one block: MSE  loss[0] = sum_{b,t} w_b tw_t m_bt e^2 / sum m,  dP = 2 w tw m e / sum m   (m = isfinite(y), e = p - y)
//            MAE  |e| in place of e^2, dP = w tw m sign(e) / sum m (sign(0) = 0, as torch's abs)
//            RMSE sqrt of the MSE value, dP = the MSE's dP / (2 loss) (0 where the loss is 0)
// lt / gt (nullable, row stride ldm): the bounded variants' residual (reg_residual)
__global__ void __launch_bounds__(1024)
k_regression_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy,
                  const float* __restrict__ w, const float* __restrict__ tw, const uint8_t* __restrict__ lt,
                  const uint8_t* __restrict__ gt, int64_t ldm, int64_t B, int T, int kind, float* __restrict__ loss,
                  float* __restrict__ dP, int64_t lddp) {
  __shared__ float s_l[32], s_n[32];
  __shared__ float s_tot[2];
  const int64_t n = B * (int64_t)T;
  float l = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float y = Y[b * ldy + t];
    if (isfinite(y)) {
      const float e = reg_residual(P[b * ldp + t], y, lt, gt, b * ldm + t);
      if (kind == kMaeLoss) l = fmaf((w ? w[b] : 1.f) * (tw ? tw[t] : 1.f), fabsf(e), l);
      else l = fmaf((w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * e, e, l);
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
    const float mse = tn > 0.f ? tl / tn : 0.f;
    s_tot[0] = kind == kRmseLoss ? sqrtf(mse) : mse;
    s_tot[1] = tn;
    loss[0] = s_tot[0];
  }
  __syncthreads();
  const float inv_n = s_tot[1] > 0.f ? 1.f / s_tot[1] : 0.f;
  const float rmse_scale = kind == kRmseLoss ? (s_tot[0] > 0.f ? 0.5f / s_tot[0] : 0.f) : 1.f;
  if (dP != nullptr)
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t b = i / T;
      const int t = (int)(i - b * T);
      const float y = Y[b * ldy + t];
      float g = 0.f;
      if (isfinite(y)) {
        const float e = reg_residual(P[b * ldp + t], y, lt, gt, b * ldm + t);
        if (kind == kMaeLoss)
          g = (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f)) * inv_n;
        else
          g = 2.f * (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f) * e * inv_n;
        if (kind == kRmseLoss) g *= rmse_scale;
      }
      dP[b * lddp + t] = g;
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

// ---- uncertainty predictors (chemprop/nn/predictors.py:172-228, 250-270, 319-336; nn/metrics.py:202-257, 502-544,
// 588-613) ------------------------------------------------------------------------------------------------------------
enum PredKind { kRegression = 0, kMve = 1, kEvidential = 2, kQuantile = 3, kDirichlet = 4, kDirichletProbs = 5,
                kDirichletBinary = 6, kSoftplus = 7 };

// F.softplus(x) (beta 1, threshold 20) and its derivative as torch's softplus_backward computes it
__device__ __forceinline__ float softplus20(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float softplus20_grad(float x) {
  if (x > 20.f) return 1.f;
  const float z = expf(x);
  return z / (z + 1.f);
}

// digamma and trigamma for x >= 1 (every argument the losses pass: softplus + 1, y + (1 - y) alpha, sums of those):
// the recurrence lifts x to >= 6, where the asymptotic series is below f32 resolution after the terms kept
constexpr float kPsiSwitch = 6.f;
__device__ __forceinline__ float digamma_ge1(float x) {
  float acc = 0.f;
  while (x < kPsiSwitch) { acc -= 1.f / x; x += 1.f; }
  const float r = 1.f / x, r2 = r * r;
  return acc + logf(x) - 0.5f * r - r2 * (1.f / 12.f - r2 * (1.f / 120.f - r2 * (1.f / 252.f)));
}
__device__ __forceinline__ float trigamma_ge1(float x) {
  float acc = 0.f;
  while (x < kPsiSwitch) { acc += 1.f / (x * x); x += 1.f; }
  const float r = 1.f / x, r2 = r * r;
  return acc + r * (1.f + r * (0.5f + r * (1.f / 6.f - r2 * (1.f / 30.f - r2 * (1.f / 42.f - r2 * (1.f / 30.f))))));
}

// one thread per (b, t): raw MLP output X (B x (T*u)) -> predictor output (B x T x u).  Regression family: target j of task
// t is column j*T + t (torch.chunk); Dirichlet family: class c of task t is column t*u + c (reshape).  mean / scale
// (nullable, T entries) apply UnscaleTransform's eval mode; products and sums are rounded one by one as torch does.
__global__ void __launch_bounds__(256)
k_pred_transform(const float* __restrict__ X, int64_t ldx, int64_t B, int T, int kind, int u, const float* __restrict__ mean,
                 const float* __restrict__ scale, float* __restrict__ out, int64_t ldo) {
  const int64_t n = B * (int64_t)T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float* x = X + b * ldx;
    float* o = out + b * ldo + (int64_t)t * u;
    const float s = scale ? scale[t] : 1.f, m = mean ? mean[t] : 0.f;
    const float s2 = __fmul_rn(s, s);
    auto unscale = [&](float v) { return scale ? __fadd_rn(__fmul_rn(v, s), m) : v; };
    auto unscale_var = [&](float v) { return scale ? __fmul_rn(v, s2) : v; };
    switch (kind) {
      case kRegression: o[0] = unscale(x[t]); break;
      case kSoftplus: o[0] = softplus20(x[t]); break;
      case kMve:
        o[0] = unscale(x[t]);
        o[1] = unscale_var(softplus20(x[T + t]));
        break;
      case kEvidential:
        o[0] = unscale(x[t]);
        o[1] = softplus20(x[T + t]);
        o[2] = softplus20(x[2 * T + t]) + 1.f;
        o[3] = unscale_var(softplus20(x[3 * T + t]));
        break;
      case kQuantile: {
        const float lo = unscale(x[t]), hi = unscale(x[T + t]);
        o[0] = (lo + hi) * 0.5f;
        o[1] = hi - lo;
        break;
      }
      default: {                                   // Dirichlet family: alpha = softplus + 1 per class
        const float* xr = x + (int64_t)t * u;
        if (kind == kDirichlet) {
          for (int c = 0; c < u; ++c) o[c] = softplus20(xr[c]) + 1.f;
          break;
        }
        float S = 0.f;
        for (int c = 0; c < u; ++c) S += softplus20(xr[c]) + 1.f;
        if (kind == kDirichletProbs) {
          for (int c = 0; c < u; ++c) o[c] = (softplus20(xr[c]) + 1.f) / S;
        } else {                                   // binary: (alpha_1 / S, 2 / S)
          o[0] = (softplus20(xr[1]) + 1.f) / S;
          o[1] = 2.f / S;
        }
      }
    }
  }
}

// mirror of k_pred_transform for kinds kRegression .. kDirichlet and kSoftplus: dOut (B x T x u) -> dX (B x (T*u))
__global__ void __launch_bounds__(256)
k_pred_transform_bwd(const float* __restrict__ X, int64_t ldx, const float* __restrict__ dO, int64_t lddo, int64_t B, int T,
                     int kind, int u, const float* __restrict__ scale, float* __restrict__ dX, int64_t lddx) {
  const int64_t n = B * (int64_t)T;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float* x = X + b * ldx;
    const float* g = dO + b * lddo + (int64_t)t * u;
    float* d = dX + b * lddx;
    const float s = scale ? scale[t] : 1.f, s2 = s * s;
    switch (kind) {
      case kRegression: d[t] = g[0] * s; break;
      case kSoftplus: d[t] = g[0] * softplus20_grad(x[t]); break;
      case kMve:
        d[t] = g[0] * s;
        d[T + t] = g[1] * s2 * softplus20_grad(x[T + t]);
        break;
      case kEvidential:
        d[t] = g[0] * s;
        d[T + t] = g[1] * softplus20_grad(x[T + t]);
        d[2 * T + t] = g[2] * softplus20_grad(x[2 * T + t]);
        d[3 * T + t] = g[3] * s2 * softplus20_grad(x[3 * T + t]);
        break;
      case kQuantile:                              // mean = (lo + hi) / 2, interval = hi - lo
        d[t] = (0.5f * g[0] - g[1]) * s;
        d[T + t] = (0.5f * g[0] + g[1]) * s;
        break;
      default:
        for (int c = 0; c < u; ++c) d[(int64_t)t * u + c] = g[c] * softplus20_grad(x[(int64_t)t * u + c]);
    }
  }
}

__device__ __forceinline__ float loss_weight(const float* w, const float* tw, int64_t b, int t) {
  return (w ? w[b] : 1.f) * (tw ? tw[t] : 1.f);
}

// MVELoss (metrics.py:213-219) on preds (mean, var): L = (mean - y)^2 / (2 var) + log(2 pi var) / 2
__device__ __forceinline__ float mve_term(const float* p, float y, float* g) {
  const float e = p[0] - y, v = p[1];
  if (g) {
    g[0] = e / v;
    g[1] = 0.5f / v - e * e / (2.f * v * v);
  }
  return e * e / (2.f * v) + 0.5f * logf(2.f * CUDART_PI_F * v);
}

// EvidentialLoss (metrics.py:241-257) on preds (mean, v, alpha, beta); d|r|/dr = 0 at r = 0, as torch's abs
__device__ __forceinline__ float evidential_term(const float* p, float y, float v_kl, float eps, float* g) {
  const float mu = p[0], v = p[1], a = p[2], be = p[3];
  const float r = y - mu, ar = fabsf(r);
  const float om = 2.f * be * (1.f + v);
  const float D = v * r * r + om;
  if (g) {
    const float sg = r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f);
    g[0] = -(a + 0.5f) * 2.f * v * r / D - v_kl * (2.f * v + a) * sg;
    g[1] = -0.5f / v - a * 2.f * be / om + (a + 0.5f) * (r * r + 2.f * be) / D + v_kl * 2.f * ar;
    g[2] = -logf(om) + logf(D) + digamma_ge1(a) - digamma_ge1(a + 0.5f) + v_kl * ar;
    g[3] = -a * 2.f * (1.f + v) / om + (a + 0.5f) * 2.f * (1.f + v) / D;
  }
  const float nll = 0.5f * logf(CUDART_PI_F / v) - a * logf(om) + (a + 0.5f) * logf(D) + lgammaf(a) - lgammaf(a + 0.5f);
  return nll + v_kl * ((2.f * v + a) * ar - eps);
}

// amax over two candidates with torch's backward: a tie splits the gradient evenly
__device__ __forceinline__ float amax2(float x0, float x1, float t0, float t1, float* dt) {
  if (x0 > x1) { *dt = t0; return x0; }
  if (x1 > x0) { *dt = t1; return x1; }
  *dt = 0.5f * (t0 + t1);
  return x0;
}

// QuantileLoss (metrics.py:602-610) on preds (mean, interval): bounds mean -/+ interval / 2, pinball loss at alpha / 2 and
// 1 - alpha / 2 with tau = [[alpha/2, 1 - alpha/2], [alpha/2 - 1, -alpha/2]]
__device__ __forceinline__ float quantile_term(const float* p, float y, float alpha, float* g) {
  const float m = p[0], I = p[1];
  const float e0 = y - (m + (-0.5f) * I), e1 = y - (m + 0.5f * I);
  const float ta = 0.5f * alpha;
  float d0, d1;
  const float l0 = amax2(ta * e0, (ta - 1.f) * e0, ta, ta - 1.f, &d0);
  const float l1 = amax2((1.f - ta) * e1, -ta * e1, 1.f - ta, -ta, &d1);
  if (g) {
    g[0] = -(d0 + d1);
    g[1] = 0.5f * d0 - 0.5f * d1;
  }
  return l0 + l1;
}

// label of torch.eye(C)[targets.long()]: truncation, then [-C, 0) counts from the end; -1 where torch would raise
__device__ __forceinline__ int wrapped_class_of(float y, int C) {
  const float k = truncf(y);
  if (k >= 0.f && k < (float)C) return (int)k;
  if (k < 0.f && k >= -(float)C) return (int)k + C;
  return -1;
}

// DirichletLoss (metrics.py:517-541) on alpha (C entries): L = sum (onehot - p)^2 + sum p (1 - p) / (S + 1) + v_kl KL, with
// KL = lgamma(Sa) - sum lgamma(a~) - lgamma(C) + sum (a~ - 1)(psi(a~) - psi(Sa)), a~ = onehot + (1 - onehot) alpha
__device__ __forceinline__ float dirichlet_term(const float* a, float y, int C, float v_kl, float* g) {
  const int k = wrapped_class_of(y, C);
  if (k < 0) {
    if (g) for (int c = 0; c < C; ++c) g[c] = CUDART_NAN_F;
    return CUDART_NAN_F;
  }
  float S = 0.f, Sa = 0.f;
  for (int c = 0; c < C; ++c) {
    S += a[c];
    Sa += c == k ? 1.f : a[c];
  }
  float A = 0.f, Bq = 0.f, sp = 0.f, sp2 = 0.f, lg = 0.f, kl = 0.f, sam1 = 0.f;
  const float psiS = digamma_ge1(Sa);
  for (int c = 0; c < C; ++c) {
    const float p = a[c] / S, yc = c == k ? 1.f : 0.f, at = c == k ? 1.f : a[c];
    A += (yc - p) * (yc - p);
    Bq += p * (1.f - p);
    sp += p;
    sp2 += p * p;
    lg += lgammaf(at);
    kl += (at - 1.f) * (digamma_ge1(at) - psiS);
    sam1 += at - 1.f;
  }
  if (g) {
    const float pk = a[k] / S, inv1 = 1.f / (S + 1.f), tS = trigamma_ge1(Sa);
    for (int c = 0; c < C; ++c) {
      const float p = a[c] / S, yc = c == k ? 1.f : 0.f;
      const float dA = -2.f / S * ((yc - p) - (pk - sp2));
      const float dB = ((1.f - 2.f * p) - sp + 2.f * sp2) / S * inv1 - Bq * inv1 * inv1;
      const float dK = c == k ? 0.f : (a[c] - 1.f) * trigamma_ge1(a[c]) - tS * sam1;
      g[c] = dA + dB + v_kl * dK;
    }
  }
  return A + Bq * (1.f / (S + 1.f)) + v_kl * (lgammaf(Sa) - lg - lgammaf((float)C) + kl);
}

// one block; row (b, t) = preds P[b, t*u : (t+1)*u].  loss[0] = sum w_b tw_t m_bt L / sum m, dP = dL/dP w tw m / sum m
template <int KIND>
__global__ void __launch_bounds__(1024)
k_uq_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ w,
          const float* __restrict__ tw, int64_t B, int T, int u, float p1, float p2, float* __restrict__ loss,
          float* __restrict__ dP, int64_t lddp) {
  const int64_t n = B * (int64_t)T;
  auto term = [&](const float* p, float y, float* g) {
    if constexpr (KIND == kMve) return mve_term(p, y, g);
    else if constexpr (KIND == kEvidential) return evidential_term(p, y, p1, p2, g);
    else if constexpr (KIND == kQuantile) return quantile_term(p, y, p1, g);
    else return dirichlet_term(p, y, u, p1, g);
  };
  float l = 0.f, cnt = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t b = i / T;
    const int t = (int)(i - b * T);
    const float y = Y[b * ldy + t];
    if (!isfinite(y)) continue;
    l = fmaf(loss_weight(w, tw, b, t), term(P + b * ldp + (int64_t)t * u, y, nullptr), l);
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
      float* d = dP + b * lddp + (int64_t)t * u;
      if (!isfinite(y)) {
        for (int c = 0; c < u; ++c) d[c] = 0.f;
        continue;
      }
      term(P + b * ldp + (int64_t)t * u, y, d);
      const float sc = loss_weight(w, tw, b, t) * inv_n;
      for (int c = 0; c < u; ++c) d[c] *= sc;
    }
}

// ---- NLogProbEnrichment (chemprop/nn/metrics.py:616-692) ----------------------------------------------------------------
enum EnrichMethod { kEnrichSqrt = 0, kEnrichScore = 1, kEnrichWald = 2 };

// training_step's nan_to_num(nan=0.0): NaN -> 0, +-inf -> +-FLT_MAX
__device__ __forceinline__ float nan_to_num0(float y) {
  return isnan(y) ? 0.f : fminf(fmaxf(y, -FLT_MAX), FLT_MAX);
}

// the loss term of one molecule and dL/dR (*g): z = get_zstats(R, k1, k2) with Rd = R / d, c = clamp(z / zscale, +-zi),
// L = -log(1 - erf(|c| / sqrt 2)).  1 - erf(x) is erfc(x) = erfcx(x) e^{-x^2}, so L = x^2 - log(erfcx(x)): a sum of two
// non-negative terms, exact to f32 rounding at any |c| (the reference's f32 1 - erf cancels near its default zi = 5), and
// dL/d|c| = sqrt(2 / pi) / erfcx(x).  The gradient follows torch's autograd: the clamp passes it at its bounds (inclusive)
// and not outside, d|c|/dc = 0 at c = 0.  A NaN z stays NaN through the clamp, so L and *g are NaN.
__device__ __forceinline__ float enrichment_term(float R, float k1, float k2, float d, int method, float zscale, float zi,
                                                 float* g) {
  const float Rd = R / d;
  float z, dz;                                                 // z and dz / dRd
  if (method == kEnrichScore) {
    const float D = sqrtf((k1 + k2) * Rd);
    z = (k1 - k2 * Rd) / D;
    dz = -k2 / D - z / (2.f * Rd);
  } else if (method == kEnrichWald) {
    const float D = sqrtf(k1 + k2 * (Rd * Rd));
    z = (k1 - k2 * Rd) / D;
    dz = -k2 / D - z * k2 * Rd / (D * D);
  } else {
    const float A = sqrtf(k1 + 0.375f), Bq = sqrtf((k2 + 0.375f) * Rd), S = sqrtf(1.f + Rd);
    z = 2.f * (A - Bq) / S;
    dz = -(k2 + 0.375f) / (Bq * S) - z / (2.f * (1.f + Rd));
  }
  const float c = z / zscale;
  const float cl = c < -zi ? -zi : (c > zi ? zi : c);          // NaN compares false both ways and stays NaN
  const float x = fabsf(cl) * 0.70710678118654752f;
  const float ex = erfcxf(x);
  const float dLdc = (cl > 0.f ? 1.f : (cl < 0.f ? -1.f : 0.f)) * 0.79788456080286536f / ex;
  const float pass = (c >= -zi && c <= zi) ? 1.f / zscale : 0.f;
  *g = dLdc * pass * dz / d;
  return x * x - logf(ex);
}

// one block: loss[0] = sum_b L_b w_b (tw_0 m_b0 + tw_1 m_b1) / sum m (m = isfinite(Y), the reference's b x 1 loss broadcast
// against its b x 2 mask), dR = dloss/dR.  Every molecule's term enters the sum, masked ones with weight 0, so a NaN z
// anywhere (the reference raises) makes loss[0] NaN.
__global__ void __launch_bounds__(1024)
k_enrichment_loss(const float* __restrict__ R, int64_t ldr, const float* __restrict__ Y, int64_t ldy,
                  const float* __restrict__ w, const float* __restrict__ tw, int64_t B, float d, int method, float zscale,
                  float zi, float* __restrict__ loss, float* __restrict__ dR, int64_t lddr) {
  const float tw0 = tw ? tw[0] : 1.f, tw1 = tw ? tw[1] : 1.f;
  auto row = [&](int64_t b, float* wr, float* g) {
    const float y1 = Y[b * ldy], y2 = Y[b * ldy + 1];
    const bool m1 = isfinite(y1), m2 = isfinite(y2);
    *wr = (w ? w[b] : 1.f) * ((m1 ? tw0 : 0.f) + (m2 ? tw1 : 0.f));
    return enrichment_term(R[b * ldr], nan_to_num0(y1), nan_to_num0(y2), d, method, zscale, zi, g);
  };
  float l = 0.f, cnt = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    float wr, g;
    const float L = row(b, &wr, &g);
    l = fmaf(wr, L, l);
    cnt += (float)(isfinite(Y[b * ldy]) + isfinite(Y[b * ldy + 1]));
  }
  const float2 tot = block_sum2(l, cnt);
  if (threadIdx.x == 0) loss[0] = tot.y > 0.f ? tot.x / tot.y : tot.x;      // all masked: 0, or NaN from a NaN z
  const float inv_n = tot.y > 0.f ? 1.f / tot.y : 0.f;
  if (dR != nullptr)
    for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
      float wr, g;
      row(b, &wr, &g);
      dR[b * lddr] = wr * inv_n * g;
    }
}

// ---- spectral predictor (chemprop/nn/predictors.py:339-376; nn/metrics.py:547-585) ---------------------------------------
// One CTA of kRowThreads per spectrum row (b); a row of T bins is walked in chunks of kRowThreads, so any T works.  Every
// sum and scan runs in thread order, then warp order: deterministic.
constexpr int kRowThreads = 256;
constexpr int kCountBlocks = 128;       // partial mask counts of the count prepass (workspace entries)
enum SpecAct { kSpecSoftplus = 0, kSpecExp = 1 };

// a(a(x)) (SpectralFFN's activation is applied twice) and its derivative; softplus is the predictors' softplus20
template <int ACT>
__device__ __forceinline__ float spec_act2(float x) {
  if constexpr (ACT == kSpecExp) return expf(expf(x));
  else return softplus20(softplus20(x));
}
template <int ACT>
__device__ __forceinline__ float spec_act2_grad(float x) {
  if constexpr (ACT == kSpecExp) {
    const float e = expf(x);
    return expf(e) * e;
  } else {
    return softplus20_grad(softplus20(x)) * softplus20_grad(x);
  }
}

// inclusive prefix sum over the block in thread order (lanes by shuffles, then the preceding warps' totals in order); *total
// gets the block's total.  Contains two __syncthreads.
__device__ __forceinline__ float block_scan(float v, float* total) {
  __shared__ float s_w[kRowThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_w[warp] = v;
  __syncthreads();
  float off = 0.f, tot = 0.f;
#pragma unroll
  for (int k = 0; k < kRowThreads / 32; ++k) {
    if (k == warp) off = tot;
    tot += s_w[k];
  }
  __syncthreads();
  *total = tot;
  return v + off;
}

// out row = a(a(x)) / sum_j a(a(x_j))
template <int ACT>
__global__ void __launch_bounds__(kRowThreads)
k_spectral_transform(const float* __restrict__ X, int64_t ldx, int T, float* __restrict__ out, int64_t ldo) {
  const float* x = X + blockIdx.x * ldx;
  float* o = out + blockIdx.x * ldo;
  float s = 0.f;
  for (int j = threadIdx.x; j < T; j += kRowThreads) s += spec_act2<ACT>(x[j]);
  const float S = block_sum2(s, 0.f).x;
  for (int j = threadIdx.x; j < T; j += kRowThreads) o[j] = spec_act2<ACT>(x[j]) / S;
}

// mirror: y = a(a(x)), S = sum y, dX_j = (g_j - sum_i g_i y_i / S) / S * a'(a(x_j)) a'(x_j)
template <int ACT>
__global__ void __launch_bounds__(kRowThreads)
k_spectral_transform_bwd(const float* __restrict__ X, int64_t ldx, const float* __restrict__ dO, int64_t lddo, int T,
                         float* __restrict__ dX, int64_t lddx) {
  const float* x = X + blockIdx.x * ldx;
  const float* g = dO + blockIdx.x * lddo;
  float* d = dX + blockIdx.x * lddx;
  float s = 0.f, gy = 0.f;
  for (int j = threadIdx.x; j < T; j += kRowThreads) {
    const float y = spec_act2<ACT>(x[j]);
    s += y;
    gy = fmaf(g[j], y, gy);
  }
  const float2 tot = block_sum2(s, gy);
  const float S = tot.x, dot = tot.y / tot.x;
  for (int j = threadIdx.x; j < T; j += kRowThreads) d[j] = (g[j] - dot) / S * spec_act2_grad<ACT>(x[j]);
}

// count prepass: cnt[k] = number of finite targets in rows k, k + gridDim.x, ... (exact integers)
__global__ void __launch_bounds__(kRowThreads)
k_spectral_count(const float* __restrict__ Y, int64_t ldy, int64_t B, int T, long long* __restrict__ cnt) {
  __shared__ long long s_c[kRowThreads / 32];
  long long c = 0;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x)
    for (int j = threadIdx.x; j < T; j += kRowThreads) c += isfinite(Y[b * ldy + j]) ? 1 : 0;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s_c[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int k = 0; k < kRowThreads / 32; ++k) t += s_c[k];
    cnt[blockIdx.x] = t;
  }
}

// sum m over the batch from the prepass' n_cnt partials (integers: any order is exact)
__device__ __forceinline__ long long spectral_total_count(const long long* cnt, int n_cnt) {
  __shared__ long long s_n;
  if (threadIdx.x < 32) {
    long long c = 0;
    for (int k = threadIdx.x; k < n_cnt; k += 32) c += cnt[k];
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if (threadIdx.x == 0) s_n = c;
  }
  __syncthreads();
  return s_n;
}

// pred clamped at the threshold (NaN: no clamp; NaN preds stay NaN as in torch.clamp) and whether clamp passes the
// gradient (torch: where pred >= threshold)
__device__ __forceinline__ float spec_clamp(float p, float thr, bool* pass) {
  if (isnan(thr)) { *pass = true; return p; }
  *pass = p >= thr;
  return p < thr ? thr : p;
}

// One CTA per row b.  c = clamp(p), S = sum_j m_j c_j, pn = c / S.  row_loss[b] = sum_j w tw m L_j (not yet divided by
// sum m); dP (nullable) = dLoss / dp, also used as the row's scratch between passes.  A row with no finite target writes
// row_loss 0 and dP 0.
//   SID          L_j = pn log(pn / t) + t log(t / pn) on the masked-in bins; dL/dpn = log(pn / t) + 1 - t / pn
//   Wasserstein  L_j = |cumsum(t0)_j - cumsum(pn)_j|, t0 = t with masked bins 0, pn over every bin;
//                dLoss/dpn_k = G_k = -sum_{j >= k} w tw m_j sign(D_j)  (a reverse scan; sign(0) = 0)
// then dLoss/dc_k = (G_k - m_k sum_i G_i pn_i) / S, times [p_k >= threshold].
template <bool WASS>
__global__ void __launch_bounds__(kRowThreads)
k_spectral_loss(const float* __restrict__ P, int64_t ldp, const float* __restrict__ Y, int64_t ldy,
                const float* __restrict__ w, const float* __restrict__ tw, int T, float thr,
                const long long* __restrict__ cnt, int n_cnt, float* __restrict__ row_loss, float* __restrict__ dP,
                int64_t lddp) {
  const int64_t b = blockIdx.x;
  const float* p = P + b * ldp;
  const float* y = Y + b * ldy;
  float* d = dP ? dP + b * lddp : nullptr;
  const float wb = w ? w[b] : 1.f;
  bool pass;
  float s = 0.f, n = 0.f;
  for (int j = threadIdx.x; j < T; j += kRowThreads)
    if (isfinite(y[j])) { s += spec_clamp(p[j], thr, &pass); n += 1.f; }
  const float2 sn = block_sum2(s, n);
  if (sn.y == 0.f) {                                 // every bin masked: no loss, no gradient
    if (threadIdx.x == 0) row_loss[b] = 0.f;
    if (d) for (int j = threadIdx.x; j < T; j += kRowThreads) d[j] = 0.f;
    return;
  }
  const float S = sn.x;
  float l = 0.f, gpn = 0.f;
  if constexpr (!WASS) {
    for (int j = threadIdx.x; j < T; j += kRowThreads) {
      const float t = y[j];
      float g = 0.f;
      if (isfinite(t)) {
        const float pn = spec_clamp(p[j], thr, &pass) / S;
        const float W = wb * (tw ? tw[j] : 1.f);
        const float lr = logf(pn / t);
        l = fmaf(W, pn * lr + t * logf(t / pn), l);
        g = t == 0.f ? CUDART_NAN_F : W * (lr + 1.f - t / pn);
        gpn = fmaf(g, pn, gpn);
      }
      if (d) d[j] = g;
    }
  } else {
    float ct = 0.f, cp = 0.f;                        // carries of the two cumsums
    for (int base = 0; base < T; base += kRowThreads) {
      const int j = base + threadIdx.x;
      const bool in = j < T;
      const float t = in ? y[j] : 0.f;
      const bool m = in && isfinite(t);
      const float pn = in ? spec_clamp(p[j], thr, &pass) / S : 0.f;
      float tt, tp;
      const float Ct = block_scan(m ? t : 0.f, &tt) + ct;
      const float Cp = block_scan(pn, &tp) + cp;
      ct += tt;
      cp += tp;
      const float D = Ct - Cp;
      const float W = m ? wb * (tw ? tw[j] : 1.f) : 0.f;
      l = fmaf(W, fabsf(D), l);
      if (d && in) d[j] = W * (D > 0.f ? 1.f : (D < 0.f ? -1.f : 0.f));
    }
    if (d) {
      __syncthreads();                               // the sign terms of other threads' bins
      float cg = 0.f;
      for (int base = (T - 1) / kRowThreads * kRowThreads; base >= 0; base -= kRowThreads) {
        const int j = base + (kRowThreads - 1 - threadIdx.x);       // thread order = descending bins
        const bool in = j < T;
        float tg;
        const float G = -(block_scan(in ? d[j] : 0.f, &tg) + cg);
        cg += tg;
        if (in) {
          d[j] = G;
          gpn = fmaf(G, spec_clamp(p[j], thr, &pass) / S, gpn);
        }
      }
    }
  }
  const float2 lg = block_sum2(l, gpn);              // also orders the scratch writes before the reads below
  if (threadIdx.x == 0) row_loss[b] = lg.x;
  if (!d) return;
  const long long N = spectral_total_count(cnt, n_cnt);
  const float inv_n = 1.f / (float)N;
  for (int j = threadIdx.x; j < T; j += kRowThreads) {
    const bool m = isfinite(y[j]);
    spec_clamp(p[j], thr, &pass);
    const float G = d[j];
    d[j] = (WASS || m) && pass ? (G - (m ? lg.y : 0.f)) / S * inv_n : 0.f;
  }
}

// loss[0] = sum_b row_loss[b] / sum m (0 when every target is masked), one block, fixed order
__global__ void __launch_bounds__(1024)
k_spectral_loss_finish(const float* __restrict__ row_loss, int64_t B, const long long* __restrict__ cnt, int n_cnt,
                       float* __restrict__ loss) {
  float l = 0.f;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) l += row_loss[b];
  const float tot = block_sum2(l, 0.f).x;
  const long long N = spectral_total_count(cnt, n_cnt);
  if (threadIdx.x == 0) loss[0] = N > 0 ? tot / (float)N : 0.f;
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

extern "C" int dmpnn_regression_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                     const float* task_weights, const uint8_t* lt_mask, const uint8_t* gt_mask, int64_t ldm,
                                     int64_t B, int64_t T, int kind, float* loss, float* dP, int64_t lddp, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(kind >= head::kMseLoss && kind <= head::kRmseLoss, "regression_loss: unknown kind");
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && loss && (B == 0 || (P && Y)), "regression_loss: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T) && ((!lt_mask && !gt_mask) || ldm >= T),
                  "regression_loss: row strides too small");
  head::k_regression_loss<<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, lt_mask, gt_mask, ldm, B, (int)T,
                                              kind, loss, dP, lddp);
  DMPNN_CHECK_LAUNCH("regression_loss", 1);
  return 0;
}

extern "C" int dmpnn_mse_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                              const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                              void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && loss && (B == 0 || (P && Y)), "mse_loss: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "mse_loss: row strides too small");
  head::k_regression_loss<<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, nullptr, nullptr, 0, B, (int)T,
                                              head::kMseLoss, loss, dP, lddp);
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

// outputs per task of each kind; 0 = any u >= 1 (the Dirichlet kinds: the number of classes)
static int pred_kind_u(int kind) {
  switch (kind) {
    case head::kRegression: case head::kSoftplus: return 1;
    case head::kMve: case head::kQuantile: case head::kDirichletBinary: return 2;
    case head::kEvidential: return 4;
    default: return 0;
  }
}

extern "C" int dmpnn_pred_transform(const float* X, int64_t ldx, int64_t B, int64_t T, int kind, int64_t u,
                                    const float* mean, const float* scale, float* out, int64_t ldo, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(kind >= head::kRegression && kind <= head::kSoftplus, "pred_transform: unknown kind");
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && u > 0 && T * u <= INT32_MAX && (B == 0 || (X && out)), "pred_transform: bad args");
  DMPNN_CHECK_ARG(pred_kind_u(kind) == 0 || pred_kind_u(kind) == u, "pred_transform: u does not match the kind");
  DMPNN_CHECK_ARG((mean == nullptr && scale == nullptr) || (kind <= head::kQuantile && mean && scale),
                  "pred_transform: mean and scale go together, and only with the regression kinds");
  DMPNN_CHECK_ARG(ldx >= T * u && ldo >= T * u, "pred_transform: row strides too small");
  if (B == 0) return 0;
  const unsigned blocks = (unsigned)std::min<int64_t>((B * T + 255) / 256, 1024);
  head::k_pred_transform<<<blocks, 256, 0, st>>>(X, ldx, B, (int)T, kind, (int)u, mean, scale, out, ldo);
  DMPNN_CHECK_LAUNCH("pred_transform", 1);
  return 0;
}

extern "C" int dmpnn_pred_transform_bwd(const float* X, int64_t ldx, const float* dOut, int64_t lddo, int64_t B, int64_t T,
                                        int kind, int64_t u, const float* scale, float* dX, int64_t lddx, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG((kind >= head::kRegression && kind <= head::kDirichlet) || kind == head::kSoftplus,
                  "pred_transform_bwd: unknown kind");
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && u > 0 && T * u <= INT32_MAX && (B == 0 || (X && dOut && dX)),
                  "pred_transform_bwd: bad args");
  DMPNN_CHECK_ARG(pred_kind_u(kind) == 0 || pred_kind_u(kind) == u, "pred_transform_bwd: u does not match the kind");
  DMPNN_CHECK_ARG(scale == nullptr || kind <= head::kQuantile, "pred_transform_bwd: scale only with the regression kinds");
  DMPNN_CHECK_ARG(ldx >= T * u && lddo >= T * u && lddx >= T * u, "pred_transform_bwd: row strides too small");
  if (B == 0) return 0;
  const unsigned blocks = (unsigned)std::min<int64_t>((B * T + 255) / 256, 1024);
  head::k_pred_transform_bwd<<<blocks, 256, 0, st>>>(X, ldx, dOut, lddo, B, (int)T, kind, (int)u, scale, dX, lddx);
  DMPNN_CHECK_LAUNCH("pred_transform_bwd", 1);
  return 0;
}

// shared host checks and launch of the four uncertainty losses (u outputs per task)
template <int KIND>
static int uq_loss(const char* name, const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                   const float* task_weights, int64_t B, int64_t T, int64_t u, float p1, float p2, float* loss, float* dP,
                   int64_t lddp, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && u > 0 && T * u <= INT32_MAX && loss && (B == 0 || (P && Y)), name);
  DMPNN_CHECK_ARG(ldp >= T * u && ldy >= T && (dP == nullptr || lddp >= T * u), name);
  head::k_uq_loss<KIND><<<1, 1024, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, B, (int)T, (int)u, p1, p2, loss, dP,
                                              lddp);
  DMPNN_CHECK_LAUNCH(name, 1);
  return 0;
}

extern "C" int dmpnn_mve_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                              const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                              void* stream) {
  return uq_loss<head::kMve>("mve_loss: bad args or row strides too small", P, ldp, Y, ldy, weights, task_weights, B, T, 2,
                             0.f, 0.f, loss, dP, lddp, stream);
}

extern "C" int dmpnn_evidential_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                     const float* task_weights, int64_t B, int64_t T, float v_kl, float eps, float* loss,
                                     float* dP, int64_t lddp, void* stream) {
  DMPNN_CHECK_ARG(std::isfinite(v_kl) && std::isfinite(eps), "evidential_loss: v_kl and eps must be finite");
  return uq_loss<head::kEvidential>("evidential_loss: bad args or row strides too small", P, ldp, Y, ldy, weights,
                                    task_weights, B, T, 4, v_kl, eps, loss, dP, lddp, stream);
}

extern "C" int dmpnn_quantile_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                   const float* task_weights, int64_t B, int64_t T, float alpha, float* loss, float* dP,
                                   int64_t lddp, void* stream) {
  DMPNN_CHECK_ARG(std::isfinite(alpha), "quantile_loss: alpha must be finite");
  return uq_loss<head::kQuantile>("quantile_loss: bad args or row strides too small", P, ldp, Y, ldy, weights, task_weights,
                                  B, T, 2, alpha, 0.f, loss, dP, lddp, stream);
}

extern "C" int dmpnn_dirichlet_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                    const float* task_weights, int64_t B, int64_t T, int64_t C, float v_kl, float* loss,
                                    float* dP, int64_t lddp, void* stream) {
  DMPNN_CHECK_ARG(std::isfinite(v_kl), "dirichlet_loss: v_kl must be finite");
  DMPNN_CHECK_ARG(C >= 1, "dirichlet_loss: bad args (C must be >= 1)");
  return uq_loss<head::kDirichlet>("dirichlet_loss: bad args or row strides too small", P, ldp, Y, ldy, weights,
                                   task_weights, B, T, C, v_kl, 0.f, loss, dP, lddp, stream);
}

extern "C" int dmpnn_spectral_transform(const float* X, int64_t ldx, int64_t B, int64_t T, int act, float* out, int64_t ldo,
                                        void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(act == head::kSpecSoftplus || act == head::kSpecExp, "spectral_transform: unknown activation");
  DMPNN_CHECK_ARG(B >= 0 && B <= INT32_MAX && T > 0 && T <= INT32_MAX && (B == 0 || (X && out)),
                  "spectral_transform: bad args");
  DMPNN_CHECK_ARG(ldx >= T && ldo >= T, "spectral_transform: row strides too small");
  if (B == 0) return 0;
  if (act == head::kSpecExp)
    head::k_spectral_transform<head::kSpecExp><<<(unsigned)B, head::kRowThreads, 0, st>>>(X, ldx, (int)T, out, ldo);
  else
    head::k_spectral_transform<head::kSpecSoftplus><<<(unsigned)B, head::kRowThreads, 0, st>>>(X, ldx, (int)T, out, ldo);
  DMPNN_CHECK_LAUNCH("spectral_transform", 1);
  return 0;
}

extern "C" int dmpnn_spectral_transform_bwd(const float* X, int64_t ldx, const float* dOut, int64_t lddo, int64_t B,
                                            int64_t T, int act, float* dX, int64_t lddx, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(act == head::kSpecSoftplus || act == head::kSpecExp, "spectral_transform_bwd: unknown activation");
  DMPNN_CHECK_ARG(B >= 0 && B <= INT32_MAX && T > 0 && T <= INT32_MAX && (B == 0 || (X && dOut && dX)),
                  "spectral_transform_bwd: bad args");
  DMPNN_CHECK_ARG(ldx >= T && lddo >= T && lddx >= T, "spectral_transform_bwd: row strides too small");
  if (B == 0) return 0;
  if (act == head::kSpecExp)
    head::k_spectral_transform_bwd<head::kSpecExp><<<(unsigned)B, head::kRowThreads, 0, st>>>(X, ldx, dOut, lddo, (int)T,
                                                                                             dX, lddx);
  else
    head::k_spectral_transform_bwd<head::kSpecSoftplus><<<(unsigned)B, head::kRowThreads, 0, st>>>(X, ldx, dOut, lddo,
                                                                                                  (int)T, dX, lddx);
  DMPNN_CHECK_LAUNCH("spectral_transform_bwd", 1);
  return 0;
}

// workspace of the two spectral losses: the count prepass' partials, then one loss partial per row
static int64_t spectral_count_blocks(int64_t B) { return std::min<int64_t>(B, head::kCountBlocks); }
static size_t spectral_row_offset(int64_t B) { return (size_t)spectral_count_blocks(B) * sizeof(long long); }

extern "C" int dmpnn_spectral_loss_workspace_bytes(int64_t B, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && B <= INT32_MAX && bytes, "spectral_loss_workspace_bytes: bad args");
  *bytes = spectral_row_offset(B) + (size_t)B * sizeof(float);
  return 0;
}

template <bool WASS>
static int spectral_loss(const char* name, const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                         const float* task_weights, int64_t B, int64_t T, float threshold, float* loss, float* dP,
                         int64_t lddp, void* workspace, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && B <= INT32_MAX && T > 0 && T <= INT32_MAX && loss && (B == 0 || (P && Y && workspace)),
                  "%s: bad args", name);
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (dP == nullptr || lddp >= T), "%s: row strides too small", name);
  DMPNN_CHECK_ARG(!std::isinf(threshold), "%s: threshold must be finite, or NaN for none", name);
  const int n_cnt = (int)spectral_count_blocks(B);
  long long* cnt = (long long*)workspace;
  float* row_loss = B ? (float*)((char*)workspace + spectral_row_offset(B)) : nullptr;
  if (B > 0) {
    head::k_spectral_count<<<(unsigned)n_cnt, head::kRowThreads, 0, st>>>(Y, ldy, B, (int)T, cnt);
    head::k_spectral_loss<WASS><<<(unsigned)B, head::kRowThreads, 0, st>>>(P, ldp, Y, ldy, weights, task_weights, (int)T,
                                                                          threshold, cnt, n_cnt, row_loss, dP, lddp);
  }
  head::k_spectral_loss_finish<<<1, 1024, 0, st>>>(row_loss, B, cnt, n_cnt, loss);
  DMPNN_CHECK_LAUNCH(name, B > 0 ? 3 : 1);
  return 0;
}

extern "C" int dmpnn_sid_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                              const float* task_weights, int64_t B, int64_t T, float threshold, float* loss, float* dP,
                              int64_t lddp, void* workspace, void* stream) {
  return spectral_loss<false>("sid_loss", P, ldp, Y, ldy, weights, task_weights, B, T, threshold, loss, dP, lddp, workspace,
                              stream);
}

extern "C" int dmpnn_wasserstein_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                                      const float* task_weights, int64_t B, int64_t T, float threshold, float* loss,
                                      float* dP, int64_t lddp, void* workspace, void* stream) {
  return spectral_loss<true>("wasserstein_loss", P, ldp, Y, ldy, weights, task_weights, B, T, threshold, loss, dP, lddp,
                             workspace, stream);
}

extern "C" int dmpnn_enrichment_loss(const float* R, int64_t ldr, const float* Y, int64_t ldy, const float* weights,
                                     const float* task_weights, int64_t B, float d, int method, float zscale, float zinterval,
                                     float* loss, float* dR, int64_t lddr, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(method >= head::kEnrichSqrt && method <= head::kEnrichWald, "enrichment_loss: unknown method");
  DMPNN_CHECK_ARG(std::isfinite(d) && d > 0.f && std::isfinite(zscale) && zscale != 0.f && std::isfinite(zinterval) &&
                      zinterval >= 0.f, "enrichment_loss: d must be finite and > 0, zscale finite and nonzero, zinterval "
                  "finite and >= 0");
  DMPNN_CHECK_ARG(B >= 0 && loss && (B == 0 || (R && Y)), "enrichment_loss: bad args");
  DMPNN_CHECK_ARG(ldr >= 1 && ldy >= 2 && (dR == nullptr || lddr >= 1), "enrichment_loss: row strides too small");
  head::k_enrichment_loss<<<1, 1024, 0, st>>>(R, ldr, Y, ldy, weights, task_weights, B, d, method, zscale, zinterval, loss,
                                              dR, lddr);
  DMPNN_CHECK_LAUNCH("enrichment_loss", 1);
  return 0;
}
