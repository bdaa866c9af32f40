// Per-element terms of the criteria, shared by the molecule-level kernels (head.cu) and the atom- and bond-level ones
// (row_head.cu), so that both levels compute every term alike.
#pragma once
#include <stdint.h>

namespace dmpnn {

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

// class index of a finite label as torch's `.long()` truncates it; -1 when outside [0, C)
__device__ __forceinline__ int class_of(float y, int C) {
  const float k = truncf(y);
  return (k >= 0.f && k < (float)C) ? (int)k : -1;
}

// p - y, or 0 where BoundedMixin (metrics.py:144-149) replaces the prediction by the target: p < y with lt_mask set, or
// p > y with gt_mask set (a censored target the prediction already satisfies; torch.where passes no gradient there).
// lt / gt are nullable; i indexes both.
__device__ __forceinline__ float reg_residual(float p, float y, const uint8_t* lt, const uint8_t* gt, int64_t i) {
  if ((lt && lt[i] && p < y) || (gt && gt[i] && p > y)) return 0.f;
  return p - y;
}

// PointQuantileLoss (metrics.py:282-285): alpha (y - p) where y - p > 0, (1 - alpha)(p - y) otherwise; *g = dL/dp, which at
// y == p is torch.where's second branch, 1 - alpha
__device__ __forceinline__ float pinball_term(float p, float y, float alpha, float* g) {
  const float d = y - p;
  if (d > 0.f) {
    *g = -alpha;
    return alpha * d;
  }
  *g = 1.f - alpha;
  return (1.f - alpha) * -d;
}

}  // namespace dmpnn
