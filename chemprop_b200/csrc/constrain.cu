// ConstrainerFFN's segmented part (chemprop/nn/ffn.py:119-141) in one launch each way:
//
//   dmpnn_constrain_fwd   P'[r, j] = P[r, j] + w[r, i] * (C[s, j] - sum_{r' in s} P[r', j]) for every constrained column j,
//                         w[r, i] = exp(Kl[r, i]) / sum_{r' in s} exp(Kl[r', i]); unconstrained columns copied
//   dmpnn_constrain_bwd   dP and dKl of the above (no gradient to C)
//
// One warp per molecule s, rows [ptr[s], ptr[s+1]) walked with a lane stride.  Every per-molecule sum is a lane-ordered
// partial followed by a butterfly shuffle tree: the order depends on the row count only, and every lane ends with the same
// bits (each butterfly level adds the same two values in both partner lanes).  So results are bitwise repeatable and a
// graph replay reproduces the eager call.
//
// Column j is constrained iff C[0, j] is not NaN (ffn.py:135 reads row 0 only); q is its rank among the constrained
// columns.  The w column paired with j is i = q when n_c equals the number of constrained columns nq, i = 0 when n_c == 1
// (ffn.py:138 broadcasts); any other (n_c, nq >= 1) fails the reference's broadcasting, and here writes NaN to every
// constrained column and nq to *status.
//
// Backward.  With D_j = C[s, j] - S_j, S_j = sum_s P[., j], Z_i = sum_s exp(Kl[., i]):
//   dP'[r', j] / dP[r, j]  = delta_rr' - w[r', i]              (S_j holds P[r, j] once)
//   dP'[r', j] / dKl[r, i] = D_j * w[r', i] * (delta_rr' - w[r, i])   (softmax derivative of w[., i] within s)
// so with a_j = sum_{r' in s} G[r', j] * w[r', i]:
//   dP[r, j]   = G[r, j] - a_j
//   dKl[r, i]  = sum over the constrained j paired with i of D_j * w[r, i] * (G[r, j] - a_j)
// (one j per i when n_c == nq; all constrained j when n_c == 1).  Z_i, S_j, D_j and a_j are recomputed per molecule in
// the same order as the forward's instead of being saved: they cost one extra read of Kl and P (R x (n_c + t) floats,
// a fraction of the G / dP / dKl traffic), and the backward stays one launch with no workspace.  dKl[., i] is
// accumulated over its j in place by the lane that owns the row, in increasing j: deterministic, no atomics.
#include <math_constants.h>

#include "common.cuh"

namespace dmpnn {
namespace constrain {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Shape {
  int nq;         // constrained columns
  bool ok;        // (n_c, nq) is a combination the reference accepts with nq >= 1
};

__device__ __forceinline__ Shape shape_of(const float* __restrict__ C, int64_t t, int64_t n_c) {
  int nq = 0;
  for (int64_t j = 0; j < t; ++j) nq += isnan(C[j]) ? 0 : 1;
  return {nq, nq > 0 && (n_c == nq || n_c == 1)};
}

// per-molecule sums of column i of exp(Kl) and column j of P
__device__ __forceinline__ void seg_sums(const float* __restrict__ Kl, int64_t ldk, int64_t i, const float* __restrict__ P,
                                         int64_t ldp, int64_t j, int64_t lo, int64_t hi, int lane, float& Z, float& S) {
  float z = 0.f, p = 0.f;
  for (int64_t r = lo + lane; r < hi; r += 32) {
    z += expf(Kl[r * ldk + i]);
    p += P[r * ldp + j];
  }
  Z = warp_sum(z);
  S = warp_sum(p);
}

__global__ void __launch_bounds__(kThreads)
k_constrain_fwd(const float* __restrict__ Kl, int64_t ldk, int64_t n_c, const float* __restrict__ P, int64_t ldp,
                const int32_t* __restrict__ ptr, int64_t m, const float* __restrict__ C, int64_t ldc, int64_t t,
                float* __restrict__ out, int64_t ldo, int32_t* __restrict__ status) {
  const Shape sh = shape_of(C, t, n_c);
  if (blockIdx.x == 0 && threadIdx.x == 0) *status = (sh.nq > 0 && !sh.ok) ? sh.nq : 0;
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (s >= m) return;
  const int64_t lo = ptr[s], hi = ptr[s + 1];
  if (lo >= hi) return;
  int q = 0;
  for (int64_t j = 0; j < t; ++j) {
    const bool con = !isnan(C[j]);
    if (!con || !sh.ok) {
      for (int64_t r = lo + lane; r < hi; r += 32) out[r * ldo + j] = con ? CUDART_NAN_F : P[r * ldp + j];
      q += con;
      continue;
    }
    const int64_t i = n_c == 1 ? 0 : q++;
    float Z, S;
    seg_sums(Kl, ldk, i, P, ldp, j, lo, hi, lane, Z, S);
    const float D = C[s * ldc + j] - S;
    for (int64_t r = lo + lane; r < hi; r += 32) out[r * ldo + j] = P[r * ldp + j] + expf(Kl[r * ldk + i]) / Z * D;
  }
}

// minBlocks 1 lets ptxas go past 64 registers: without it the kernel spills
__global__ void __launch_bounds__(kThreads, 1)
k_constrain_bwd(const float* __restrict__ G, int64_t ldg, const float* __restrict__ Kl, int64_t ldk, int64_t n_c,
                const float* __restrict__ P, int64_t ldp, const int32_t* __restrict__ ptr, int64_t m,
                const float* __restrict__ C, int64_t ldc, int64_t t, float* __restrict__ dP, int64_t lddp,
                float* __restrict__ dKl, int64_t lddk) {
  const Shape sh = shape_of(C, t, n_c);
  const int lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  if (s >= m) return;
  const int64_t lo = ptr[s], hi = ptr[s + 1];
  if (lo >= hi) return;
  if (!sh.ok) {        // no constrained column (P' = P), or a rejected shape (P' NaN in the constrained columns)
    for (int64_t r = lo + lane; r < hi; r += 32) {
      for (int64_t j = 0; j < t; ++j) dP[r * lddp + j] = (sh.nq == 0 || isnan(C[j])) ? G[r * ldg + j] : CUDART_NAN_F;
      for (int64_t i = 0; i < n_c; ++i) dKl[r * lddk + i] = sh.nq == 0 ? 0.f : CUDART_NAN_F;
    }
    return;
  }
  int q = 0;
  for (int64_t j = 0; j < t; ++j) {
    if (isnan(C[j])) {
      for (int64_t r = lo + lane; r < hi; r += 32) dP[r * lddp + j] = G[r * ldg + j];
      continue;
    }
    const bool first = n_c != 1 || q == 0;          // first constrained column paired with w column i
    const int64_t i = n_c == 1 ? 0 : q;
    ++q;
    float Z, S;
    seg_sums(Kl, ldk, i, P, ldp, j, lo, hi, lane, Z, S);
    const float D = C[s * ldc + j] - S;
    const float* __restrict__ Gj = G + j;
    const float* __restrict__ Ki = Kl + i;
    float a = 0.f;
    for (int64_t r = lo + lane; r < hi; r += 32) a += Gj[r * ldg] * (expf(Ki[r * ldk]) / Z);
    a = warp_sum(a);
    for (int64_t r = lo + lane; r < hi; r += 32) {
      const float g = Gj[r * ldg] - a;
      const float c = D * (expf(Ki[r * ldk]) / Z) * g;
      dP[r * lddp + j] = g;
      float* d = dKl + r * lddk + i;
      *d = first ? c : *d + c;
    }
  }
}

static unsigned blocks(int64_t m) { return (unsigned)((m + kWarps - 1) / kWarps); }

}  // namespace constrain
}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_constrain_fwd(const float* Kl, int64_t ldk, int64_t n_c, const float* P, int64_t ldp,
                                   const int32_t* ptr, int64_t m, const float* C, int64_t ldc, int64_t t, float* out,
                                   int64_t ldo, int32_t* status, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(n_c > 0 && t > 0 && m >= 0 && m < INT32_MAX && ptr && status && (m == 0 || (Kl && P && C && out)),
                  "constrain_fwd: bad args");
  DMPNN_CHECK_ARG(ldk >= n_c && ldp >= t && ldc >= t && ldo >= t, "constrain_fwd: row strides too small");
  if (m == 0) return 0;
  constrain::k_constrain_fwd<<<constrain::blocks(m), constrain::kThreads, 0, st>>>(Kl, ldk, n_c, P, ldp, ptr, m, C, ldc,
                                                                                   t, out, ldo, status);
  DMPNN_CHECK_LAUNCH("constrain_fwd", 1);
  return 0;
}

extern "C" int dmpnn_constrain_bwd(const float* G, int64_t ldg, const float* Kl, int64_t ldk, int64_t n_c, const float* P,
                                   int64_t ldp, const int32_t* ptr, int64_t m, const float* C, int64_t ldc, int64_t t,
                                   float* dP, int64_t lddp, float* dKl, int64_t lddk, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(n_c > 0 && t > 0 && m >= 0 && m < INT32_MAX && ptr && (m == 0 || (G && Kl && P && C && dP && dKl)),
                  "constrain_bwd: bad args");
  DMPNN_CHECK_ARG(ldg >= t && ldk >= n_c && ldp >= t && ldc >= t && lddp >= t && lddk >= n_c,
                  "constrain_bwd: row strides too small");
  if (m == 0) return 0;
  constrain::k_constrain_bwd<<<constrain::blocks(m), constrain::kThreads, 0, st>>>(G, ldg, Kl, ldk, n_c, P, ldp, ptr, m, C,
                                                                                   ldc, t, dP, lddp, dKl, lddk);
  DMPNN_CHECK_LAUNCH("constrain_bwd", 1);
  return 0;
}
