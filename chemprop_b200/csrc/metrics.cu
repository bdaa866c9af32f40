// Validation and test metrics accumulated on the device (chemprop/nn/metrics.py:59-499, the torchmetrics classes it wraps):
//
//   dmpnn_metric_accumulate       the element-wise family: MSE / MAE (bounded or not), R2's pooled sums, the pooled
//                                 confusion counts of accuracy and F1, and binary MCC's per-task soft counts
//   dmpnn_metric_multiclass_mcc   the per-task p, t, c, s sums of the multiclass soft MCC
//   dmpnn_metric_rank_format      one update of AUROC / AUPRC: formatted score, label and keep flag per element
//   dmpnn_rank_curve              AUROC and AUPRC of every formatted element: one device radix sort, one scan
//
// Every sum is two-phase, as in row_head.cu: CTA k of the first launch reduces a fixed contiguous chunk of rows into its
// partials in the workspace, and one CTA of the second launch sums the partials in a fixed order and ADDS the totals to the
// caller's state (f64 sums, int64 counts).  The grid depends on the shape only, so results are bitwise repeatable; no
// floating-point atomics; no host synchronisation.  The classification kinds first run a range pass (one flag per CTA):
// where any considered prediction of the call lies outside [0, 1] -- or is NaN -- the whole call reads sigmoid(P) (softmax
// over the classes for the multiclass MCC), which is torchmetrics' per-update input formatting.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <math_constants.h>

#include <algorithm>

#include "common.cuh"
#include "loss_terms.cuh"

namespace dmpnn {
namespace metric {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 1024;
constexpr int64_t kMinChunk = 2048;      // elements per CTA at least

enum Kind { kSqErr = 0, kAbsErr = 1, kR2 = 2, kConfusion = 3, kSoftMcc = 4 };

struct Args {
  const float* P;
  int64_t ldp;
  const float* Y;
  int64_t ldy;
  const uint8_t* M;     // nullable: then m = isfinite(Y)
  const float* w;
  const float* tw;
  const uint8_t* lt;
  const uint8_t* gt;
  int64_t ldm;          // row stride of M, lt, gt
  int64_t B;
  int T;
  int C;
};

// fixed-order block sum: lanes by a shuffle tree, then the warp partials in order; every thread gets the total
template <typename V>
__device__ __forceinline__ V block_sum(V v) {
  __shared__ V s_w[kThreads / 32];
  __shared__ V s_t;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    V a = 0;
    for (int k = 0; k < kThreads / 32; ++k) a += s_w[k];
    s_t = a;
  }
  __syncthreads();
  const V r = s_t;
  __syncthreads();      // s_w / s_t are reused by the next call
  return r;
}

__device__ __forceinline__ bool masked_in(const Args& a, int64_t b, int t) {
  return a.M ? a.M[b * a.ldm + t] != 0 : isfinite(a.Y[b * a.ldy + t]);
}

// torch's sigmoid in f32: 1 / (1 + exp(-x))
__device__ __forceinline__ float sigmoid_torch(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ bool in_unit(float p) { return p >= 0.f && p <= 1.f; }   // false for NaN

// binary label of a masked-in target as `.long()` gives it; -1 (an error) outside {0, 1}
__device__ __forceinline__ int binary_label(float y) { return class_of(y, 2); }

static int blocks_for(int64_t n) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(kMaxBlocks, (n + kMinChunk - 1) / kMinChunk));
}

// rows of CTA k: [k * rchunk, min(B, (k + 1) * rchunk))
struct Grid {
  int G;
  int64_t rchunk;
};

static Grid grid_of(int64_t B, int64_t cols) {
  const int G0 = blocks_for(B * std::max<int64_t>(cols, 1));
  const int G = (int)std::max<int64_t>(1, std::min<int64_t>(G0, B));
  return {G, std::max<int64_t>(1, (B + G - 1) / G)};
}

// ---- range pass: flag[k] = 1 when CTA k's rows hold a considered prediction outside [0, 1] ------------------------------
// masked != 0: only masked-in elements (b, t) of the b x T predictions count (ClassificationMixin passes preds[mask]);
// masked == 0: every one of the b x ncols predictions (binary / multiclass MCC test the whole tensor)
__global__ void __launch_bounds__(kThreads)
k_range_flags(Args a, int64_t ncols, int masked, int64_t rchunk, int* __restrict__ flags) {
  const int64_t lo = (int64_t)blockIdx.x * rchunk, hi = min(a.B, lo + rchunk);
  int bad = 0;
  for (int64_t e = lo * ncols + threadIdx.x; e < hi * ncols; e += kThreads) {
    const int64_t b = e / ncols;
    const int64_t c = e - b * ncols;
    if (masked && !masked_in(a, b, (int)c)) continue;
    bad |= !in_unit(a.P[b * a.ldp + c]);
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) flags[blockIdx.x] = bad;
}

__device__ __forceinline__ bool any_flag(const int* flags, int G) {
  int f = 0;
  for (int k = threadIdx.x; k < G; k += kThreads) f |= flags[k];
  return __syncthreads_or(f) != 0;
}

// ---- element-wise family ------------------------------------------------------------------------------------------------
template <int K> struct Counts;
template <> struct Counts<kSqErr> { static constexpr int F = 1, I = 1; static constexpr bool per_task = false; };
template <> struct Counts<kAbsErr> { static constexpr int F = 1, I = 1; static constexpr bool per_task = false; };
template <> struct Counts<kR2> { static constexpr int F = 3, I = 1; static constexpr bool per_task = false; };
template <> struct Counts<kConfusion> { static constexpr int F = 0, I = 4; static constexpr bool per_task = false; };
template <> struct Counts<kSoftMcc> { static constexpr int F = 4, I = 0; static constexpr bool per_task = true; };

// adds element (b, t), masked in, to f / n
template <int K>
__device__ __forceinline__ void add_term(const Args& a, int64_t b, int t, bool sig, double* f, long long* n,
                                         int32_t* status) {
  const float y = a.Y[b * a.ldy + t];
  float p = a.P[b * a.ldp + t];
  if (K == kSqErr || K == kAbsErr) {
    // BoundedMixin's replacement of the prediction by the target (reg_residual), the residual itself in f64
    const double e = reg_residual(p, y, a.lt, a.gt, b * a.ldm + t) == 0.f ? 0.0 : (double)p - (double)y;
    const double ww = (double)(a.w ? a.w[b] : 1.f) * (double)(a.tw ? a.tw[t] : 1.f);
    f[0] += (K == kSqErr ? e * e : fabs(e)) * ww;
    n[0] += 1;
  } else if (K == kR2) {
    const double yd = y, r = (double)y - (double)p;
    f[0] += yd;
    f[1] += yd * yd;
    f[2] += r * r;
    n[0] += 1;
  } else {
    const int l = binary_label(y);
    if (l < 0) { status[0] = 1; return; }
    if (sig) p = sigmoid_torch(p);
    if (K == kConfusion) {
      const bool hit = p > 0.5f;
      n[0] += hit && l == 1;     // TP
      n[1] += hit && l == 0;     // FP
      n[2] += !hit && l == 0;    // TN
      n[3] += !hit && l == 1;    // FN
    } else {                     // soft counts weighted by w * m (metrics.py:347-353)
      const double wm = a.w ? (double)a.w[b] : 1.0, pd = p, yl = l;
      f[0] += yl * pd * wm;
      f[1] += (1.0 - yl) * pd * wm;
      f[2] += (1.0 - yl) * (1.0 - pd) * wm;
      f[3] += yl * (1.0 - pd) * wm;
    }
  }
}

// phase 1: CTA k reduces its rows into slot partials partF[(k * NS + s) * F + j], partI[(k * NS + s) * I + j] (NS = T for
// the per-task kinds, 1 for the pooled ones)
template <int K>
__global__ void __launch_bounds__(kThreads)
k_metric_partials(Args a, int64_t rchunk, const int* __restrict__ flags, int G, double* __restrict__ partF,
                  long long* __restrict__ partI, int32_t* status) {
  using Cn = Counts<K>;
  constexpr int F = Cn::F > 0 ? Cn::F : 1, I = Cn::I > 0 ? Cn::I : 1;
  const bool sig = (K == kConfusion || K == kSoftMcc) ? any_flag(flags, G) : false;
  const int64_t lo = (int64_t)blockIdx.x * rchunk, hi = min(a.B, lo + rchunk);
  const int NS = Cn::per_task ? a.T : 1;
  for (int s = 0; s < NS; ++s) {
    double f[F] = {};
    long long n[I] = {};
    if (Cn::per_task) {
      for (int64_t b = lo + threadIdx.x; b < hi; b += kThreads)
        if (masked_in(a, b, s)) add_term<K>(a, b, s, sig, f, n, status);
    } else {
      for (int64_t e = lo * a.T + threadIdx.x; e < hi * a.T; e += kThreads) {
        const int64_t b = e / a.T;
        const int t = (int)(e - b * a.T);
        if (masked_in(a, b, t)) add_term<K>(a, b, t, sig, f, n, status);
      }
    }
#pragma unroll
    for (int j = 0; j < Cn::F; ++j) {
      const double v = block_sum(f[j]);
      if (threadIdx.x == 0) partF[((int64_t)blockIdx.x * NS + s) * Cn::F + j] = v;
    }
#pragma unroll
    for (int j = 0; j < Cn::I; ++j) {
      const long long v = block_sum(n[j]);
      if (threadIdx.x == 0) partI[((int64_t)blockIdx.x * NS + s) * Cn::I + j] = v;
    }
  }
}

// phase 2 (one CTA): state value (s, j) += the G partials of slot s, summed in one fixed order; states are laid out
// value-major, fstate[j * NS + s]
__global__ void __launch_bounds__(kThreads)
k_metric_finish(int G, int NS, int F, int I, const double* __restrict__ partF, const long long* __restrict__ partI,
                double* __restrict__ fstate, int64_t* __restrict__ istate) {
  for (int s = 0; s < NS; ++s) {
    for (int j = 0; j < F; ++j) {
      double v = 0.0;
      for (int k = threadIdx.x; k < G; k += kThreads) v += partF[((int64_t)k * NS + s) * F + j];
      v = block_sum(v);
      if (threadIdx.x == 0) fstate[(int64_t)j * NS + s] += v;
    }
    for (int j = 0; j < I; ++j) {
      long long v = 0;
      for (int k = threadIdx.x; k < G; k += kThreads) v += partI[((int64_t)k * NS + s) * I + j];
      v = block_sum(v);
      if (threadIdx.x == 0) istate[(int64_t)j * NS + s] += v;
    }
  }
}

// ---- multiclass MCC -------------------------------------------------------------------------------------------------------
// formatted class probability q_c of row b, task t (softmax over the C classes where `soft`)
struct ClassRow {
  const float* p;
  int C;
  bool soft;
  float mx, inv;
  __device__ ClassRow(const float* p_, int C_, bool soft_) : p(p_), C(C_), soft(soft_), mx(0.f), inv(1.f) {
    if (soft) {
      mx = p[0];
      for (int c = 1; c < C; ++c) mx = fmaxf(mx, p[c]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(p[c] - mx);
      inv = 1.f / s;
    }
  }
  __device__ float q(int c) const { return soft ? expf(p[c] - mx) * inv : p[c]; }
  __device__ int argmax() const {      // first maximum, as torch.argmax
    int k = 0;
    float best = q(0);
    for (int c = 1; c < C; ++c) {
      const float v = q(c);
      if (v > best) { best = v; k = c; }
    }
    return k;
  }
};

// torch.eye(C)[targets.long()]: trunc(y) in [0, C), or in [-C, 0) counting from the end; -1 outside
__device__ __forceinline__ int mc_label(float y, int C) {
  const float k = truncf(y);
  if (!(k >= -(float)C && k < (float)C)) return -1;
  return k < 0.f ? (int)k + C : (int)k;
}

// CTA k, task t: values j in [0, C) p_j, [C, 2C) t_j, 2C c, 2C + 1 s (metrics.py:423-434), weight w * m
__global__ void __launch_bounds__(kThreads)
k_mcc_partials(Args a, int64_t rchunk, const int* __restrict__ flags, int G, double* __restrict__ partF,
               int32_t* status) {
  const bool soft = any_flag(flags, G);
  const int64_t lo = (int64_t)blockIdx.x * rchunk, hi = min(a.B, lo + rchunk);
  const int C = a.C, NV = 2 * C + 2;
  for (int t = 0; t < a.T; ++t) {
    double* out = partF + ((int64_t)blockIdx.x * a.T + t) * NV;
    // class by class, so that no thread keeps a per-class array: C passes over the chunk (L1 / L2 resident)
    for (int c = 0; c < C; ++c) {
      double pc = 0.0, tc = 0.0;
      for (int64_t b = lo + threadIdx.x; b < hi; b += kThreads) {
        if (!masked_in(a, b, t)) continue;
        const int l = mc_label(a.Y[b * a.ldy + t], C);
        if (l < 0) { status[0] = 1; continue; }
        const double wm = a.w ? (double)a.w[b] : 1.0;
        const ClassRow r(a.P + b * a.ldp + (int64_t)t * C, C, soft);
        pc += r.argmax() == c ? wm : 0.0;
        tc += l == c ? wm : 0.0;
      }
      pc = block_sum(pc);
      tc = block_sum(tc);
      if (threadIdx.x == 0) { out[c] = pc; out[C + c] = tc; }
    }
    double cc = 0.0, ss = 0.0;
    for (int64_t b = lo + threadIdx.x; b < hi; b += kThreads) {
      if (!masked_in(a, b, t)) continue;
      const int l = mc_label(a.Y[b * a.ldy + t], C);
      if (l < 0) continue;
      const double wm = a.w ? (double)a.w[b] : 1.0;
      const ClassRow r(a.P + b * a.ldp + (int64_t)t * C, C, soft);
      cc += r.argmax() == l ? wm : 0.0;
      double s = 0.0;
      for (int c = 0; c < C; ++c) s += (double)r.q(c);
      ss += s * wm;
    }
    cc = block_sum(cc);
    ss = block_sum(ss);
    if (threadIdx.x == 0) { out[2 * C] = cc; out[2 * C + 1] = ss; }
  }
}

// ---- ranking: format -----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_rank_format(Args a, const int* __restrict__ flags, int G, float* __restrict__ score, uint8_t* __restrict__ label,
              uint8_t* __restrict__ keep, int32_t* status) {
  const bool sig = any_flag(flags, G);
  const int64_t n = a.B * (int64_t)a.T;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < n; e += (int64_t)gridDim.x * kThreads) {
    const int64_t b = e / a.T;
    const int t = (int)(e - b * a.T);
    const bool m = masked_in(a, b, t);
    int l = 0;
    if (m) {
      l = binary_label(a.Y[b * a.ldy + t]);
      if (l < 0) { status[0] = 1; l = 0; }
    }
    const float p = a.P[b * a.ldp + t];
    score[e] = m ? (sig ? sigmoid_torch(p) : p) : 0.f;
    label[e] = (uint8_t)l;
    keep[e] = m;
  }
}

// ---- ranking: curve ------------------------------------------------------------------------------------------------------
// sort key of a kept score: the float's bits mapped to an order-preserving unsigned integer; masked entries get 0, below
// every finite score, so that a descending sort puts them after all kept ones
__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct ScanItem {
  int32_t tps;      // positives at positions <= i
  int32_t start;    // first position of i's run of equal keys
};

struct ScanOp {
  __device__ __forceinline__ ScanItem operator()(const ScanItem& x, const ScanItem& y) const {
    return {x.tps + y.tps, max(x.start, y.start)};
  }
};

__global__ void __launch_bounds__(kThreads)
k_curve_keys(const float* __restrict__ score, const uint8_t* __restrict__ label, const uint8_t* __restrict__ keep, int64_t n,
             uint32_t* __restrict__ key, uint8_t* __restrict__ val) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const bool k = keep[i] != 0;
    key[i] = k ? order_key(score[i]) : 0u;
    val[i] = k ? (label[i] != 0) : 0;
  }
}

__global__ void __launch_bounds__(kThreads)
k_curve_items(const uint32_t* __restrict__ key, const uint8_t* __restrict__ val, int64_t n, ScanItem* __restrict__ item) {
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    item[i] = {(int32_t)val[i], (i == 0 || key[i - 1] != key[i]) ? (int32_t)i : 0};
}

// the curve's points are the ends of the runs of equal kept keys (distinct thresholds), in descending score order; the
// point before run [s, e] is position s - 1's, or the origin.  Each CTA sums the terms of the run ends in its chunk:
// AUROC's (fps_e - fps_prev) * (tps_e + tps_prev) exactly in int64, AUPRC's trapezoid in f64
__global__ void __launch_bounds__(kThreads)
k_curve_partials(const uint32_t* __restrict__ key, const ScanItem* __restrict__ item, int64_t n, int64_t chunk,
                 long long* __restrict__ part_roc, double* __restrict__ part_prc, long long* __restrict__ part_kept) {
  const int64_t lo = (int64_t)blockIdx.x * chunk, hi = min(n, lo + chunk);
  const double P = (double)item[n - 1].tps;
  long long roc = 0, kept = 0;
  double prc = 0.0;
  for (int64_t e = lo + threadIdx.x; e < hi; e += kThreads) {
    if (key[e] == 0u) continue;
    ++kept;
    if (e + 1 < n && key[e + 1] == key[e]) continue;
    const ScanItem it = item[e];
    const long long tp = it.tps, fp = e + 1 - (long long)it.tps;
    const int64_t s = it.start;
    const long long tp0 = s > 0 ? item[s - 1].tps : 0, fp0 = s > 0 ? s - tp0 : 0;
    roc += (fp - fp0) * (tp + tp0);
    const double r = tp / P, r0 = tp0 / P;
    const double pr = (double)tp / (double)(tp + fp), pr0 = s > 0 ? (double)tp0 / (double)(tp0 + fp0) : 1.0;
    prc += (r - r0) * (pr + pr0) * 0.5;
  }
  roc = block_sum(roc);
  prc = block_sum(prc);
  kept = block_sum(kept);
  if (threadIdx.x == 0) {
    part_roc[blockIdx.x] = roc;
    part_prc[blockIdx.x] = prc;
    part_kept[blockIdx.x] = kept;
  }
}

__global__ void __launch_bounds__(kThreads)
k_curve_finish(const ScanItem* __restrict__ item, int64_t n, int G, const long long* __restrict__ part_roc,
               const double* __restrict__ part_prc, const long long* __restrict__ part_kept, double* __restrict__ out) {
  long long roc = 0, kept = 0;
  double prc = 0.0;
  for (int k = threadIdx.x; k < G; k += kThreads) {
    roc += part_roc[k];
    prc += part_prc[k];
    kept += part_kept[k];
  }
  roc = block_sum(roc);
  prc = block_sum(prc);
  kept = block_sum(kept);
  if (threadIdx.x == 0) {
    const long long P = n > 0 ? item[n - 1].tps : 0, N = kept - P;
    // torchmetrics zeroes fpr (no negatives) or tpr (no positives): the area is 0
    out[0] = (P > 0 && N > 0) ? (double)roc / (2.0 * (double)P * (double)N) : 0.0;
    out[1] = P > 0 ? prc : CUDART_NAN;     // P == 0: recall 0 / 0, NaN as the reference's auc(recall, precision)
  }
}

// ---- sizes ---------------------------------------------------------------------------------------------------------------
static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct CurveLayout {
  size_t key_in, key_out, val_in, val_out, items, part_roc, part_prc, part_kept, temp, temp_bytes, total;
  int G;
  int64_t chunk;
};

static int curve_layout(int64_t n, CurveLayout* L) {
  size_t sort_bytes = 0, scan_bytes = 0;
  cudaError_t e = cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                                            (const uint8_t*)nullptr, (uint8_t*)nullptr, (int)n);
  if (e == cudaSuccess)
    e = cub::DeviceScan::InclusiveScan(nullptr, scan_bytes, (const ScanItem*)nullptr, (ScanItem*)nullptr, ScanOp(), (int)n);
  if (e != cudaSuccess) {
    set_error("rank_curve: cub size query failed: %s", cudaGetErrorString(e));
    return -2;
  }
  L->G = blocks_for(n);
  L->chunk = std::max<int64_t>(1, (n + L->G - 1) / L->G);
  size_t o = 0;
  L->key_in = o;   o += align256(n * sizeof(uint32_t));
  L->key_out = o;  o += align256(n * sizeof(uint32_t));
  L->val_in = o;   o += align256(n);
  L->val_out = o;  o += align256(n);
  L->items = o;    o += align256(n * sizeof(ScanItem));
  L->part_roc = o; o += align256(L->G * sizeof(long long));
  L->part_prc = o; o += align256(L->G * sizeof(double));
  L->part_kept = o; o += align256(L->G * sizeof(long long));
  L->temp = o;
  L->temp_bytes = std::max(sort_bytes, scan_bytes);
  o += align256(std::max<size_t>(L->temp_bytes, 1));
  L->total = o;
  return 0;
}

}  // namespace metric
}  // namespace dmpnn

using namespace dmpnn;

// workspace of the accumulating entry points: flags and partials for every kind at B x T (x C)
extern "C" int dmpnn_metric_workspace_bytes(int64_t B, int64_t T, int64_t C, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && C >= 1 && T * C <= INT32_MAX && bytes,
                  "metric_workspace_bytes: bad args");
  const metric::Grid g = metric::grid_of(B, T * C);
  const int64_t nv = std::max<int64_t>(4 * T, T * (2 * C + 2));       // per-CTA values of the widest kind
  *bytes = metric::align256((size_t)g.G * sizeof(int)) + (size_t)g.G * nv * sizeof(double);
  return 0;
}

extern "C" int dmpnn_metric_accumulate(int kind, const float* P, int64_t ldp, const float* Y, int64_t ldy,
                                       const uint8_t* mask, const float* weights, const float* task_weights,
                                       const uint8_t* lt_mask, const uint8_t* gt_mask, int64_t ldm, int64_t B, int64_t T,
                                       double* fstate, int64_t* istate, int32_t* status, void* workspace, void* stream_) {
  using namespace metric;
  DMPNN_CHECK_ARG(kind >= kSqErr && kind <= kSoftMcc, "metric_accumulate: unknown kind %d", kind);
  const bool needs_f = kind != kConfusion, needs_i = kind != kSoftMcc, classify = kind >= kConfusion;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && (B == 0 || (P && Y && workspace)) && (!needs_f || fstate) &&
                      (!needs_i || istate) && (!classify || status),
                  "metric_accumulate: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && ((!mask && !lt_mask && !gt_mask) || ldm >= T),
                  "metric_accumulate: row strides too small");
  DMPNN_CHECK_ARG(!(lt_mask || gt_mask) || kind <= kAbsErr, "metric_accumulate: bound masks only for MSE / MAE");
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream_;
  const Args a{P, ldp, Y, ldy, mask, weights, task_weights, lt_mask, gt_mask, ldm, B, (int)T, 1};
  const Grid g = grid_of(B, T);
  int* flags = (int*)workspace;
  double* partF = (double*)((char*)workspace + align256((size_t)g.G * sizeof(int)));
  long long* partI = (long long*)partF;          // the integer kinds use the same bytes
  int n_launch = 2;
  if (classify) {
    k_range_flags<<<(unsigned)g.G, kThreads, 0, st>>>(a, T, kind == kConfusion, g.rchunk, flags);
    ++n_launch;
  }
  int F = 0, I = 0, NS = 1;
  switch (kind) {
    case kSqErr:
      k_metric_partials<kSqErr><<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, partI + g.G, status);
      F = 1, I = 1;
      break;
    case kAbsErr:
      k_metric_partials<kAbsErr><<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, partI + g.G, status);
      F = 1, I = 1;
      break;
    case kR2:
      k_metric_partials<kR2><<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, partI + 3 * g.G, status);
      F = 3, I = 1;
      break;
    case kConfusion:
      k_metric_partials<kConfusion><<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, partI, status);
      F = 0, I = 4;
      break;
    default:
      k_metric_partials<kSoftMcc><<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, partI, status);
      F = 4, I = 0, NS = (int)T;
      break;
  }
  const long long* pI = kind == kConfusion ? partI : partI + (int64_t)g.G * F;
  k_metric_finish<<<1, kThreads, 0, st>>>(g.G, NS, F, I, partF, pI, fstate, istate);
  DMPNN_CHECK_LAUNCH("metric_accumulate", n_launch);
  return 0;
}

extern "C" int dmpnn_metric_multiclass_mcc(const float* P, int64_t ldp, const float* Y, int64_t ldy, const uint8_t* mask,
                                           int64_t ldm, const float* weights, int64_t B, int64_t T, int64_t C,
                                           double* fstate, int32_t* status, void* workspace, void* stream_) {
  using namespace metric;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && C >= 2 && T * C <= INT32_MAX && fstate && status && (B == 0 || (P && Y && workspace)),
                  "metric_multiclass_mcc: bad args (C >= 2)");
  DMPNN_CHECK_ARG(ldp >= T * C && ldy >= T && (!mask || ldm >= T), "metric_multiclass_mcc: row strides too small");
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream_;
  const Args a{P, ldp, Y, ldy, mask, weights, nullptr, nullptr, nullptr, ldm, B, (int)T, (int)C};
  const Grid g = grid_of(B, T * C);
  int* flags = (int*)workspace;
  double* partF = (double*)((char*)workspace + align256((size_t)g.G * sizeof(int)));
  k_range_flags<<<(unsigned)g.G, kThreads, 0, st>>>(a, T * C, 0, g.rchunk, flags);
  k_mcc_partials<<<(unsigned)g.G, kThreads, 0, st>>>(a, g.rchunk, flags, g.G, partF, status);
  k_metric_finish<<<1, kThreads, 0, st>>>(g.G, 1, (int)(T * (2 * C + 2)), 0, partF, nullptr, fstate, nullptr);
  DMPNN_CHECK_LAUNCH("metric_multiclass_mcc", 3);
  return 0;
}

extern "C" int dmpnn_metric_rank_format(const float* P, int64_t ldp, const float* Y, int64_t ldy, const uint8_t* mask,
                                        int64_t ldm, int64_t B, int64_t T, float* score, uint8_t* label, uint8_t* keep,
                                        int32_t* status, void* workspace, void* stream_) {
  using namespace metric;
  DMPNN_CHECK_ARG(B >= 0 && T > 0 && T <= INT32_MAX && status &&
                      (B == 0 || (P && Y && score && label && keep && workspace)),
                  "metric_rank_format: bad args");
  DMPNN_CHECK_ARG(ldp >= T && ldy >= T && (!mask || ldm >= T), "metric_rank_format: row strides too small");
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream_;
  const Args a{P, ldp, Y, ldy, mask, nullptr, nullptr, nullptr, nullptr, ldm, B, (int)T, 1};
  const Grid g = grid_of(B, T);
  int* flags = (int*)workspace;
  k_range_flags<<<(unsigned)g.G, kThreads, 0, st>>>(a, T, 1, g.rchunk, flags);
  const unsigned blocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>((B * T + kThreads - 1) / kThreads, 132 * 16));
  k_rank_format<<<blocks, kThreads, 0, st>>>(a, flags, g.G, score, label, keep, status);
  DMPNN_CHECK_LAUNCH("metric_rank_format", 2);
  return 0;
}

extern "C" int dmpnn_rank_curve_workspace_bytes(int64_t n, size_t* bytes) {
  DMPNN_CHECK_ARG(n >= 0 && n <= INT32_MAX && bytes, "rank_curve_workspace_bytes: bad args (n <= 2^31 - 1)");
  if (n == 0) {
    *bytes = 0;
    return 0;
  }
  metric::CurveLayout L;
  if (int rc = metric::curve_layout(n, &L)) return rc;
  *bytes = L.total;
  return 0;
}

extern "C" int dmpnn_rank_curve(const float* score, const uint8_t* label, const uint8_t* keep, int64_t n, double* out,
                                void* workspace, size_t workspace_bytes, void* stream_) {
  using namespace metric;
  DMPNN_CHECK_ARG(n >= 0 && n <= INT32_MAX && out && (n == 0 || (score && label && keep && workspace)),
                  "rank_curve: bad args (n <= 2^31 - 1)");
  cudaStream_t st = (cudaStream_t)stream_;
  if (n == 0) {       // no pair: AUROC 0, AUPRC NaN
    k_curve_finish<<<1, kThreads, 0, st>>>(nullptr, 0, 0, nullptr, nullptr, nullptr, out);
    DMPNN_CHECK_LAUNCH("rank_curve", 1);
    return 0;
  }
  CurveLayout L;
  if (int rc = curve_layout(n, &L)) return rc;
  DMPNN_CHECK_ARG(workspace_bytes >= L.total, "rank_curve: workspace of %zu bytes, %zu needed", workspace_bytes, L.total);
  char* ws = (char*)workspace;
  uint32_t* key_in = (uint32_t*)(ws + L.key_in);
  uint32_t* key_out = (uint32_t*)(ws + L.key_out);
  uint8_t* val_in = (uint8_t*)(ws + L.val_in);
  uint8_t* val_out = (uint8_t*)(ws + L.val_out);
  ScanItem* items = (ScanItem*)(ws + L.items);
  long long* part_roc = (long long*)(ws + L.part_roc);
  double* part_prc = (double*)(ws + L.part_prc);
  long long* part_kept = (long long*)(ws + L.part_kept);
  const unsigned blocks = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, 132 * 16));
  k_curve_keys<<<blocks, kThreads, 0, st>>>(score, label, keep, n, key_in, val_in);
  size_t tb = L.temp_bytes;
  cudaError_t e = cub::DeviceRadixSort::SortPairsDescending(ws + L.temp, tb, key_in, key_out, val_in, val_out, (int)n, 0, 32, st);
  if (e == cudaSuccess) {
    k_curve_items<<<blocks, kThreads, 0, st>>>(key_out, val_out, n, items);
    tb = L.temp_bytes;
    e = cub::DeviceScan::InclusiveScan(ws + L.temp, tb, items, items, ScanOp(), (int)n, st);
  }
  if (e != cudaSuccess) {
    set_error("rank_curve: cub failed: %s", cudaGetErrorString(e));
    return -2;
  }
  k_curve_partials<<<(unsigned)L.G, kThreads, 0, st>>>(key_out, items, n, L.chunk, part_roc, part_prc, part_kept);
  k_curve_finish<<<1, kThreads, 0, st>>>(items, n, L.G, part_roc, part_prc, part_kept, out);
  DMPNN_CHECK_LAUNCH("rank_curve", 4);
  return 0;
}
