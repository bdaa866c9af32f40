// Device-resident packed dataset: assemble a BatchMolGraph for a list of molecule ids with ONE launch.
//
// Replaces, for pre-featurised data, `[dataset[i] for i in ids]` + collate_batch + the host -> device copy of the
// batch (chemprop/data/datasets.py:222-244, chemprop/data/collate.py:37-97): the dataset's flat arrays stay in HBM
// (1 M ~25-atom molecules: 7.2 GB of atom features, 3 GB of bond features, 0.8 GB of local indices -- of the H100's 80 GB), a
// training step uploads only the ids and the output offsets (24 bytes per molecule) and this kernel copies each
// selected molecule's rows to its place in the batch, turning molecule-local indices into batch-global ones.
// Pure HBM streaming: 2 x (4 d_v V + 4 d_e E) + 40 E + 8 V bytes per batch, no reuse, no arithmetic beyond the offsets.
#include "common.cuh"

namespace {

// copy n contiguous elements; W = elements per vector access (the caller guarantees both pointers are W-aligned)
template <int W>
__device__ __forceinline__ void copy_span(const float* __restrict__ src, float* __restrict__ dst, int64_t n) {
  if constexpr (W == 4) {
    const float4* s = reinterpret_cast<const float4*>(src);
    float4* d = reinterpret_cast<float4*>(dst);
    for (int64_t i = threadIdx.x; i < n / 4; i += blockDim.x) d[i] = s[i];
  } else if constexpr (W == 2) {
    const float2* s = reinterpret_cast<const float2*>(src);
    float2* d = reinterpret_cast<float2*>(dst);
    for (int64_t i = threadIdx.x; i < n / 2; i += blockDim.x) d[i] = s[i];
  } else {
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
  }
}

// one block per selected molecule
template <int WV, int WE>
__global__ void __launch_bounds__(128)
k_dataset_gather(const int64_t* __restrict__ ids, const int64_t* __restrict__ out_atom_ptr,
                 const int64_t* __restrict__ out_edge_ptr, const int64_t* __restrict__ atom_ptr,
                 const int64_t* __restrict__ edge_ptr, const float* __restrict__ V_all, const float* __restrict__ E_all,
                 const int32_t* __restrict__ ei_local, const int32_t* __restrict__ rev_local, int64_t E_all_total,
                 int d_v, int d_e, float* __restrict__ V_out, float* __restrict__ E_out, int64_t* __restrict__ ei_out,
                 int64_t* __restrict__ rev_out, int64_t* __restrict__ batch_out, int64_t E_out_total) {
  const int64_t m = blockIdx.x;
  const int64_t id = ids[m];
  const int64_t sa = atom_ptr[id], se = edge_ptr[id];
  const int64_t na = atom_ptr[id + 1] - sa, ne = edge_ptr[id + 1] - se;
  const int64_t oa = out_atom_ptr[m], oe = out_edge_ptr[m];
  if (d_v > 0) copy_span<WV>(V_all + sa * d_v, V_out + oa * d_v, na * d_v);
  if (d_e > 0) copy_span<WE>(E_all + se * d_e, E_out + oe * d_e, ne * d_e);
  const int32_t* s0 = ei_local + se;
  const int32_t* s1 = ei_local + E_all_total + se;
  const int32_t* rv = rev_local + se;
  for (int64_t j = threadIdx.x; j < ne; j += blockDim.x) {
    ei_out[oe + j] = (int64_t)s0[j] + oa;                  // collate.py:51
    ei_out[E_out_total + oe + j] = (int64_t)s1[j] + oa;
    rev_out[oe + j] = (int64_t)rv[j] + oe;                 // collate.py:52
  }
  for (int64_t j = threadIdx.x; j < na; j += blockDim.x) batch_out[oa + j] = m;   // collate.py:53
}

template <int WV>
int launch_we(int we, dim3 grid, cudaStream_t st, const int64_t* ids, const int64_t* oap, const int64_t* oep,
              const int64_t* ap, const int64_t* ep, const float* V_all, const float* E_all, const int32_t* ei,
              const int32_t* rv, int64_t Eall, int d_v, int d_e, float* V_out, float* E_out, int64_t* ei_out,
              int64_t* rev_out, int64_t* batch_out, int64_t Eout) {
#define DMPNN_GATHER_LAUNCH(WE)                                                                                        \
  k_dataset_gather<WV, WE><<<grid, 128, 0, st>>>(ids, oap, oep, ap, ep, V_all, E_all, ei, rv, Eall, d_v, d_e, V_out, \
                                                 E_out, ei_out, rev_out, batch_out, Eout)
  if (we == 4) DMPNN_GATHER_LAUNCH(4);
  else if (we == 2) DMPNN_GATHER_LAUNCH(2);
  else DMPNN_GATHER_LAUNCH(1);
#undef DMPNN_GATHER_LAUNCH
  return 0;
}

inline int vec_width(int64_t d, const void* a, const void* b) {
  const uintptr_t bits = reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b);
  if (d % 4 == 0 && bits % 16 == 0) return 4;     // every row offset is then a multiple of 16 bytes
  if (d % 2 == 0 && bits % 8 == 0) return 2;
  return 1;
}

}  // namespace

extern "C" int dmpnn_dataset_gather(const int64_t* ids, const int64_t* out_atom_ptr, const int64_t* out_edge_ptr,
                                    int64_t n_sel, const int64_t* atom_ptr, const int64_t* edge_ptr, const float* V_all,
                                    const float* E_all, const int32_t* ei_local, const int32_t* rev_local,
                                    int64_t E_all_total, int64_t d_v, int64_t d_e, float* V_out, float* E_out,
                                    int64_t* ei_out, int64_t* rev_out, int64_t* batch_out, int64_t E_out_total,
                                    void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(n_sel >= 0 && d_v >= 0 && d_e >= 0 && E_all_total >= 0 && E_out_total >= 0 && n_sel < (1LL << 31),
                  "dataset_gather: bad sizes");
  if (n_sel == 0) return 0;
  DMPNN_CHECK_ARG(ids && out_atom_ptr && out_edge_ptr && atom_ptr && edge_ptr && batch_out, "dataset_gather: null table");
  DMPNN_CHECK_ARG((d_v == 0 || (V_all && V_out)) && (d_e == 0 || E_out_total == 0 || (E_all && E_out)),
                  "dataset_gather: null feature array");
  DMPNN_CHECK_ARG(E_out_total == 0 || (ei_local && rev_local && ei_out && rev_out), "dataset_gather: null index array");
  const int wv = vec_width(d_v, V_all, V_out), we = vec_width(d_e, E_all, E_out);
  dim3 grid((unsigned)n_sel);
#define DMPNN_GATHER_WV(WV)                                                                                          \
  launch_we<WV>(we, grid, st, ids, out_atom_ptr, out_edge_ptr, atom_ptr, edge_ptr, V_all, E_all, ei_local, rev_local, \
                E_all_total, (int)d_v, (int)d_e, V_out, E_out, ei_out, rev_out, batch_out, E_out_total)
  if (wv == 4) DMPNN_GATHER_WV(4);
  else if (wv == 2) DMPNN_GATHER_WV(2);
  else DMPNN_GATHER_WV(1);
#undef DMPNN_GATHER_WV
  DMPNN_CHECK_LAUNCH("dmpnn_dataset_gather", 1);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Dropout application (base.py:139, :182): OUT = X * M * scale over a flat, contiguous buffer of n elements (the hidden
// matrix including its zero padding columns), M a {0, 1} keep mask of the same element type drawn by the caller's RNG.
// In place allowed (OUT == X).  The product is formed in f32 with the exact scale 1 / (1 - p) and rounded once.
namespace {
template <typename T>
__global__ void __launch_bounds__(256) k_scale_mask(const T* __restrict__ X, const T* __restrict__ M, T* OUT, int64_t n,
                                                    float scale, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    const int64_t n4 = n / 4;
    for (int64_t q = i; q < n4; q += stride) {
      float x[4], m[4];
      dmpnn::ld4(X + 4 * q, x);
      dmpnn::ld4(M + 4 * q, m);
#pragma unroll
      for (int k = 0; k < 4; ++k) x[k] = x[k] * m[k] * scale;
      dmpnn::st4(OUT + 4 * q, x);
    }
    for (int64_t j = 4 * n4 + i; j < n; j += stride)
      dmpnn::st_from_float(OUT + j, dmpnn::ld_as_float(X + j) * dmpnn::ld_as_float(M + j) * scale);
  } else {
    for (int64_t j = i; j < n; j += stride)
      dmpnn::st_from_float(OUT + j, dmpnn::ld_as_float(X + j) * dmpnn::ld_as_float(M + j) * scale);
  }
}
}  // namespace

// ---- dropout keep bits (Philox4x32-10, the counter-based generator torch's CUDA stream uses) -----------------------
// One thread = one (row, 16-column block): 16 keep bits, bit q = [u16_q >= thr], u16_q = 16 random bits of the block's
// 256-bit Philox output (2 counters), thr = round(p * 65536): P(drop) = thr / 65536.  Counter = (word index, offset);
// key = seed: the same (seed, offset) gives the same bits on every launch, whatever the grid.
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
}
__device__ __forceinline__ void philox4x32_10(uint64_t seed, uint64_t ctr_lo, uint64_t ctr_hi, uint32_t (&out)[4]) {
  uint32_t c[4] = {(uint32_t)ctr_lo, (uint32_t)(ctr_lo >> 32), (uint32_t)ctr_hi, (uint32_t)(ctr_hi >> 32)};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = c[i];
}
__global__ void k_dropout_bits(uint16_t* __restrict__ bits, int64_t n_words, uint64_t seed, uint64_t offset, uint32_t thr) {
  const int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  uint32_t a[4], b[4];
  philox4x32_10(seed, (uint64_t)(2 * w), offset, a);
  philox4x32_10(seed, (uint64_t)(2 * w + 1), offset, b);
  const uint32_t u[8] = {a[0], a[1], a[2], a[3], b[0], b[1], b[2], b[3]};
  uint32_t m = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    m |= ((u[q] & 0xffffu) >= thr ? 1u : 0u) << (2 * q);
    m |= ((u[q] >> 16) >= thr ? 1u : 0u) << (2 * q + 1);
  }
  bits[w] = (uint16_t)m;
}

extern "C" int dmpnn_dropout_bits(void* bits, int64_t n_rows, int64_t words_per_row, float p, uint64_t seed, uint64_t offset,
                                  void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(bits && n_rows >= 0 && words_per_row > 0 && p >= 0.f && p < 1.f, "dropout_bits: bad args (0 <= p < 1)");
  const int64_t n = n_rows * words_per_row;
  if (n == 0) return 0;
  const uint32_t thr = (uint32_t)(p * 65536.0f + 0.5f);
  k_dropout_bits<<<dmpnn::ceil_div_i64(n, 256), 256, 0, st>>>((uint16_t*)bits, n, seed, offset, thr);
  DMPNN_CHECK_LAUNCH("dropout_bits", 1);
  return 0;
}

extern "C" int dmpnn_scale_mask(const void* X, const void* M, void* OUT, int dtype, int64_t n, float scale, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(n >= 0 && (n == 0 || (X && M && OUT)), "scale_mask: bad args");
  DMPNN_CHECK_ARG(dtype == DMPNN_F32 || dtype == DMPNN_BF16, "scale_mask: bad dtype");
  if (n == 0) return 0;
  int64_t blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (sm_count <= 0) sm_count = 132;
  }
  if (blocks > (int64_t)sm_count * 16) blocks = (int64_t)sm_count * 16;
  if (dtype == DMPNN_F32) {
    const int vec = dmpnn::vec4_ok<float>(X, 4) && dmpnn::vec4_ok<float>(M, 4) && dmpnn::vec4_ok<float>(OUT, 4);
    k_scale_mask<float><<<(unsigned)blocks, 256, 0, st>>>((const float*)X, (const float*)M, (float*)OUT, n, scale, vec);
  } else {
    const int vec = dmpnn::vec4_ok<__nv_bfloat16>(X, 4) && dmpnn::vec4_ok<__nv_bfloat16>(M, 4) &&
                    dmpnn::vec4_ok<__nv_bfloat16>(OUT, 4);
    k_scale_mask<__nv_bfloat16><<<(unsigned)blocks, 256, 0, st>>>((const __nv_bfloat16*)X, (const __nv_bfloat16*)M,
                                                                   (__nv_bfloat16*)OUT, n, scale, vec);
  }
  DMPNN_CHECK_LAUNCH("dmpnn_scale_mask", 1);
  return 0;
}
