// Hardware check of the two kernels added after the round's GPU budget was spent, WITHOUT Python (starts in ~1 s):
//   dmpnn_dataset_gather  vs  dmpnn_dataset_gather_host  (bit-exact, all five BatchMolGraph arrays)
//   dmpnn_scale_mask      vs  a host computation          (f32 and bf16, in place)
// Build (cross-compiles without a GPU):  see tests/native/Makefile.   Run on an H100:  ./tests/native/check_new_kernels
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../include/dmpnn.h"

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e__ = (x);                                                         \
    if (e__ != cudaSuccess) {                                                      \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return 2;                                                                    \
    }                                                                              \
  } while (0)

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint32_t rnd() {
  rng_state ^= rng_state << 13;
  rng_state ^= rng_state >> 7;
  rng_state ^= rng_state << 17;
  return (uint32_t)(rng_state >> 32);
}

template <typename T>
static T* to_dev(const std::vector<T>& h) {
  T* d = nullptr;
  if (cudaMalloc(&d, h.size() * sizeof(T) + 16) != cudaSuccess) return nullptr;
  cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  return d;
}

static int check_gather(int64_t d_v, int64_t d_e) {
  const int64_t n = 3000, n_sel = 2200;
  std::vector<int64_t> atom_ptr(n + 1, 0), edge_ptr(n + 1, 0);
  std::vector<int32_t> max_indeg(n, 3);
  for (int64_t m = 0; m < n; ++m) {
    const int64_t na = 1 + rnd() % 40, nb = (na == 1) ? 0 : (na - 1 + rnd() % 3);
    atom_ptr[m + 1] = atom_ptr[m] + na;
    edge_ptr[m + 1] = edge_ptr[m] + 2 * nb;
  }
  const int64_t Vt = atom_ptr[n], Et = edge_ptr[n];
  std::vector<float> V_all(Vt * d_v), E_all(Et * d_e);
  for (auto& x : V_all) x = (float)(rnd() % 2048) / 64.f - 16.f;
  for (auto& x : E_all) x = (float)(rnd() % 2048) / 64.f - 16.f;
  std::vector<int32_t> ei(2 * Et), rev(Et);
  for (int64_t m = 0; m < n; ++m) {
    const int64_t na = atom_ptr[m + 1] - atom_ptr[m], se = edge_ptr[m], ne = edge_ptr[m + 1] - se;
    for (int64_t j = 0; j < ne; j += 2) {
      const int32_t u = (int32_t)(rnd() % na), v = (int32_t)(rnd() % na);
      ei[se + j] = u; ei[Et + se + j] = v; ei[se + j + 1] = v; ei[Et + se + j + 1] = u;
      rev[se + j] = (int32_t)(j + 1); rev[se + j + 1] = (int32_t)j;
    }
  }
  std::vector<int64_t> ids(n_sel), oap(n_sel + 1), oep(n_sel + 1);
  for (auto& x : ids) x = rnd() % n;
  int32_t meta[DMPNN_META_WORDS];
  if (dmpnn_dataset_batch_meta_host(n_sel, ids.data(), n, atom_ptr.data(), edge_ptr.data(), max_indeg.data(), oap.data(),
                                    oep.data(), meta) != 0) { printf("meta_host failed: %s\n", dmpnn_last_error()); return 1; }
  const int64_t Vo = oap[n_sel], Eo = oep[n_sel];
  std::vector<float> hV(Vo * d_v), hE(Eo * d_e);
  std::vector<int64_t> hei(2 * Eo), hrev(Eo), hb(Vo);
  if (dmpnn_dataset_gather_host(n_sel, ids.data(), oap.data(), oep.data(), atom_ptr.data(), edge_ptr.data(), V_all.data(),
                                E_all.data(), ei.data(), rev.data(), Et, d_v, d_e, hV.data(), hE.data(), hei.data(), hrev.data(),
                                hb.data(), nullptr, nullptr, nullptr, nullptr, nullptr, 0) != 0) {
    printf("gather_host failed: %s\n", dmpnn_last_error()); return 1; }
  int64_t *d_ids = to_dev(ids), *d_oap = to_dev(oap), *d_oep = to_dev(oep), *d_ap = to_dev(atom_ptr), *d_ep = to_dev(edge_ptr);
  float *d_V = to_dev(V_all), *d_E = to_dev(E_all);
  int32_t *d_ei = to_dev(ei), *d_rev = to_dev(rev);
  float *o_V, *o_E; int64_t *o_ei, *o_rev, *o_b;
  CK(cudaMalloc(&o_V, Vo * d_v * 4 + 16)); CK(cudaMalloc(&o_E, Eo * d_e * 4 + 16));
  CK(cudaMalloc(&o_ei, 2 * Eo * 8 + 16)); CK(cudaMalloc(&o_rev, Eo * 8 + 16)); CK(cudaMalloc(&o_b, Vo * 8 + 16));
  CK(cudaMemset(o_V, 0xff, Vo * d_v * 4)); CK(cudaMemset(o_E, 0xff, Eo * d_e * 4));
  cudaStream_t st; CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  int rc = 0;
  for (int it = 0; it < 3; ++it) {
    CK(cudaEventRecord(e0, st));
    rc = dmpnn_dataset_gather(d_ids, d_oap, d_oep, n_sel, d_ap, d_ep, d_V, d_E, d_ei, d_rev, Et, d_v, d_e, o_V, o_E, o_ei, o_rev,
                              o_b, Eo, st);
    CK(cudaEventRecord(e1, st));
  }
  if (rc != 0) { printf("dataset_gather failed: %s\n", dmpnn_last_error()); return 1; }
  CK(cudaStreamSynchronize(st));
  float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
  std::vector<float> gV(Vo * d_v), gE(Eo * d_e);
  std::vector<int64_t> gei(2 * Eo), grev(Eo), gb(Vo);
  CK(cudaMemcpy(gV.data(), o_V, gV.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gE.data(), o_E, gE.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gei.data(), o_ei, gei.size() * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(grev.data(), o_rev, grev.size() * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(gb.data(), o_b, gb.size() * 8, cudaMemcpyDeviceToHost));
  const bool ok = !memcmp(gV.data(), hV.data(), gV.size() * 4) && !memcmp(gE.data(), hE.data(), gE.size() * 4) &&
                  !memcmp(gei.data(), hei.data(), gei.size() * 8) && !memcmp(grev.data(), hrev.data(), grev.size() * 8) &&
                  !memcmp(gb.data(), hb.data(), gb.size() * 8);
  const double bytes = 2.0 * (gV.size() + gE.size()) * 4 + 40.0 * Eo + 8.0 * Vo;
  printf("dataset_gather d_v=%lld d_e=%lld: %lld molecules, %lld atoms, %lld edges, tiles=%d: %s  (%.1f us, %.0f GB/s)\n",
         (long long)d_v, (long long)d_e, (long long)n_sel, (long long)Vo, (long long)Eo, meta[DMPNN_META_N_TILES],
         ok ? "BIT-EXACT vs host gather" : "MISMATCH", ms * 1e3, bytes / ms / 1e6);
  return ok ? 0 : 1;
}

static int check_scale_mask() {
  const int64_t n = 1000003;
  const float scale = 1.0f / 0.7f;
  std::vector<float> x(n), m(n);
  for (int64_t i = 0; i < n; ++i) { x[i] = (float)(rnd() % 4096) / 256.f - 8.f; m[i] = (rnd() % 10) < 7 ? 1.f : 0.f; }
  float *dx = to_dev(x), *dm = to_dev(m);
  if (dmpnn_scale_mask(dx, dm, dx, DMPNN_F32, n, scale, nullptr) != 0) { printf("scale_mask f32: %s\n", dmpnn_last_error()); return 1; }
  std::vector<float> g(n);
  CK(cudaMemcpy(g.data(), dx, n * 4, cudaMemcpyDeviceToHost));
  int64_t bad = 0;
  for (int64_t i = 0; i < n; ++i) bad += g[i] != x[i] * m[i] * scale;
  std::vector<__nv_bfloat16> xb(n), mb(n);
  for (int64_t i = 0; i < n; ++i) { xb[i] = __float2bfloat16_rn(x[i]); mb[i] = __float2bfloat16_rn(m[i]); }
  __nv_bfloat16 *dxb = to_dev(xb), *dmb = to_dev(mb);
  if (dmpnn_scale_mask(dxb, dmb, dxb, DMPNN_BF16, n, scale, nullptr) != 0) { printf("scale_mask bf16: %s\n", dmpnn_last_error()); return 1; }
  std::vector<__nv_bfloat16> gb(n);
  CK(cudaMemcpy(gb.data(), dxb, n * 2, cudaMemcpyDeviceToHost));
  int64_t badb = 0;
  for (int64_t i = 0; i < n; ++i) {
    const __nv_bfloat16 want = __float2bfloat16_rn(__bfloat162float(xb[i]) * __bfloat162float(mb[i]) * scale);
    badb += memcmp(&want, &gb[i], 2) != 0;
  }
  printf("scale_mask: f32 %lld mismatches, bf16 %lld mismatches of %lld: %s\n", (long long)bad, (long long)badb, (long long)n,
         (bad == 0 && badb == 0) ? "EXACT" : "MISMATCH");
  return (bad == 0 && badb == 0) ? 0 : 1;
}

int main() {
  if (dmpnn_device_ok() != 1) { printf("no H100 (sm_90) device\n"); return 3; }
  int rc = 0;
  rc |= check_gather(72, 14);
  rc |= check_gather(106, 28);
  rc |= check_gather(7, 3);
  rc |= check_scale_mask();
  printf(rc == 0 ? "ALL OK\n" : "FAILED\n");
  return rc;
}
