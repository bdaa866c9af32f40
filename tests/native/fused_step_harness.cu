// Kernel-development harness for the fused depth step, WITHOUT Python (a gpurun call costs ~75 s of budget instead of
// ~200 s with a torch import): synthetic molecules -> dmpnn_layout_build -> dmpnn_bond_step_fused_bf16, timed with CUDA
// events (median of 20) and checked against a host computation on a sample of rows.
//   ./tests/native/fused_step_harness [n_mols=10000] [h=300] [pack=0|1|2 (2 = both orders)]
// Reports per order: tiles, fill, us per launch (t >= 2 and first step), algorithmic GB/s, fraction of the H100 SXM data sheet's 3350 GB/s.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../include/dmpnn.h"

#define CK(x)                                                                                  \
  do {                                                                                         \
    cudaError_t e__ = (x);                                                                     \
    if (e__ != cudaSuccess) {                                                                  \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__);         \
      exit(2);                                                                                 \
    }                                                                                          \
  } while (0)
#define DM(x)                                                                                  \
  do {                                                                                         \
    if ((x) != 0) {                                                                            \
      printf("dmpnn error at %s:%d: %s\n", __FILE__, __LINE__, dmpnn_last_error());            \
      exit(1);                                                                                 \
    }                                                                                          \
  } while (0)

static uint64_t rs = 0x2545F4914F6CDD1Dull;
static uint32_t rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return (uint32_t)(rs >> 32); }
static float rndn() {  // ~N(0,1): sum of 12 uniforms (molecule sizes only: a few thousand calls)
  float s = 0;
  for (int i = 0; i < 12; ++i) s += (rnd() & 0xffffff) / 16777216.f;
  return s - 6.f;
}
static inline float rndu() {  // cheap zero-mean unit-variance value for the big buffers (one xorshift per value)
  return ((int32_t)rnd()) * (1.7320508f / 2147483648.f);
}
template <typename T> static T* dalloc(size_t n) { T* p; CK(cudaMalloc(&p, (n ? n : 1) * sizeof(T) + 256)); return p; }
template <typename T> static T* to_dev(const std::vector<T>& h) {
  T* d = dalloc<T>(h.size());
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}
static float bf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

struct Mol { int na; std::vector<int> u, v; };   // bonds (u, v)

static Mol make_mol() {  // random tree + a few ring closures, degree <= 4 (like chemprop_b200/data/synthetic.py)
  Mol m;
  int n = (int)lroundf(25.f + 5.f * rndn());
  m.na = std::min(60, std::max(2, n));
  std::vector<int> deg(m.na, 0);
  for (int a = 1; a < m.na; ++a) {
    int p = -1;
    for (int tries = 0; tries < 16 && p < 0; ++tries) {
      int c = std::max(0, a - 6) + (int)(rnd() % (a - std::max(0, a - 6)));
      if (deg[c] < 4) p = c;
    }
    if (p < 0) p = a - 1;
    m.u.push_back(p); m.v.push_back(a); ++deg[p]; ++deg[a];
  }
  int rings = 0;
  for (int a = 0; a < m.na; ++a) rings += (rnd() % 100) < 6;
  for (int r = 0; r < rings; ++r) {
    int a = (int)(rnd() % m.na), b = (int)(rnd() % m.na);
    if (a == b || deg[a] >= 4 || deg[b] >= 4) continue;
    m.u.push_back(std::min(a, b)); m.v.push_back(std::max(a, b)); ++deg[a]; ++deg[b];
  }
  return m;
}

// the two big random operands are generated ONCE (the row count is the same in either molecule order)
static std::vector<__nv_bfloat16> g_H0, g_Hp;

static void run(const std::vector<Mol>& mols, const std::vector<int64_t>& order, int h, const char* tag) {
  const int64_t B = (int64_t)order.size();
  std::vector<int64_t> src, dst, rev, batch;
  int64_t a0 = 0;
  for (int64_t k = 0; k < B; ++k) {
    const Mol& m = mols[(size_t)order[k]];
    for (size_t b = 0; b < m.u.size(); ++b) {
      const int64_t e = (int64_t)src.size();
      src.push_back(a0 + m.u[b]); dst.push_back(a0 + m.v[b]); rev.push_back(e + 1);
      src.push_back(a0 + m.v[b]); dst.push_back(a0 + m.u[b]); rev.push_back(e);
    }
    for (int a = 0; a < m.na; ++a) batch.push_back(k);
    a0 += m.na;
  }
  const int64_t V = a0, E = (int64_t)src.size();
  std::vector<int64_t> ei(2 * E);
  memcpy(ei.data(), src.data(), E * 8); memcpy(ei.data() + E, dst.data(), E * 8);
  int64_t *d_ei = to_dev(ei), *d_rev = to_dev(rev), *d_batch = to_dev(batch);
  int32_t *perm = dalloc<int32_t>(E), *inv = dalloc<int32_t>(E), *rowptr = dalloc<int32_t>(V + 1), *srow = dalloc<int32_t>(E),
          *drow = dalloc<int32_t>(E), *rrow = dalloc<int32_t>(E), *map = dalloc<int32_t>(B + 2), *mrp = dalloc<int32_t>(B + 2),
          *tmp = dalloc<int32_t>(B + 2), *trp = dalloc<int32_t>(B + 2), *tap = dalloc<int32_t>(B + 2), *meta = dalloc<int32_t>(8);
  CK(cudaMemset(map, 0, (B + 2) * 4)); CK(cudaMemset(mrp, 0, (B + 2) * 4)); CK(cudaMemset(tmp, 0, (B + 2) * 4));
  CK(cudaMemset(trp, 0, (B + 2) * 4)); CK(cudaMemset(tap, 0, (B + 2) * 4)); CK(cudaMemset(meta, 0, 32));
  size_t wsb = 0; DM(dmpnn_layout_workspace_bytes(V, E, B, &wsb));
  void* ws = dalloc<char>(wsb);
  DM(dmpnn_layout_build(d_ei, d_rev, d_batch, V, E, B, perm, inv, rowptr, srow, drow, rrow, map, mrp, tmp, trp, tap, meta, ws, nullptr));
  int32_t hm[8]; CK(cudaMemcpy(hm, meta, 32, cudaMemcpyDeviceToHost));
  const int n_tiles = hm[DMPNN_META_N_TILES];
  if (hm[DMPNN_META_FLAGS] != 7 || hm[DMPNN_META_MAX_TILE_ROWS] > 128) { printf("bad layout: flags %d max rows %d\n", hm[1], hm[3]); exit(1); }
  const int64_t ld = (h + 63) / 64 * 64;
  if (g_H0.size() != (size_t)E * ld) {
    g_H0.assign((size_t)E * ld, __float2bfloat16_rn(0.f));
    g_Hp.assign((size_t)E * ld, __float2bfloat16_rn(0.f));
    for (int64_t r = 0; r < E; ++r)
      for (int c = 0; c < h; ++c) {
        g_H0[(size_t)r * ld + c] = __float2bfloat16_rn(0.5f * rndu());
        g_Hp[(size_t)r * ld + c] = __float2bfloat16_rn(fmaxf(0.5f * rndu(), 0.f));
      }
  }
  const std::vector<__nv_bfloat16>&H0 = g_H0, &Hp = g_Hp;
  std::vector<float> W((size_t)h * h);
  for (auto& w : W) w = rndu() / sqrtf((float)h);
  __nv_bfloat16 *dH0 = to_dev(H0), *dHp = to_dev(Hp), *dHn = dalloc<__nv_bfloat16>((size_t)E * ld);
  float* dW = to_dev(W);
  size_t pkb = 0; DM(dmpnn_pack_weight_bf16_bytes(h, h, &pkb));
  void* Wpk = dalloc<char>(pkb);
  DM(dmpnn_pack_weight_bf16(dW, h, h, h, Wpk, nullptr));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  float med[2];
  for (int first = 0; first < 2; ++first) {
    std::vector<float> ts;
    for (int it = 0; it < 23; ++it) {
      CK(cudaEventRecord(e0));
      DM(dmpnn_bond_step_fused_bf16(first ? dH0 : dHp, dH0, dHn, ld, E, h, Wpk, nullptr, rowptr, rrow, trp, tap, n_tiles,
                                    DMPNN_ACT_RELU, 0.f, first, nullptr, nullptr, nullptr, nullptr, nullptr, 1.f, nullptr));
      CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
      if (it >= 3) ts.push_back(ms);
    }
    std::sort(ts.begin(), ts.end());
    med[first] = ts[ts.size() / 2];
  }
  // correctness of the t >= 2 launch (re-run it last) on a sample of atoms: rows of atom v are [rowptr[v], rowptr[v+1])
  DM(dmpnn_bond_step_fused_bf16(dHp, dH0, dHn, ld, E, h, Wpk, nullptr, rowptr, rrow, trp, tap, n_tiles, DMPNN_ACT_RELU, 0.f, 0, nullptr, nullptr, nullptr, nullptr, nullptr, 1.f, nullptr));
  CK(cudaDeviceSynchronize());
  std::vector<__nv_bfloat16> Hn((size_t)E * ld);
  CK(cudaMemcpy(Hn.data(), dHn, Hn.size() * 2, cudaMemcpyDeviceToHost));
  std::vector<int32_t> h_rowptr(V + 1), h_rrow(E);
  CK(cudaMemcpy(h_rowptr.data(), rowptr, (V + 1) * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h_rrow.data(), rrow, E * 4, cudaMemcpyDeviceToHost));
  double max_err = 0; int64_t checked = 0;
  std::vector<float> s(h), Mrow(h);
  for (int64_t v = 0; v < V; v += std::max<int64_t>(1, V / 400)) {
    const int r0 = h_rowptr[v], r1 = h_rowptr[v + 1];
    std::fill(s.begin(), s.end(), 0.f);
    for (int r = r0; r < r1; ++r)
      for (int c = 0; c < h; ++c) s[c] += __bfloat162float(Hp[(size_t)r * ld + c]);
    for (int r = r0; r < r1; ++r) {                       // in-edge row r of atom v: the message goes to row rev(r)
      const int out = h_rrow[r];
      for (int c = 0; c < h; ++c) Mrow[c] = bf(s[c] - __bfloat162float(Hp[(size_t)r * ld + c]));
      for (int n = 0; n < h; n += 7) {                    // a sample of output columns
        float z = __bfloat162float(H0[(size_t)out * ld + n]);
        for (int c = 0; c < h; ++c) z += Mrow[c] * bf(W[(size_t)n * h + c]);
        const float want = fmaxf(z, 0.f), got = __bfloat162float(Hn[(size_t)out * ld + n]);
        max_err = std::max(max_err, (double)fabsf(want - got) / (1.0 + fabs(want)));
        ++checked;
      }
    }
  }
  const double bytes[2] = {3.0 * E * h * 2 + 12.0 * E + 4.0 * V, 2.0 * E * h * 2 + 12.0 * E + 4.0 * V};
  printf("[%s] mols %lld atoms %lld rows %lld tiles %d fill %.3f | t>=2: %.1f us %.0f GB/s frac %.3f | first: %.1f us %.0f GB/s | "
         "check: %lld values, max rel err %.2e %s\n", tag, (long long)B, (long long)V, (long long)E, n_tiles, E / (128.0 * n_tiles),
         med[0] * 1e3, bytes[0] / med[0] / 1e6, bytes[0] / med[0] / 1e6 / 3350.0, med[1] * 1e3, bytes[1] / med[1] / 1e6,
         (long long)checked, max_err, max_err < 3e-2 ? "OK" : "MISMATCH");
}

int main(int argc, char** argv) {
  setvbuf(stdout, nullptr, _IOLBF, 0);
  const int64_t n = argc > 1 ? atoll(argv[1]) : 10000;
  const int h = argc > 2 ? atoi(argv[2]) : 300;
  const int pack = argc > 3 ? atoi(argv[3]) : 2;
  const bool dry = getenv("HARNESS_DRY") != nullptr;     // host preparation only (timing it without a GPU)
  if (!dry && dmpnn_device_ok() != 1) { printf("no H100 (sm_90) device\n"); return 3; }
  std::vector<Mol> mols((size_t)n);
  std::vector<int64_t> na((size_t)n), ne((size_t)n), ident((size_t)n), packed((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    mols[(size_t)i] = make_mol();
    na[(size_t)i] = mols[(size_t)i].na; ne[(size_t)i] = 2 * (int64_t)mols[(size_t)i].u.size(); ident[(size_t)i] = i;
  }
  DM(dmpnn_tile_pack_order(n, na.data(), ne.data(), packed.data()));
  if (dry) {
    std::vector<__nv_bfloat16> buf((size_t)n * 50 * 320);
    for (auto& x : buf) x = __float2bfloat16_rn(0.5f * rndu());
    printf("dry run: %lld molecules prepared, %zu values filled\n", (long long)n, buf.size());
    return 0;
  }
  if (pack == 0 || pack == 2) run(mols, ident, h, "arrival order");
  if (pack == 1 || pack == 2) run(mols, packed, h, "tile-packed  ");
  return 0;
}
