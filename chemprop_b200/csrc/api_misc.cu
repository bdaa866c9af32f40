// Version / error plumbing and the host-side collate of libdmpnn_sm90.so.
#include <stdarg.h>
#include <atomic>
#include <string.h>
#include <algorithm>
#include <functional>
#include <thread>
#include <vector>

#include "common.cuh"

namespace dmpnn {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
}  // namespace dmpnn

extern "C" {

long long dmpnn_launch_count(void) { return dmpnn::g_launches.load(std::memory_order_relaxed); }

int dmpnn_version(void) { return DMPNN_VERSION; }

const char* dmpnn_last_error(void) { return dmpnn::g_err; }

int dmpnn_device_ok(void) {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return 0; }
  int major = 0, minor = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return (major == 9 && minor == 0) ? 1 : 0;   // sm_90a code runs on compute capability 9.0 only
}

// Replaces the per-molecule Python loop of BatchMolGraph.__post_init__
// (chemprop/data/collate.py:37-62): concatenate V/E, offset edge_index by the running atom
// count (:51), rev_edge_index by the running edge count (:52), batch[i-th mol's atoms] = i (:53).
int dmpnn_collate_host(int64_t n_mols, const int64_t* n_atoms, const int64_t* n_edges,
                       const float* const* V_ptrs, const float* const* E_ptrs,
                       const int64_t* const* edge_index_ptrs, const int64_t* const* rev_ptrs,
                       int64_t d_v, int64_t d_e, float* V_out, float* E_out,
                       int64_t* edge_index_out, int64_t* rev_out, int64_t* batch_out) {
  DMPNN_CHECK_ARG(n_mols >= 0 && d_v >= 0 && d_e >= 0, "collate_host: negative size");
  int64_t E_tot = 0;
  for (int64_t i = 0; i < n_mols; ++i) {
    DMPNN_CHECK_ARG(n_atoms[i] >= 0 && n_edges[i] >= 0, "collate_host: negative molecule size");
    E_tot += n_edges[i];
  }
  int64_t a0 = 0, e0 = 0;
  for (int64_t i = 0; i < n_mols; ++i) {
    const int64_t na = n_atoms[i], ne = n_edges[i];
    if (na > 0 && d_v > 0) memcpy(V_out + a0 * d_v, V_ptrs[i], sizeof(float) * na * d_v);
    if (ne > 0 && d_e > 0) memcpy(E_out + e0 * d_e, E_ptrs[i], sizeof(float) * ne * d_e);
    const int64_t* ei = edge_index_ptrs[i];
    const int64_t* rv = rev_ptrs[i];
    for (int64_t j = 0; j < ne; ++j) {
      edge_index_out[e0 + j] = ei[j] + a0;
      edge_index_out[E_tot + e0 + j] = ei[ne + j] + a0;
      rev_out[e0 + j] = rv[j] + e0;
    }
    for (int64_t j = 0; j < na; ++j) batch_out[a0 + j] = i;
    a0 += na;
    e0 += ne;
  }
  return 0;
}

static inline uint16_t f32_to_bf16_rne(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  if ((x & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((x >> 16) | 0x40u);   // NaN stays NaN (quiet)
  x += 0x7fffu + ((x >> 16) & 1u);                                             // round to nearest, ties to even
  return (uint16_t)(x >> 16);
}

// Compact transfer copy of the same batch (bf16 features, int32 indices): what BatchMolGraph(transfer_dtype=bfloat16)
// ships over PCIe.  One pass over the per-molecule arrays, same offsets as dmpnn_collate_host.
int dmpnn_collate_host_compact(int64_t n_mols, const int64_t* n_atoms, const int64_t* n_edges,
                               const float* const* V_ptrs, const float* const* E_ptrs,
                               const int64_t* const* edge_index_ptrs, const int64_t* const* rev_ptrs,
                               int64_t d_v, int64_t d_e, uint16_t* V_out, uint16_t* E_out,
                               int32_t* edge_index_out, int32_t* rev_out, int32_t* batch_out) {
  DMPNN_CHECK_ARG(n_mols >= 0 && d_v >= 0 && d_e >= 0, "collate_host_compact: negative size");
  int64_t E_tot = 0, V_tot = 0;
  for (int64_t i = 0; i < n_mols; ++i) {
    DMPNN_CHECK_ARG(n_atoms[i] >= 0 && n_edges[i] >= 0, "collate_host_compact: negative molecule size");
    E_tot += n_edges[i];
    V_tot += n_atoms[i];
  }
  DMPNN_CHECK_ARG(E_tot < (1LL << 31) && V_tot < (1LL << 31) && n_mols < (1LL << 31),
                  "collate_host_compact: batch too large for int32 indices");
  int64_t a0 = 0, e0 = 0;
  for (int64_t i = 0; i < n_mols; ++i) {
    const int64_t na = n_atoms[i], ne = n_edges[i];
    const float* v = V_ptrs[i];
    const float* e = E_ptrs[i];
    for (int64_t j = 0; j < na * d_v; ++j) V_out[a0 * d_v + j] = f32_to_bf16_rne(v[j]);
    for (int64_t j = 0; j < ne * d_e; ++j) E_out[e0 * d_e + j] = f32_to_bf16_rne(e[j]);
    const int64_t* ei = edge_index_ptrs[i];
    const int64_t* rv = rev_ptrs[i];
    for (int64_t j = 0; j < ne; ++j) {
      edge_index_out[e0 + j] = (int32_t)(ei[j] + a0);
      edge_index_out[E_tot + e0 + j] = (int32_t)(ei[ne + j] + a0);
      rev_out[e0 + j] = (int32_t)(rv[j] + e0);
    }
    for (int64_t j = 0; j < na; ++j) batch_out[a0 + j] = (int32_t)i;
    a0 += na;
    e0 += ne;
  }
  return 0;
}

// The layout meta words of a batch (dmpnn_layout_build's `meta`), computed on the HOST from the batch's index arrays:
// validity flags, max in-degree and the greedy molecule-aligned tile packing (tile count, largest tile).  A loader
// calls this once per batch next to the collate, so the training step never has to read `meta` back from the device
// (no host <-> device synchronisation inside the step).  Bit-exact w.r.t. oracle/layout_np.py for valid batches; for
// an invalid batch only the flags are meaningful (the tile words are 0).
int dmpnn_batch_meta_host(const int64_t* edge_index /*2 x E*/, const int64_t* rev, const int64_t* batch, int64_t V,
                          int64_t E, int64_t B, int32_t* meta /*DMPNN_META_WORDS*/) {
  DMPNN_CHECK_ARG(V >= 0 && E >= 0 && B >= 0 && meta, "batch_meta_host: bad sizes");
  DMPNN_CHECK_ARG(E == 0 || (edge_index && rev), "batch_meta_host: null index array");
  DMPNN_CHECK_ARG(V == 0 || batch, "batch_meta_host: null batch");
  DMPNN_CHECK_ARG(V < (1LL << 31) && E < (1LL << 31) && B < (1LL << 31), "batch_meta_host: batch too large for int32");
  for (int i = 0; i < DMPNN_META_WORDS; ++i) meta[i] = 0;
  const int64_t* src = edge_index;
  const int64_t* dst = edge_index + E;
  bool in_range = true;
  for (int64_t e = 0; e < E && in_range; ++e)
    in_range = src[e] >= 0 && src[e] < V && dst[e] >= 0 && dst[e] < V && rev[e] >= 0 && rev[e] < E;
  for (int64_t v = 0; v < V && in_range; ++v) in_range = batch[v] >= 0 && batch[v] < B;
  if (!in_range) return 0;                                  // flags = 0: nothing else can be trusted
  bool invol = true, sorted = true;
  for (int64_t e = 0; e < E && invol; ++e) {
    const int64_t r = rev[e];
    invol = rev[r] == e && src[r] == dst[e] && dst[r] == src[e];
  }
  for (int64_t v = 1; v < V && sorted; ++v) sorted = batch[v] >= batch[v - 1];
  for (int64_t e = 0; e < E && sorted; ++e) sorted = batch[src[e]] == batch[dst[e]];
  meta[DMPNN_META_FLAGS] = DMPNN_FLAG_INDEX_IN_RANGE | (invol ? DMPNN_FLAG_REV_INVOLUTION : 0) |
                           (sorted ? DMPNN_FLAG_BATCH_SORTED : 0);
  std::vector<int32_t> deg((size_t)V, 0);
  for (int64_t e = 0; e < E; ++e) ++deg[(size_t)dst[e]];
  int32_t max_indeg = 0;
  for (int64_t v = 0; v < V; ++v) max_indeg = deg[(size_t)v] > max_indeg ? deg[(size_t)v] : max_indeg;
  meta[DMPNN_META_MAX_INDEG] = max_indeg;
  if (!sorted || B == 0) return 0;
  // molecule offsets: atoms of molecule m are [ap[m], ap[m+1]); its edge rows (edges are intra-molecule) [rp[m], rp[m+1])
  std::vector<int64_t> ap((size_t)B + 1, 0), rp((size_t)B + 1, 0);
  for (int64_t v = 0; v < V; ++v) {
    ++ap[(size_t)batch[v] + 1];
    rp[(size_t)batch[v] + 1] += deg[(size_t)v];
  }
  for (int64_t m = 0; m < B; ++m) {
    ap[(size_t)m + 1] += ap[(size_t)m];
    rp[(size_t)m + 1] += rp[(size_t)m];
  }
  // greedy packing, restarted every 1024 molecules (layout.cu: kTileChunk; oracle/layout_np.py: TILE_CHUNK)
  const int64_t kRows = 128, kAtoms = 128, kChunk = 1024;
  int64_t t_mol = 0, n_tiles = 0, max_rows = 0, max_atoms = 0;
  for (int64_t m = 0; m < B; ++m) {
    if (m > t_mol && (m % kChunk == 0 || rp[(size_t)m + 1] - rp[(size_t)t_mol] > kRows ||
                      ap[(size_t)m + 1] - ap[(size_t)t_mol] > kAtoms)) {
      ++n_tiles;
      if (rp[(size_t)m] - rp[(size_t)t_mol] > max_rows) max_rows = rp[(size_t)m] - rp[(size_t)t_mol];
      if (ap[(size_t)m] - ap[(size_t)t_mol] > max_atoms) max_atoms = ap[(size_t)m] - ap[(size_t)t_mol];
      t_mol = m;
    }
  }
  ++n_tiles;
  if (rp[(size_t)B] - rp[(size_t)t_mol] > max_rows) max_rows = rp[(size_t)B] - rp[(size_t)t_mol];
  if (ap[(size_t)B] - ap[(size_t)t_mol] > max_atoms) max_atoms = ap[(size_t)B] - ap[(size_t)t_mol];
  meta[DMPNN_META_N_TILES] = (int32_t)n_tiles;
  meta[DMPNN_META_MAX_TILE_ROWS] = (int32_t)max_rows;
  meta[DMPNN_META_MAX_TILE_ATOMS] = (int32_t)max_atoms;
  return 0;
}

// Tile packing words from per-molecule sizes: the O(B) form of dmpnn_batch_meta_host for batches assembled from a
// packed dataset whose molecules were validated when the dataset was built (flags are then known to be all set).
static void tiles_meta_from_sizes(int64_t B, const int64_t* n_atoms, const int64_t* n_edges, const int32_t* max_indeg,
                                  int32_t* meta) {
  for (int i = 0; i < DMPNN_META_WORDS; ++i) meta[i] = 0;
  meta[DMPNN_META_FLAGS] = DMPNN_FLAG_INDEX_IN_RANGE | DMPNN_FLAG_REV_INVOLUTION | DMPNN_FLAG_BATCH_SORTED;
  if (B == 0) return;
  const int64_t kRows = 128, kAtoms = 128, kChunk = 1024;
  int64_t rows = 0, atoms = 0, n_tiles = 0, max_rows = 0, max_atoms = 0, t_mol = 0;
  int32_t mi = 0;
  for (int64_t m = 0; m < B; ++m) {
    if (m > t_mol && (m % kChunk == 0 || rows + n_edges[m] > kRows || atoms + n_atoms[m] > kAtoms)) {
      ++n_tiles;
      if (rows > max_rows) max_rows = rows;
      if (atoms > max_atoms) max_atoms = atoms;
      rows = 0;
      atoms = 0;
      t_mol = m;
    }
    rows += n_edges[m];
    atoms += n_atoms[m];
    if (max_indeg[m] > mi) mi = max_indeg[m];
  }
  ++n_tiles;
  if (rows > max_rows) max_rows = rows;
  if (atoms > max_atoms) max_atoms = atoms;
  meta[DMPNN_META_N_TILES] = (int32_t)n_tiles;
  meta[DMPNN_META_MAX_INDEG] = mi;
  meta[DMPNN_META_MAX_TILE_ROWS] = (int32_t)max_rows;
  meta[DMPNN_META_MAX_TILE_ATOMS] = (int32_t)max_atoms;
}

int dmpnn_dataset_batch_meta_host(int64_t n_sel, const int64_t* ids, int64_t n_total, const int64_t* atom_ptr,
                                  const int64_t* edge_ptr, const int32_t* mol_max_indeg, int64_t* out_atom_ptr,
                                  int64_t* out_edge_ptr, int32_t* meta) {
  DMPNN_CHECK_ARG(n_sel >= 0 && n_total >= 0 && (n_sel == 0 || ids) && atom_ptr && edge_ptr && mol_max_indeg &&
                      out_atom_ptr && out_edge_ptr && meta, "dataset_batch_meta_host: bad args");
  std::vector<int64_t> na((size_t)n_sel), ne((size_t)n_sel);
  std::vector<int32_t> mi((size_t)n_sel);
  out_atom_ptr[0] = 0;
  out_edge_ptr[0] = 0;
  for (int64_t m = 0; m < n_sel; ++m) {
    const int64_t id = ids[m];
    DMPNN_CHECK_ARG(id >= 0 && id < n_total, "dataset_batch_meta_host: molecule id %lld out of range", (long long)id);
    na[(size_t)m] = atom_ptr[id + 1] - atom_ptr[id];
    ne[(size_t)m] = edge_ptr[id + 1] - edge_ptr[id];
    mi[(size_t)m] = mol_max_indeg[id];
    out_atom_ptr[m + 1] = out_atom_ptr[m] + na[(size_t)m];
    out_edge_ptr[m + 1] = out_edge_ptr[m] + ne[(size_t)m];
  }
  DMPNN_CHECK_ARG(out_atom_ptr[n_sel] < (1LL << 31) && out_edge_ptr[n_sel] < (1LL << 31),
                  "dataset_batch_meta_host: batch too large for int32 rows");
  tiles_meta_from_sizes(n_sel, na.data(), ne.data(), mi.data(), meta);
  return 0;
}

// Host-side batch assembly from a packed dataset: replaces `[dataset[i] for i in ids]` + collate_batch
// (chemprop/data/datasets.py:222-244, collate.py:37-62) by contiguous copies of each selected molecule's rows.
// Molecules are independent, so the selection is split over `n_threads` host threads (<= 0: one per 2048 molecules, at
// most 8 and at most the hardware concurrency).
struct GatherHostArgs {
  const int64_t *ids, *out_atom_ptr, *out_edge_ptr, *atom_ptr, *edge_ptr;
  const float *V_all, *E_all;
  const int32_t *ei_local, *rev_local;
  int64_t E_all_total, d_v, d_e, Et;
  float *V_out, *E_out;
  int64_t *ei_out, *rev_out, *batch_out;
  uint16_t *Vb_out, *Eb_out;
  int32_t *ei32_out, *rev32_out, *batch32_out;
};

static void gather_host_range(const GatherHostArgs& a, int64_t lo, int64_t hi) {
  const bool compact = a.Vb_out || a.Eb_out || a.ei32_out || a.rev32_out || a.batch32_out;
  const int64_t d_v = a.d_v, d_e = a.d_e, Et = a.Et;
  for (int64_t m = lo; m < hi; ++m) {
    const int64_t id = a.ids[m];
    const int64_t sa = a.atom_ptr[id], se = a.edge_ptr[id];
    const int64_t na = a.atom_ptr[id + 1] - sa, ne = a.edge_ptr[id + 1] - se;
    const int64_t oa = a.out_atom_ptr[m], oe = a.out_edge_ptr[m];
    if (a.V_out && na > 0 && d_v > 0) memcpy(a.V_out + oa * d_v, a.V_all + sa * d_v, sizeof(float) * na * d_v);
    if (a.E_out && ne > 0 && d_e > 0) memcpy(a.E_out + oe * d_e, a.E_all + se * d_e, sizeof(float) * ne * d_e);
    const int32_t* s0 = a.ei_local + se;
    const int32_t* s1 = a.ei_local + a.E_all_total + se;
    const int32_t* rv = a.rev_local + se;
    if (a.ei_out)
      for (int64_t j = 0; j < ne; ++j) {
        a.ei_out[oe + j] = (int64_t)s0[j] + oa;            // collate.py:51
        a.ei_out[Et + oe + j] = (int64_t)s1[j] + oa;
        a.rev_out[oe + j] = (int64_t)rv[j] + oe;           // collate.py:52
      }
    if (a.batch_out)
      for (int64_t j = 0; j < na; ++j) a.batch_out[oa + j] = m;   // collate.py:53
    if (compact) {
      const float* v = a.V_all + sa * d_v;
      const float* e = a.E_all + se * d_e;
      for (int64_t j = 0; j < na * d_v; ++j) a.Vb_out[oa * d_v + j] = f32_to_bf16_rne(v[j]);
      for (int64_t j = 0; j < ne * d_e; ++j) a.Eb_out[oe * d_e + j] = f32_to_bf16_rne(e[j]);
      for (int64_t j = 0; j < ne; ++j) {
        a.ei32_out[oe + j] = (int32_t)(s0[j] + oa);
        a.ei32_out[Et + oe + j] = (int32_t)(s1[j] + oa);
        a.rev32_out[oe + j] = (int32_t)(rv[j] + oe);
      }
      for (int64_t j = 0; j < na; ++j) a.batch32_out[oa + j] = (int32_t)m;
    }
  }
}

int dmpnn_dataset_gather_host(int64_t n_sel, const int64_t* ids, const int64_t* out_atom_ptr, const int64_t* out_edge_ptr,
                              const int64_t* atom_ptr, const int64_t* edge_ptr, const float* V_all, const float* E_all,
                              const int32_t* ei_local, const int32_t* rev_local, int64_t E_all_total, int64_t d_v,
                              int64_t d_e, float* V_out, float* E_out, int64_t* ei_out, int64_t* rev_out,
                              int64_t* batch_out, uint16_t* Vb_out, uint16_t* Eb_out, int32_t* ei32_out,
                              int32_t* rev32_out, int32_t* batch32_out, int n_threads) {
  DMPNN_CHECK_ARG(n_sel >= 0 && d_v >= 0 && d_e >= 0 && E_all_total >= 0, "dataset_gather_host: bad sizes");
  if (n_sel == 0) return 0;
  DMPNN_CHECK_ARG(ids && out_atom_ptr && out_edge_ptr && atom_ptr && edge_ptr, "dataset_gather_host: null table");
  const bool compact = Vb_out || Eb_out || ei32_out || rev32_out || batch32_out;
  DMPNN_CHECK_ARG(!compact || (Vb_out && Eb_out && ei32_out && rev32_out && batch32_out),
                  "dataset_gather_host: the compact copy needs all five outputs");
  DMPNN_CHECK_ARG(!ei_out == !rev_out, "dataset_gather_host: edge_index and rev_edge_index go together");
  GatherHostArgs a{ids, out_atom_ptr, out_edge_ptr, atom_ptr, edge_ptr, V_all, E_all, ei_local, rev_local, E_all_total,
                   d_v, d_e, out_edge_ptr[n_sel], V_out, E_out, ei_out, rev_out, batch_out, Vb_out, Eb_out, ei32_out,
                   rev32_out, batch32_out};
  int T = n_threads;
  if (T <= 0) {
    const unsigned hw = std::thread::hardware_concurrency();
    T = (int)((n_sel + 2047) / 2048);
    if (T > 8) T = 8;
    if (hw > 0 && T > (int)hw) T = (int)hw;
  }
  if (T > n_sel) T = (int)n_sel;
  if (T <= 1) {
    gather_host_range(a, 0, n_sel);
    return 0;
  }
  // split by output atoms (not by molecule count) so that threads copy similar byte counts
  std::vector<std::thread> pool;
  std::vector<int64_t> cut((size_t)T + 1, 0);
  cut[(size_t)T] = n_sel;
  const int64_t Vt = out_atom_ptr[n_sel];
  int64_t m = 0;
  for (int t = 1; t < T; ++t) {
    const int64_t target = Vt * t / T;
    while (m < n_sel && out_atom_ptr[m] < target) ++m;
    cut[(size_t)t] = m;
  }
  for (int t = 1; t < T; ++t) pool.emplace_back(gather_host_range, std::cref(a), cut[(size_t)t], cut[(size_t)t + 1]);
  gather_host_range(a, cut[0], cut[1]);
  for (auto& th : pool) th.join();
  return 0;
}

// Order the molecules of a batch so that the engine's greedy molecule-aligned tiles (<= 128 edge rows and <= 128 atoms of
// CONSECUTIVE molecules, dmpnn_layout_build) come out nearly full: best-fit-decreasing bin packing on the edge counts.
// The fused depth step spends the same time on a tile whatever its fill, so fewer, fuller tiles are a direct gain
// (10 k ~25-atom molecules: 4856 tiles at 0.81 fill in arrival order -> 4186 tiles at 0.94).  A heuristic on the ORDER
// only: tiles are always re-derived exactly from whatever order the batch ends up in, so correctness never depends on
// it.  order_out receives a permutation of [0, n): bins in creation order, members in insertion order.
int dmpnn_tile_pack_order(int64_t n, const int64_t* n_atoms, const int64_t* n_edges, int64_t* order_out) {
  DMPNN_CHECK_ARG(n >= 0 && (n == 0 || (n_atoms && n_edges && order_out)), "tile_pack_order: bad args");
  const int64_t kRows = 128, kAtoms = 128;
  std::vector<int64_t> ids((size_t)n);
  for (int64_t i = 0; i < n; ++i) {
    DMPNN_CHECK_ARG(n_atoms[i] >= 0 && n_edges[i] >= 0, "tile_pack_order: negative molecule size");
    ids[(size_t)i] = i;
  }
  std::stable_sort(ids.begin(), ids.end(), [&](int64_t a, int64_t b) { return n_edges[a] > n_edges[b]; });
  struct Bin { int64_t rows, atoms, head, tail; };
  std::vector<Bin> bins;
  std::vector<int64_t> next((size_t)n, -1);
  std::vector<std::vector<int64_t>> by_rem((size_t)kRows + 1);   // open bins by remaining row capacity
  for (int64_t k = 0; k < n; ++k) {
    const int64_t i = ids[(size_t)k], e = n_edges[i], a = n_atoms[i];
    int64_t hit = -1;
    if (e <= kRows && a <= kAtoms) {
      for (int64_t r = e; r <= kRows && hit < 0; ++r) {           // best fit: the fullest bin that still takes it
        auto& st = by_rem[(size_t)r];
        for (size_t j = st.size(); j-- > 0;) {
          if (bins[(size_t)st[j]].atoms + a <= kAtoms) {
            hit = st[j];
            st.erase(st.begin() + (std::ptrdiff_t)j);
            break;
          }
        }
      }
    }
    if (hit < 0) {
      bins.push_back(Bin{e, a, i, i});
      hit = (int64_t)bins.size() - 1;
    } else {
      Bin& b = bins[(size_t)hit];
      next[(size_t)b.tail] = i;
      b.tail = i;
      b.rows += e;
      b.atoms += a;
    }
    const Bin& b = bins[(size_t)hit];
    if (b.rows <= kRows && b.atoms < kAtoms) by_rem[(size_t)(kRows - b.rows)].push_back(hit);   // still open
  }
  int64_t o = 0;
  for (const Bin& b : bins)
    for (int64_t i = b.head; i >= 0; i = next[(size_t)i]) order_out[o++] = i;
  DMPNN_CHECK_ARG(o == n, "tile_pack_order: internal error");
  // safety net: the engine packs CONSECUTIVE molecules greedily (restarting every 1024); keep the arrival order
  // whenever the bin-packed one would not give fewer tiles under that exact rule
  auto greedy_tiles = [&](bool packed) {
    const int64_t kChunk = 1024;
    int64_t rows = 0, atoms = 0, tiles = n > 0 ? 1 : 0, t_mol = 0;
    for (int64_t m = 0; m < n; ++m) {
      const int64_t i = packed ? order_out[m] : m;
      if (m > t_mol && (m % kChunk == 0 || rows + n_edges[i] > kRows || atoms + n_atoms[i] > kAtoms)) {
        ++tiles;
        rows = 0;
        atoms = 0;
        t_mol = m;
      }
      rows += n_edges[i];
      atoms += n_atoms[i];
    }
    return tiles;
  };
  if (greedy_tiles(true) >= greedy_tiles(false))
    for (int64_t i = 0; i < n; ++i) order_out[i] = i;
  return 0;
}

}  // extern "C"
