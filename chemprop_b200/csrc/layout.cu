// Device layout build: reference BatchMolGraph index tensors -> dst-sorted CSR + tile table.
// Replaces the per-call index materialisation of chemprop/nn/message_passing/mixins.py:12-15
// and chemprop/nn/agg.py:74-75 with a one-off integer preprocessing pass per batch.
// All outputs are deterministic (stable sort by destination) and bit-exact w.r.t.
// oracle/layout_np.py.
#include "common.cuh"

namespace dmpnn {

constexpr int kTileRows = 128;
constexpr int kTileAtoms = 128;

struct LayoutWs {
  int32_t* deg;     // V+1
  int32_t* cursor;  // V
  int32_t* tmp;     // E
  int32_t* bsum;    // nblk_scan + 1
  int32_t* viol;    // 4 words: [0]=violation bits, [1]=max indeg
  int32_t* seg_tiles;  // n_chunks * kTileChunkWs
  int32_t* seg_info;   // n_chunks * 4
};
constexpr int kTileChunkWs = 1024;

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t carve(LayoutWs* ws, void* base, int64_t V, int64_t E, int64_t B) {
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) { char* p = b ? b + off : nullptr; off += align_up(bytes, 256); return p; };
  int32_t* deg = (int32_t*)take(sizeof(int32_t) * (V + 1));
  int32_t* cursor = (int32_t*)take(sizeof(int32_t) * (V + 1));
  int32_t* tmp = (int32_t*)take(sizeof(int32_t) * (E + 1));
  int64_t nblk = (V + 1 + 2047) / 2048;
  int32_t* bsum = (int32_t*)take(sizeof(int32_t) * (nblk + 1));
  int32_t* viol = (int32_t*)take(sizeof(int32_t) * 4);
  int64_t n_chunks = (B + kTileChunkWs - 1) / kTileChunkWs;
  if (n_chunks < 1) n_chunks = 1;
  int32_t* seg_tiles = (int32_t*)take(sizeof(int32_t) * n_chunks * kTileChunkWs);
  int32_t* seg_info = (int32_t*)take(sizeof(int32_t) * n_chunks * 4);
  if (ws) { ws->deg = deg; ws->cursor = cursor; ws->tmp = tmp; ws->bsum = bsum; ws->viol = viol;
            ws->seg_tiles = seg_tiles; ws->seg_info = seg_info; }
  return off;
}

// bits in viol[0]
enum { V_RANGE = 1, V_INVOL = 2, V_BATCH = 4 };

__global__ void k_count(const int64_t* __restrict__ ei, const int64_t* __restrict__ rev,
                        const int64_t* __restrict__ batch, int64_t V, int64_t E, int64_t B,
                        int32_t* deg, int32_t* viol) {
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  int64_t s = ei[e], d = ei[E + e], r = rev[e];
  int bad = 0;
  if (s < 0 || s >= V || d < 0 || d >= V || r < 0 || r >= E) {
    bad |= V_RANGE;
  } else {
    int64_t rs = ei[r], rd = ei[E + r], rr = rev[r];
    if (rr != e || rs != d || rd != s) bad |= V_INVOL;
    int64_t bs = batch[s], bd = batch[d];
    if (bs != bd) bad |= V_BATCH;
    atomicAdd(&deg[d], 1);
  }
  if (bad) atomicOr(&viol[0], bad);
}

__global__ void k_batch_check(const int64_t* __restrict__ batch, int64_t V, int64_t B, int32_t* viol) {
  int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (v >= V) return;
  int64_t b = batch[v];
  int bad = 0;
  if (b < 0 || b >= B) bad |= V_RANGE;
  if (v + 1 < V && batch[v + 1] < b) bad |= V_BATCH;
  if (bad) atomicOr(&viol[0], bad);
}

// ---- exclusive scan (n elements, int32), 2048 per block ------------------------------
__global__ void k_scan_block(const int32_t* __restrict__ in, int32_t* __restrict__ out,
                             int32_t* __restrict__ bsum, int64_t n) {
  __shared__ int32_t warp_tot[8];
  const int tid = threadIdx.x;  // 256 threads x 8 items
  const int64_t base = blockIdx.x * 2048LL + tid * 8;
  int32_t v[8];
  int32_t s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[i] = (base + i < n) ? in[base + i] : 0;
    s += v[i];
  }
  // warp inclusive scan of s
  int32_t inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if ((tid & 31) >= o) inc += t;
  }
  if ((tid & 31) == 31) warp_tot[tid >> 5] = inc;
  __syncthreads();
  int32_t woff = 0;
  for (int w = 0; w < (tid >> 5); ++w) woff += warp_tot[w];
  int32_t run = woff + inc - s;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (base + i < n) out[base + i] = run;
    run += v[i];
  }
  if (tid == 255) bsum[blockIdx.x] = woff + inc;
}

__global__ void k_scan_bsums(int32_t* bsum, int64_t nblk) {
  // single block: sequential chunks of 1024 with a running carry
  __shared__ int32_t sh[1024];
  __shared__ int32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int64_t base = 0; base < nblk; base += 1024) {
    int64_t i = base + threadIdx.x;
    int32_t x = (i < nblk) ? bsum[i] : 0;
    sh[threadIdx.x] = x;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      int32_t t = (threadIdx.x >= o) ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    int32_t c = carry;
    if (i < nblk) bsum[i] = c + sh[threadIdx.x] - x;
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + sh[1023];
    __syncthreads();
  }
}

__global__ void k_scan_add(int32_t* out, const int32_t* __restrict__ bsum, int64_t n) {
  int64_t i = blockIdx.x * 2048LL + threadIdx.x;
  int32_t add = bsum[blockIdx.x];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int64_t j = i + k * 256;
    if (j < n) out[j] += add;
  }
}

__global__ void k_place(const int64_t* __restrict__ ei, int64_t V, int64_t E,
                        const int32_t* __restrict__ rowptr, int32_t* cursor, int32_t* tmp) {
  int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  int64_t d = ei[E + e];
  if (d < 0 || d >= V) return;
  int32_t p = atomicAdd(&cursor[d], 1);
  tmp[rowptr[d] + p] = (int32_t)e;
}

// one thread per atom: sort the bucket by edge id (stable order), emit per-row arrays
__global__ void k_bucket_sort(const int64_t* __restrict__ ei, int64_t V, int64_t E,
                              const int32_t* __restrict__ rowptr, int32_t* tmp,
                              int32_t* perm, int32_t* inv_perm, int32_t* src_row, int32_t* dst_row,
                              int32_t* viol) {
  int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (v >= V) return;
  int32_t a = rowptr[v], b = rowptr[v + 1];
  for (int32_t i = a + 1; i < b; ++i) {  // insertion sort (in-degree is tiny for molecules)
    int32_t x = tmp[i];
    int32_t j = i - 1;
    while (j >= a && tmp[j] > x) { tmp[j + 1] = tmp[j]; --j; }
    tmp[j + 1] = x;
  }
  for (int32_t i = a; i < b; ++i) {
    int32_t e = tmp[i];
    perm[i] = e;
    inv_perm[e] = i;
    dst_row[i] = (int32_t)v;
    src_row[i] = (int32_t)ei[e];
  }
  if (b - a > 0) atomicMax(&viol[1], b - a);
}

__global__ void k_rev_rows(const int64_t* __restrict__ rev, int64_t E, const int32_t* __restrict__ perm,
                           const int32_t* __restrict__ inv_perm, int32_t* rev_row) {
  int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= E) return;
  int64_t q = rev[perm[r]];
  rev_row[r] = (q >= 0 && q < E) ? inv_perm[q] : 0;
}

// mol_atom_ptr[b] = first atom v with batch[v] >= b  (batch non-decreasing)
__global__ void k_mol_ptr(const int64_t* __restrict__ batch, int64_t V, int64_t B,
                          const int32_t* __restrict__ rowptr, int32_t* mol_atom_ptr, int32_t* mol_row_ptr) {
  int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;  // v in [0, V]
  if (v > V) return;
  int64_t lo = (v == 0) ? 0 : batch[v - 1] + 1;
  int64_t hi = (v == V) ? B : batch[v];
  if (lo < 0) lo = 0;
  if (hi > B) hi = B;
  if (v == V) hi = B;  // ptr[B] included below
  for (int64_t b = lo; b <= hi && b <= B; ++b) {
    if (v < V && b > batch[v]) break;
    mol_atom_ptr[b] = (int32_t)v;
    if (mol_row_ptr) mol_row_ptr[b] = rowptr[v];
  }
}

// Greedy molecule-aligned packing into tiles of <= kTileRows rows and <= kTileAtoms atoms, restarted at
// every kTileChunk-th molecule so that chunks are independent: one block per chunk walks its molecule
// offsets (staged in shared memory) and writes its tile starts to a private segment; k_tiles_gather
// then concatenates the segments in order.  (oracle/layout_np.py restates exactly this rule.)
constexpr int kTileChunk = 1024;

__global__ void k_tiles_chunk(const int32_t* __restrict__ mol_atom_ptr, const int32_t* __restrict__ mol_row_ptr,
                              int64_t B, int row_limit, int atom_limit, int32_t* __restrict__ seg_tiles /*[n_chunks][kTileChunk]*/,
                              int32_t* __restrict__ seg_info /*[n_chunks][4]: count, max_rows, max_atoms*/) {
  __shared__ int32_t s_at[kTileChunk + 1];
  __shared__ int32_t s_rw[kTileChunk + 1];
  const int64_t base = (int64_t)blockIdx.x * kTileChunk;
  const int n = (int)((B - base < kTileChunk) ? (B - base) : kTileChunk);
  for (int i = threadIdx.x; i <= n; i += blockDim.x) {
    s_at[i] = mol_atom_ptr[base + i];
    s_rw[i] = mol_row_ptr[base + i];
  }
  __syncthreads();
  // nxt[t0] = first molecule that no longer fits a tile opened at t0 (the greedy rule's closing index): both limits
  // are monotone in the closing index, so each thread finds it by bisection; thread 0 then only follows the chain.
  __shared__ int32_t s_nxt[kTileChunk];
  for (int t0 = threadIdx.x; t0 < n; t0 += blockDim.x) {
    const int32_t rlim = s_rw[t0] + row_limit, alim = s_at[t0] + atom_limit;
    int lo = t0 + 1, hi = n;               // smallest i in [t0+1, n) with s_rw[i+1] > rlim or s_at[i+1] > alim, else n
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_rw[mid + 1] > rlim || s_at[mid + 1] > alim) hi = mid; else lo = mid + 1;
    }
    s_nxt[t0] = lo;
  }
  __syncthreads();
  // thread 0 only follows the chain (one dependent shared-memory load per tile, ~420 hops per chunk); the per-tile row /
  // atom counts and their maxima are taken by the whole block afterwards (they were part of the serial walk: 28 us per
  // step at the bench size, profiles/r2_glue_ncu.md)
  __shared__ int32_t s_start[kTileChunk + 1];
  __shared__ int s_cnt;
  if (threadIdx.x == 0) {
    int cnt = 0;
    for (int t0 = 0; t0 < n; t0 = s_nxt[t0]) s_start[cnt++] = t0;
    s_start[cnt] = n;
    s_cnt = cnt;
  }
  __syncthreads();
  const int cnt = s_cnt;
  int32_t* out = seg_tiles + (int64_t)blockIdx.x * kTileChunk;
  int max_rows = 0, max_atoms = 0;
  for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
    const int t0 = s_start[k], i = s_start[k + 1];
    out[k] = (int32_t)(base + t0);
    max_rows = max(max_rows, s_rw[i] - s_rw[t0]);
    max_atoms = max(max_atoms, s_at[i] - s_at[t0]);
  }
  __shared__ int s_mr[8], s_ma[8];
  for (int o = 16; o > 0; o >>= 1) {
    max_rows = max(max_rows, __shfl_down_sync(0xffffffffu, max_rows, o));
    max_atoms = max(max_atoms, __shfl_down_sync(0xffffffffu, max_atoms, o));
  }
  if ((threadIdx.x & 31) == 0) { s_mr[threadIdx.x >> 5] = max_rows; s_ma[threadIdx.x >> 5] = max_atoms; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { max_rows = max(max_rows, s_mr[w]); max_atoms = max(max_atoms, s_ma[w]); }
    seg_info[blockIdx.x * 4 + 0] = cnt;
    seg_info[blockIdx.x * 4 + 1] = max_rows;
    seg_info[blockIdx.x * 4 + 2] = max_atoms;
  }
}

__global__ void k_tiles_gather(const int32_t* __restrict__ seg_tiles, const int32_t* __restrict__ seg_info, int n_chunks,
                               const int32_t* __restrict__ mol_atom_ptr, const int32_t* __restrict__ mol_row_ptr, int64_t B,
                               int32_t* tile_mol_ptr, int32_t* tile_row_ptr, int32_t* tile_atom_ptr, int32_t* meta,
                               const int32_t* viol) {
  __shared__ int32_t s_off[1024];
  __shared__ int32_t s_tot, s_mr, s_ma;
  // exclusive prefix of the per-chunk tile counts (n_chunks is small: B / 1024)
  if (threadIdx.x == 0) {
    int run = 0, mr = 0, ma = 0;
    for (int c = 0; c < n_chunks; ++c) {
      if (c < 1024) s_off[c] = run;
      run += seg_info[c * 4];
      mr = max(mr, seg_info[c * 4 + 1]);
      ma = max(ma, seg_info[c * 4 + 2]);
    }
    s_tot = run; s_mr = mr; s_ma = ma;
  }
  __syncthreads();
  for (int c = 0; c < n_chunks; ++c) {
    int off;
    if (c < 1024) off = s_off[c];
    else { off = 0; for (int q = 0; q < c; ++q) off += seg_info[q * 4]; }
    const int cnt = seg_info[c * 4];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const int32_t m = seg_tiles[(int64_t)c * kTileChunk + i];
      tile_mol_ptr[off + i] = m;
      tile_row_ptr[off + i] = mol_row_ptr[m];
      tile_atom_ptr[off + i] = mol_atom_ptr[m];
    }
  }
  if (threadIdx.x == 0) {
    const int n_tiles = s_tot;
    tile_mol_ptr[n_tiles] = (int32_t)B;
    tile_row_ptr[n_tiles] = mol_row_ptr[B];
    tile_atom_ptr[n_tiles] = mol_atom_ptr[B];
    int32_t vb = viol[0];
    int32_t flags = 0;
    if (!(vb & V_RANGE)) flags |= DMPNN_FLAG_INDEX_IN_RANGE;
    if (!(vb & (V_INVOL | V_RANGE))) flags |= DMPNN_FLAG_REV_INVOLUTION;
    if (!(vb & (V_BATCH | V_RANGE))) flags |= DMPNN_FLAG_BATCH_SORTED;
    meta[DMPNN_META_N_TILES] = n_tiles;
    meta[DMPNN_META_FLAGS] = flags;
    meta[DMPNN_META_MAX_INDEG] = viol[1];
    meta[DMPNN_META_MAX_TILE_ROWS] = s_mr;
    meta[DMPNN_META_MAX_TILE_ATOMS] = s_ma;
    meta[5] = 0; meta[6] = 0; meta[7] = 0;
  }
}

// the same packing with caller-given limits, tile starts only (dmpnn_tiles_build: the ATOM tiles of the fused atom step)
__global__ void k_tiles_gather_plain(const int32_t* __restrict__ seg_tiles, const int32_t* __restrict__ seg_info, int n_chunks,
                                     const int32_t* __restrict__ mol_atom_ptr, const int32_t* __restrict__ mol_row_ptr, int64_t B,
                                     int32_t* tile_row_ptr, int32_t* tile_atom_ptr, int32_t* info) {
  __shared__ int32_t s_tot, s_mr, s_ma;
  int off = 0;
  for (int c = 0; c < n_chunks; ++c) {             // n_chunks = B / 1024: a handful
    const int cnt = seg_info[c * 4];
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      const int32_t m = seg_tiles[(int64_t)c * kTileChunk + i];
      tile_row_ptr[off + i] = mol_row_ptr[m];
      tile_atom_ptr[off + i] = mol_atom_ptr[m];
    }
    off += cnt;
  }
  if (threadIdx.x == 0) {
    int mr = 0, ma = 0;
    for (int c = 0; c < n_chunks; ++c) { mr = max(mr, seg_info[c * 4 + 1]); ma = max(ma, seg_info[c * 4 + 2]); }
    tile_row_ptr[off] = mol_row_ptr[B];
    tile_atom_ptr[off] = mol_atom_ptr[B];
    info[0] = off; info[1] = mr; info[2] = ma; info[3] = 0;
  }
  (void)s_tot; (void)s_mr; (void)s_ma;
}

}  // namespace dmpnn

using namespace dmpnn;

extern "C" int dmpnn_tiles_workspace_bytes(int64_t B, size_t* bytes) {
  DMPNN_CHECK_ARG(B >= 0 && bytes, "tiles_workspace_bytes: bad args");
  const int64_t n_chunks = (B + kTileChunk - 1) / kTileChunk;
  *bytes = (size_t)(n_chunks > 0 ? n_chunks : 1) * (kTileChunk + 4) * sizeof(int32_t);
  return 0;
}

extern "C" int dmpnn_tiles_build(const int32_t* mol_atom_ptr, const int32_t* mol_row_ptr, int64_t B, int row_limit,
                                 int atom_limit, int32_t* tile_row_ptr, int32_t* tile_atom_ptr, int32_t* info,
                                 void* workspace, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(B >= 0 && row_limit > 0 && atom_limit > 0 && mol_atom_ptr && mol_row_ptr && tile_row_ptr && tile_atom_ptr &&
                      info && workspace, "tiles_build: bad args");
  const int n_chunks = (int)((B + kTileChunk - 1) / kTileChunk);
  int32_t* seg_tiles = (int32_t*)workspace;
  int32_t* seg_info = seg_tiles + (size_t)(n_chunks > 0 ? n_chunks : 1) * kTileChunk;
  if (n_chunks > 0) k_tiles_chunk<<<n_chunks, 256, 0, st>>>(mol_atom_ptr, mol_row_ptr, B, row_limit, atom_limit, seg_tiles, seg_info);
  k_tiles_gather_plain<<<1, 1024, 0, st>>>(seg_tiles, seg_info, n_chunks, mol_atom_ptr, mol_row_ptr, B, tile_row_ptr, tile_atom_ptr,
                                           info);
  DMPNN_CHECK_LAUNCH("tiles_build", 2);
  return 0;
}

extern "C" int dmpnn_layout_workspace_bytes(int64_t V, int64_t E, int64_t B, size_t* bytes) {
  DMPNN_CHECK_ARG(V >= 0 && E >= 0 && B >= 0 && bytes, "layout_workspace_bytes: bad args");
  *bytes = carve(nullptr, nullptr, V, E, B);
  return 0;
}

extern "C" int dmpnn_layout_build(const int64_t* edge_index, const int64_t* rev_edge_index,
                                  const int64_t* batch, int64_t V, int64_t E, int64_t B,
                                  int32_t* perm, int32_t* inv_perm, int32_t* rowptr, int32_t* src_row,
                                  int32_t* dst_row, int32_t* rev_row, int32_t* mol_atom_ptr,
                                  int32_t* mol_row_ptr, int32_t* tile_mol_ptr, int32_t* tile_row_ptr,
                                  int32_t* tile_atom_ptr, int32_t* meta, void* workspace, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(V >= 0 && E >= 0 && B >= 0, "layout_build: negative size");
  DMPNN_CHECK_ARG(V < (1LL << 31) - 4096 && E < (1LL << 31) - 4096, "layout_build: V/E exceed int32");
  DMPNN_CHECK_ARG(workspace && rowptr && mol_atom_ptr && mol_row_ptr && tile_mol_ptr && tile_row_ptr &&
                      tile_atom_ptr && meta,
                  "layout_build: null pointer");
  LayoutWs ws;
  size_t total = carve(&ws, workspace, V, E, B);
  cudaMemsetAsync(workspace, 0, total, st);
  const int T = 256;
  if (E > 0) {
    k_count<<<ceil_div_i64(E, T), T, 0, st>>>(edge_index, rev_edge_index, batch, V, E, B, ws.deg, ws.viol);
  }
  if (V > 0) k_batch_check<<<ceil_div_i64(V, T), T, 0, st>>>(batch, V, B, ws.viol);
  // exclusive scan of deg[0..V] -> rowptr[0..V]
  int64_t n = V + 1;
  int nblk = ceil_div_i64(n, 2048);
  k_scan_block<<<nblk, 256, 0, st>>>(ws.deg, rowptr, ws.bsum, n);
  k_scan_bsums<<<1, 1024, 0, st>>>(ws.bsum, nblk);
  k_scan_add<<<nblk, 256, 0, st>>>(rowptr, ws.bsum, n);
  if (E > 0) k_place<<<ceil_div_i64(E, T), T, 0, st>>>(edge_index, V, E, rowptr, ws.cursor, ws.tmp);
  if (V > 0)
    k_bucket_sort<<<ceil_div_i64(V, T), T, 0, st>>>(edge_index, V, E, rowptr, ws.tmp, perm, inv_perm,
                                                    src_row, dst_row, ws.viol);
  if (E > 0) k_rev_rows<<<ceil_div_i64(E, T), T, 0, st>>>(rev_edge_index, E, perm, inv_perm, rev_row);
  k_mol_ptr<<<ceil_div_i64(V + 1, T), T, 0, st>>>(batch, V, B, rowptr, mol_atom_ptr, mol_row_ptr);
  const int n_chunks = (int)((B + kTileChunk - 1) / kTileChunk);
  if (n_chunks > 0) k_tiles_chunk<<<n_chunks, 256, 0, st>>>(mol_atom_ptr, mol_row_ptr, B, kTileRows, kTileAtoms, ws.seg_tiles, ws.seg_info);
  k_tiles_gather<<<1, 1024, 0, st>>>(ws.seg_tiles, ws.seg_info, n_chunks, mol_atom_ptr, mol_row_ptr, B, tile_mol_ptr,
                                     tile_row_ptr, tile_atom_ptr, meta, ws.viol);
  DMPNN_CHECK_LAUNCH("layout_build", 11);
  return 0;
}

// Work table of the fused depth step for batches holding molecules of more than 128 directed edges or more than 128 atoms:
// every tile of the layout with <= 128 rows and <= 128 atoms becomes one work item (flag 0), every larger tile -- one
// oversized molecule -- is cut into ceil(rows / 128) windows of <= 128 consecutive rows (flag 1: siblings / reverse edges
// may lie in another window, the kernel gathers them from global memory).  A tile of <= 128 rows but more than 128 atoms
// (many fragments, e.g. a short chain and isolated atoms) is one window with flag 1: the kernel's staged row-pointer slice
// holds the row pointers of at most 128 atoms, the global gathers need none.  One block; tiles are scanned in chunks of 1024 (fixed order).
__global__ void __launch_bounds__(1024)
k_work_table(const int32_t* __restrict__ tile_row_ptr, const int32_t* __restrict__ tile_atom_ptr, int n_tiles,
             int32_t* __restrict__ work_row_ptr, int32_t* __restrict__ work_atom_ptr, int8_t* __restrict__ work_flag,
             int32_t* __restrict__ n_work) {
  __shared__ int s_warp[32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int t0 = 0; t0 < n_tiles; t0 += 1024) {
    const int t = t0 + tid;
    int r0 = 0, nr = 0, cnt = 0;
    bool far = false;
    if (t < n_tiles) {
      r0 = tile_row_ptr[t];
      nr = tile_row_ptr[t + 1] - r0;
      cnt = nr > 128 ? (nr + 127) >> 7 : 1;
      far = cnt > 1 || tile_atom_ptr[t + 1] - tile_atom_ptr[t] > 128;
    }
    int incl = cnt;                                   // inclusive scan inside the warp
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_warp[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += v;
      }
      s_warp[lane] = w;                               // inclusive totals of the warps
    }
    __syncthreads();
    const int base = s_base + (warp > 0 ? s_warp[warp - 1] : 0) + incl - cnt;
    if (t < n_tiles) {
      const int a0 = tile_atom_ptr[t];
      for (int k = 0; k < cnt; ++k) {
        work_row_ptr[base + k] = r0 + 128 * k;
        work_atom_ptr[base + k] = a0;
        work_flag[base + k] = far ? 1 : 0;
      }
    }
    __syncthreads();
    if (tid == 0) s_base += s_warp[31];
    __syncthreads();
  }
  if (tid == 0) {
    const int n = s_base;
    work_row_ptr[n] = n_tiles > 0 ? tile_row_ptr[n_tiles] : 0;
    work_atom_ptr[n] = n_tiles > 0 ? tile_atom_ptr[n_tiles] : 0;
    n_work[0] = n;
  }
}

extern "C" int dmpnn_work_table_build(const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles,
                                      int32_t* work_row_ptr, int32_t* work_atom_ptr, int8_t* work_flag, int32_t* n_work,
                                      void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(tile_row_ptr && tile_atom_ptr && work_row_ptr && work_atom_ptr && work_flag && n_work && n_tiles >= 0,
                  "work_table_build: bad args");
  k_work_table<<<1, 1024, 0, st>>>(tile_row_ptr, tile_atom_ptr, (int)n_tiles, work_row_ptr, work_atom_ptr, work_flag, n_work);
  DMPNN_CHECK_LAUNCH("work_table_build", 1);
  return 0;
}

extern "C" int dmpnn_sorted_index_to_ptr(const int64_t* index, int64_t n, int64_t n_seg, int32_t* ptr,
                                         int32_t* status, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(n >= 0 && n_seg >= 0 && ptr && status, "sorted_index_to_ptr: bad args");
  DMPNN_CHECK_ARG(n < (1LL << 31) - 4096, "sorted_index_to_ptr: n exceeds int32");
  cudaMemsetAsync(status, 0, sizeof(int32_t), st);
  const int T = 256;
  if (n > 0) k_batch_check<<<ceil_div_i64(n, T), T, 0, st>>>(index, n, n_seg, status);
  k_mol_ptr<<<ceil_div_i64(n + 1, T), T, 0, st>>>(index, n, n_seg, nullptr, ptr, nullptr);
  DMPNN_CHECK_LAUNCH("sorted_index_to_ptr", 2);
  return 0;
}
