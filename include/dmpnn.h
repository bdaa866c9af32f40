/*
 * dmpnn.h -- C ABI of libdmpnn_sm90.so, the H100 (sm_90a) D-MPNN message-passing engine.
 *
 * The reference (chemprop v2.3.1) has no FFI on this path: the hot path is ~150 lines of
 * Python dispatching stock ATen ops.  This header is therefore the boundary a maintainer
 * would bind (ctypes) from the reference's module layer; each entry point names the
 * reference code (file:line, relative to the chemprop repo root) it replaces.
 *
 * Conventions
 *  - Plain C symbols; raw device pointers; int64_t sizes; `stream` is a cudaStream_t passed
 *    as void* (torch.cuda.current_stream().cuda_stream).  No torch types.
 *  - The library never allocates, frees or synchronises; all buffers (outputs, saved
 *    activations, workspaces) are owned by the caller.  Launches are asynchronous on `stream`.
 *  - Every function returns 0 on success, <0 on error; dmpnn_last_error() gives the
 *    thread-local message.
 *  - "Hidden" matrices (edge / atom hidden states) are row-major with a row stride `ld`
 *    given in ELEMENTS; their element type is `dmpnn_dtype_t` (f32 or bf16).  Inputs V, E and
 *    all weights / weight gradients are f32.
 *  - Internal edge order: the engine keeps edge hidden states sorted by destination atom
 *    (stable), so the in-edges of atom v are the contiguous rows [rowptr[v], rowptr[v+1]).
 *    `perm[row]` is the caller's edge id of an internal row; outputs of the path are atom- or
 *    molecule-level, so this order never leaks out.
 */
#ifndef DMPNN_H_
#define DMPNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMPNN_VERSION 100 /* 0.1.0 */

typedef enum { DMPNN_F32 = 0, DMPNN_BF16 = 1 } dmpnn_dtype_t;

/* Activations of chemprop/nn/utils.py:11-55 that the engine fuses (PReLU / arbitrary modules
 * are handled by the Python host as an unfused composition). */
typedef enum {
  DMPNN_ACT_NONE = 0,
  DMPNN_ACT_RELU = 1,
  DMPNN_ACT_LEAKYRELU = 2, /* slope = act_param (reference: 0.1) */
  DMPNN_ACT_TANH = 3,
  DMPNN_ACT_ELU = 4 /* alpha = act_param (reference: 1.0) */
} dmpnn_act_t;

/* segment scaling: none; divide by the constant `scale` (NormAggregation, agg.py:112-113);
 * divide by the segment's row count (MeanAggregation, agg.py:73-78; empty segment -> 0). */
typedef enum { DMPNN_SCALE_NONE = 0, DMPNN_SCALE_DIV_CONST = 1, DMPNN_SCALE_INV_COUNT = 2 } dmpnn_scale_t;

/* Layout meta words written by dmpnn_layout_build (int32 each). */
enum {
  DMPNN_META_N_TILES = 0,      /* number of molecule-aligned tiles                              */
  DMPNN_META_FLAGS = 1,        /* bit set below                                                 */
  DMPNN_META_MAX_INDEG = 2,    /* max in-degree of any atom                                     */
  DMPNN_META_MAX_TILE_ROWS = 3,/* largest tile (edge rows); >128 => some molecule is oversized  */
  DMPNN_META_MAX_TILE_ATOMS = 4,
  DMPNN_META_WORDS = 8
};
enum {
  DMPNN_FLAG_REV_INVOLUTION = 1, /* rev[rev[e]]==e, src[rev e]==dst[e], dst[rev e]==src[e]      */
  DMPNN_FLAG_BATCH_SORTED = 2,   /* batch non-decreasing and every edge intra-molecule          */
  DMPNN_FLAG_INDEX_IN_RANGE = 4  /* all indices within [0,V) / [0,E) / [0,B)                    */
};

int dmpnn_version(void);
const char* dmpnn_last_error(void);
/* 1 if a CUDA device of compute capability 9.0 (H100) is current, else 0 (never throws). */
int dmpnn_device_ok(void);
/* Number of kernels this library has launched in this process (bench.py's `gpu_launches`). */
long long dmpnn_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Host-side collate.  Replaces BatchMolGraph.__post_init__ (chemprop/data/collate.py:37-62):
 * concatenates per-molecule arrays and offsets edge_index / rev_edge_index; produces the same
 * five public arrays (V, E f32; edge_index 2xE, rev_edge_index E, batch V -- all int64).
 * CPU code (the reference runs this in DataLoader worker processes).
 * `n_atoms[i]`, `n_edges[i]` give molecule sizes; `V_ptrs[i]` etc. point at that molecule's
 * arrays (V: n_atoms x d_v f32; E: n_edges x d_e f32; edge_index: 2 x n_edges int64 row-major;
 * rev: n_edges int64).
 * ------------------------------------------------------------------------------------- */
int dmpnn_collate_host(int64_t n_mols, const int64_t* n_atoms, const int64_t* n_edges,
                       const float* const* V_ptrs, const float* const* E_ptrs,
                       const int64_t* const* edge_index_ptrs, const int64_t* const* rev_ptrs,
                       int64_t d_v, int64_t d_e,
                       float* V_out, float* E_out, int64_t* edge_index_out /*2 x E_tot*/,
                       int64_t* rev_out, int64_t* batch_out);

/* The same batch in the compact transfer format (bf16 features, round-to-nearest-even; int32 indices): what
 * BatchMolGraph(transfer_dtype=bfloat16) copies host -> device instead of the f32 / int64 tensors.  The bf16 tier
 * rounds V / E to bf16 when it assembles its GEMM operands, so its results do not change.  Fails (< 0) when the
 * batch does not fit int32 indices. */
int dmpnn_collate_host_compact(int64_t n_mols, const int64_t* n_atoms, const int64_t* n_edges,
                               const float* const* V_ptrs, const float* const* E_ptrs,
                               const int64_t* const* edge_index_ptrs, const int64_t* const* rev_ptrs,
                               int64_t d_v, int64_t d_e,
                               uint16_t* V_out, uint16_t* E_out, int32_t* edge_index_out /*2 x E_tot*/,
                               int32_t* rev_out, int32_t* batch_out);

/* ---------------------------------------------------------------------------------------
 * Packed dataset (SURVEY.md 8f-1): all molecules of a data set in flat arrays -- V_all (sum V x d_v f32), E_all
 * (sum E x d_e f32), molecule-LOCAL edge_index (2 x sum E, int32) and rev_edge_index (sum E, int32), atom_ptr /
 * edge_ptr (n + 1, int64) -- on the host or resident in HBM.  A batch for the molecule ids `ids` is one gather:
 * replaces `[dataset[i] for i in ids]` + collate_batch (chemprop/data/datasets.py:222-244, collate.py:37-97) and,
 * for the device-resident form, the host -> device copy of the batch.
 *   dmpnn_dataset_batch_meta_host  output offsets of the selected molecules (out_atom_ptr / out_edge_ptr, n_sel + 1
 *                                  each) and the batch's layout meta words in O(n_sel) from per-molecule sizes
 *                                  (`mol_max_indeg`: max in-degree of each molecule; molecules are validated once,
 *                                  when the data set is packed, so all three flags are set).  CPU code.
 *   dmpnn_dataset_gather_host      the five public BatchMolGraph arrays (f32 / int64; any of V_out, E_out, ei_out +
 *                                  rev_out, batch_out may be NULL to skip it) and, when the five compact pointers
 *                                  are given, the bf16 / int32 transfer copy, in one pass, the selection split over host threads.
 *                                  CPU code.
 *   dmpnn_dataset_gather           the same five arrays on the device: one block per selected molecule, contiguous
 *                                  row copies (16 / 8 / 4-byte accesses by feature width), indices offset on the fly.
 *                                  All pointers are device pointers; ids / out_*_ptr are what the host computed with
 *                                  dmpnn_dataset_batch_meta_host and uploaded (24 bytes per molecule).
 * ------------------------------------------------------------------------------------- */
int dmpnn_dataset_batch_meta_host(int64_t n_sel, const int64_t* ids, int64_t n_total, const int64_t* atom_ptr,
                                  const int64_t* edge_ptr, const int32_t* mol_max_indeg, int64_t* out_atom_ptr,
                                  int64_t* out_edge_ptr, int32_t* meta /*DMPNN_META_WORDS*/);
int dmpnn_dataset_gather_host(int64_t n_sel, const int64_t* ids, const int64_t* out_atom_ptr, const int64_t* out_edge_ptr,
                              const int64_t* atom_ptr, const int64_t* edge_ptr, const float* V_all, const float* E_all,
                              const int32_t* ei_local, const int32_t* rev_local, int64_t E_all_total, int64_t d_v,
                              int64_t d_e, float* V_out, float* E_out, int64_t* ei_out /*2 x E_out*/, int64_t* rev_out,
                              int64_t* batch_out, uint16_t* Vb_out, uint16_t* Eb_out, int32_t* ei32_out,
                              int32_t* rev32_out, int32_t* batch32_out, int n_threads /* <= 0: automatic */);
int dmpnn_dataset_gather(const int64_t* ids, const int64_t* out_atom_ptr, const int64_t* out_edge_ptr, int64_t n_sel,
                         const int64_t* atom_ptr, const int64_t* edge_ptr, const float* V_all, const float* E_all,
                         const int32_t* ei_local, const int32_t* rev_local, int64_t E_all_total, int64_t d_v, int64_t d_e,
                         float* V_out, float* E_out, int64_t* ei_out /*2 x E_out_total*/, int64_t* rev_out,
                         int64_t* batch_out, int64_t E_out_total, void* stream);

/* Dropout application (chemprop/nn/message_passing/base.py:139, :182; nn.Dropout): OUT[i] = X[i] * M[i] * scale over a flat
 * contiguous buffer of n elements of type `dtype` (a hidden matrix with its padding columns), M a {0, 1} keep mask of the same
 * element type drawn by the caller's RNG (torch's Philox stream, so `torch.manual_seed` governs it as in the reference),
 * scale = 1 / (1 - p) applied in f32 with one rounding.  In place allowed (OUT == X). */
int dmpnn_scale_mask(const void* X, const void* M, void* OUT, int dtype, int64_t n, float scale, void* stream);

/* Loader-side molecule order for full tiles: a permutation of the batch's molecules (best-fit-decreasing bin packing of
 * their edge counts into the 128-row / 128-atom tiles of dmpnn_layout_build) under which the greedy tile packing of
 * CONSECUTIVE molecules comes out ~0.94 full instead of ~0.81 for ~25-atom molecules in arrival order.  The order of
 * the molecules inside a batch is the loader's to choose (the reference shuffles it every epoch, samplers.py:19-23);
 * tiles are always derived exactly from the final order, so this is a performance heuristic only.  CPU code. */
int dmpnn_tile_pack_order(int64_t n, const int64_t* n_atoms, const int64_t* n_edges, int64_t* order_out /*n*/);

/* Layout meta words of a batch computed on the HOST (same DMPNN_META_* words dmpnn_layout_build writes on the
 * device): validity flags, max in-degree, and the tile count / largest tile of the greedy molecule-aligned packing.
 * A loader calls it next to the collate (the batch's int64 index arrays are in host memory there), so that the
 * training step never reads `meta` back from the GPU: no host <-> device synchronisation inside the step.  The
 * reference has the same kind of per-batch sync in agg.py:75 (`batch.max().int() + 1`).  Bit-exact w.r.t.
 * oracle/layout_np.py; for an invalid batch only DMPNN_META_FLAGS is meaningful.  CPU code. */
int dmpnn_batch_meta_host(const int64_t* edge_index /*2 x E*/, const int64_t* rev_edge_index, const int64_t* batch,
                          int64_t V, int64_t E, int64_t B, int32_t* meta /*DMPNN_META_WORDS*/);

/* ---------------------------------------------------------------------------------------
 * Device layout build.  Consumes the reference's BatchMolGraph index tensors
 * (chemprop/data/collate.py:24-33: edge_index int64 2xE, rev_edge_index int64 E, batch int64 V)
 * and produces the engine's int32 layout: the stable sort of edges by destination atom
 * (perm / inv_perm / rowptr), per-row src / dst / rev (internal row ids), molecule atom/row
 * offsets, and a table of molecule-aligned tiles holding <=128 edge rows and <=128 atoms each
 * (a molecule larger than that gets a tile of its own; see DMPNN_META_MAX_TILE_*).
 * This replaces the index materialisation in chemprop/nn/message_passing/mixins.py:12
 * (`edge_index[1].unsqueeze(1).repeat(1, h)`) and chemprop/nn/agg.py:74-75.
 * Integer outputs are bit-exact w.r.t. oracle/layout_np.py.
 * ------------------------------------------------------------------------------------- */
int dmpnn_layout_workspace_bytes(int64_t V, int64_t E, int64_t B, size_t* bytes);
int dmpnn_layout_build(const int64_t* edge_index, const int64_t* rev_edge_index, const int64_t* batch,
                       int64_t V, int64_t E, int64_t B,
                       int32_t* perm /*E*/, int32_t* inv_perm /*E*/, int32_t* rowptr /*V+1*/,
                       int32_t* src_row /*E*/, int32_t* dst_row /*E*/, int32_t* rev_row /*E*/,
                       int32_t* mol_atom_ptr /*B+1*/, int32_t* mol_row_ptr /*B+1*/,
                       int32_t* tile_mol_ptr /*B+1, first n_tiles+1 valid*/,
                       int32_t* tile_row_ptr /*B+1: first internal row of each tile (+ sentinel)*/,
                       int32_t* tile_atom_ptr /*B+1: first atom of each tile (+ sentinel)*/,
                       int32_t* meta /*DMPNN_META_WORDS*/,
                       void* workspace, void* stream);

/* Segment offsets of a sorted int64 index (the `batch` argument of Aggregation.forward,
 * chemprop/nn/agg.py:39-59): ptr[b] = first i with index[i] >= b, ptr[n_seg] = n.  `status`
 * (1 int32, device) is set non-zero if index is not non-decreasing or leaves [0, n_seg). */
int dmpnn_sorted_index_to_ptr(const int64_t* index, int64_t n, int64_t n_seg, int32_t* ptr,
                              int32_t* status, void* stream);

/* ---------------------------------------------------------------------------------------
 * Generic fused linear:  C[cr(r), 0:N] = act( [X1[i1(r)] || X2[i2(r)]] . W^T + bias + R[r] )
 * for r in [0,R).  W is the nn.Linear weight, f32 row-major N x (K1+K2), row stride ldw.
 * X1 / X2: f32 or hidden dtype (per *_dtype); idx1 / idx2 optional int32 row gathers (NULL =
 * identity); K2 may be 0.  bias (f32, N) and residual R (hidden dtype, ldr) optional (NULL).
 * Columns [N, ldc_pad) of C are zero-filled (ldc_pad <= ldc), keeping row padding clean.
 * Covers: W_i initialise (mixins.py:8-9, :22-23), W_h update (base.py:135-141), W_o finalize
 * (base.py:180-182) and the dX = dY.W GEMMs of their autograd mirror.
 * fp32-accurate SIMT path (no tensor cores): this is the <=1e-5 tier and the fallback.
 * ------------------------------------------------------------------------------------- */
int dmpnn_linear_fwd(const void* X1, int x1_dtype, int64_t ld1, const int32_t* idx1, int64_t K1,
                     const void* X2, int x2_dtype, int64_t ld2, const int32_t* idx2, int64_t K2,
                     const float* W, int64_t ldw, const float* bias,
                     const void* Rres, int r_dtype, int64_t ldr,
                     int act, float act_param,
                     void* C, int c_dtype, int64_t ldc, int64_t ldc_pad,
                     int64_t R, int64_t N, void* stream);

/* Weight gradient: dW[n, 0:K1+K2] (+)= sum_r dY[r,n] * [X1[i1(r)] || X2[i2(r)]][k];
 * optional dbias[n] (+)= sum_r dY[r,n].  Two-pass deterministic reduction through
 * `workspace` (dmpnn_linear_wgrad_workspace_bytes).  accumulate!=0 adds into dW / dbias. */
int dmpnn_linear_wgrad_workspace_bytes(int64_t R, int64_t N, int64_t K, size_t* bytes);
int dmpnn_linear_wgrad(const void* dY, int dy_dtype, int64_t lddy,
                       const void* X1, int x1_dtype, int64_t ld1, const int32_t* idx1, int64_t K1,
                       const void* X2, int x2_dtype, int64_t ld2, const int32_t* idx2, int64_t K2,
                       float* dW, int64_t lddw, float* dbias, int accumulate,
                       int64_t R, int64_t N, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------
 * Segmented row sum:  Y[s, 0:C] = scale(s) * sum_{r in [ptr[s], ptr[s+1])} f(X[idx(r), 0:C]).
 * f = activation `act` applied on load (ACT_NONE = identity).  Covers the final atom
 * scatter-sum (base.py:208-211; segments = atoms over dst-sorted rows), the neighbour sum of
 * the atom-granular AtomMessagePassing (mixins.py:25-30), and Mean/Sum/Norm aggregation
 * (agg.py:73-78, 90-95, 112-113; segments = molecules; divide by count / nothing / norm).
 * Empty segments give zero rows (agg.py:44-45).  Accumulates in f32, deterministic order.
 * ------------------------------------------------------------------------------------- */
int dmpnn_segment_sum(const void* X, int x_dtype, int64_t ldx, const int32_t* idx,
                      const int32_t* ptr, int64_t n_seg, int64_t C,
                      int act, float act_param, int scale_mode, float scale,
                      void* Y, int y_dtype, int64_t ldy, int64_t ldy_pad, void* stream);

/* Row broadcast (autograd mirror of segment_sum with identity f):
 * Y[r, 0:C] = scale(seg(r)) * G[seg_of_row[r], 0:C]; for SCALE_INV_COUNT, `ptr` gives counts.
 * n_seg > 0 (with ptr): the rows of segment s are exactly [ptr[s], ptr[s+1]) (the segment_sum convention,
 * ptr[n_seg] == R); the kernel then walks segments -- one scaled row of G held in registers, streamed to its
 * rows -- and never reads seg_of_row.  n_seg == 0: per-row lookup through seg_of_row. */
int dmpnn_segment_bcast(const void* G, int g_dtype, int64_t ldg, const int32_t* seg_of_row,
                        const int32_t* ptr, int64_t n_seg, int64_t R, int64_t C, int scale_mode, float scale,
                        void* Y, int y_dtype, int64_t ldy, void* stream);

/* ---------------------------------------------------------------------------------------
 * Bond message (mixins.py:11-18):  M[e] = sum_{e': dst(e')=src(e)} H[e'] - H[rev(e)], computed
 * per atom v over its in-edge rows e'_1..e'_d:  s = sum_i f(X[rd(e'_i)]);
 * OUT[wr(e'_i)] = s - f(X[rd(e'_i)])  with (rd, wr) = (identity, rev) when permute_on_read==0
 * (forward: OUT = M) and (rev, identity) when permute_on_read!=0 (autograd mirror:
 * dH[e] = sum_{src(e'')=dst(e)} dM[e''] - dM[rev(e)]).  Requires DMPNN_FLAG_REV_INVOLUTION.
 * f = `act` on load (used at depth step 1 where H^0 = tau(H_0), base.py:200).
 * ------------------------------------------------------------------------------------- */
int dmpnn_bond_message(const void* X, int x_dtype, int64_t ldx,
                       const int32_t* rowptr, const int32_t* rev_row, int64_t V, int64_t C,
                       int act, float act_param, int permute_on_read,
                       void* OUT, int out_dtype, int64_t ldo, void* stream);

/* Autograd mirror of the message with tau' fused: OUT[r] = (sum_{r' in seg(dst r)} X[rev r'] - X[rev r]) * tau'(Y[r])
 * (= dZ^{t-1} from dM^t and the stored H^{t-1}); one dtype for X / Y / OUT; C % 4 == 0, 4-element aligned. */
int dmpnn_bond_message_bwd_masked(const void* X, int dtype, int64_t ldx, const int32_t* rowptr, const int32_t* rev_row,
                                  int64_t V, int64_t C, const void* Yact, int64_t ldy, int act, float act_param,
                                  void* OUT, int64_t ldo, void* stream);
/* OUT[r] = sum_{k<n_z} Z_k[r] + G[r] * tau'(Ypre[r])  (tau' from the PRE-activation; G may be NULL): the total dH_0 of
 * base.py:135-141's autograd mirror in one pass.  Z: host array of <= 8 device pointers sharing ldz / dtype. */
int dmpnn_sum_act_bwd(const void* const* Z, int n_z, int64_t ldz, const void* G, int64_t ldg, const void* Ypre, int64_t ldy,
                      int dtype, int act, float act_param, void* OUT, int out_dtype, int64_t ldo, int64_t R, int64_t C,
                      void* stream);

/* Undirected averaging (base.py:202-203): OUT[r] = (f(X[r]) + f(X[rev(r)])) / 2, f = `act` on
 * load (identity for ACT_NONE).  Self-adjoint when rev is an involution, so with ACT_NONE the
 * same call is its own autograd mirror. */
int dmpnn_rev_average(const void* X, int x_dtype, int64_t ldx, const int32_t* rev_row,
                      int64_t R, int64_t C, int act, float act_param,
                      void* OUT, int out_dtype, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------
 * Activation backward:  dZ[r,c] = G[gi(r), c] * tau'(.)  where tau' is evaluated from
 * Yact (from_preact==0: Yact holds tau(z); from_preact!=0: Yact holds z).  If ACC != NULL,
 * ACC[r,c] += dZ[r,c] (the dH_0 accumulator of the autograd mirror of base.py:135-141).
 * dZ may be NULL when only the accumulation is wanted.
 * ------------------------------------------------------------------------------------- */
int dmpnn_act_bwd(const void* G, int g_dtype, int64_t ldg, const int32_t* gidx,
                  const void* Yact, int y_dtype, int64_t ldy, int from_preact,
                  int act, float act_param,
                  void* dZ, int dz_dtype, int64_t lddz,
                  void* ACC, int acc_dtype, int64_t ldacc,
                  int64_t R, int64_t C, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fused Hopper depth step (bf16 hidden states, wgmma + TMA + mbarrier):
 *   H_next[rev(e')] = tau( H_0[rev(e')] + bias + W_h . ( sum_{in(v)} g(H_prev) - g(H_prev[e']) ) )
 * i.e. message (mixins.py:11-18) + update (base.py:135-141) in ONE launch, one CTA per SM,
 * molecule-aligned 128-row tiles from dmpnn_layout_build.  g = tau when first_step!=0
 * (H_prev = H_0 and H^0 = tau(H_0) is recomputed on load), identity otherwise.
 * Wpk is W_h packed by dmpnn_pack_weight_bf16.  Requires ld % 16 == 0, a 32-byte aligned H_next, h <= 304,
 * DMPNN_FLAG_REV_INVOLUTION; returns <0 (and does nothing) otherwise.  Without a work table (work_flag, n_work_dev and dst_row
 * NULL) every tile must hold <= 128 rows and <= 128 atoms (DMPNN_META_MAX_TILE_ROWS / _ATOMS): the kernel stages a tile's
 * row-pointer slice of natoms + 1 entries in 132 words.  A layout with a larger tile must pass dmpnn_work_table_build's
 * tables, which flag every such tile.
 * M_out (nullable; first_step only; bf16, same ld, 32-byte aligned, ld % 16 == 0): also stores the message
 * M^1[e] (mixins.py:11-18) that the step consumed, saved for the W_h gradient instead of being recomputed.
 * Precondition: columns [h, pad16(h)) of every hidden input (H_prev, H_0) are zero (finite).  The kernel reads them (its TMA
 * boxes span pad16(h) columns, the epilogue reads H_0 words there) and multiplies them by the zero rows of the packed weight:
 * a NaN or Inf there makes the whole output row NaN.  Columns [h, pad16(h)) of H_next are written as tau(H_0 there), i.e. zero.
 * ------------------------------------------------------------------------------------- */
/* ---------------------------------------------------------------------------------------
 * Tensor-core linear layers of the bf16 tier (wgmma / TMA), for the GEMMs outside the fused
 * depth step: W_i (mixins.py:8-9, 22-23), W_o (base.py:180-182) and dX = dY.W of their autograd mirror.
 *   dmpnn_concat_bf16     A[r] = bf16([X1[i1(r)] || X2[i2(r)] || 0..])  (torch.cat of mixins.py:9 / base.py:180)
 *   dmpnn_pack_weight_tc  nn.Linear weight (or its transpose: transpose != 0 packs B[n][k] = W[k][n]) ->
 *                         per-k-slab shared-memory images.  The image layout (swizzle, and the rows permuted inside
 *                         each 152-row work item so that the epilogue stores column runs) is internal to the library:
 *                         only dmpnn_linear_tc_bf16 / dmpnn_linear_tc_rows_bf16 read it
 *   dmpnn_linear_tc_bf16  C[r, 0:N] = act(A[r, 0:K] . B^T + bias + res[r, 0:N]); A, C, res (nullable; the H_0
 *                         residual of base.py:138, ldres % 8 == 0) bf16 row-major, lda/ldc % 8 == 0,
 *                         ldc >= pad16(N), K <= 448, N <= 304; C columns [N, pad16(N)) are written as zeros.
 *                         Precondition: res columns [N, pad16(N)) are zero.  The epilogue adds res to whole column
 *                         runs, so C's padding is act(res's padding); NaN there would reach the padding that the fused
 *                         depth step reads as zeros.  (A per-column guard cost 0.7 % of C2 throughput on an
 *                         H100 80GB HBM3 at 700 W; DESIGN.md section 4.2.)
 * ------------------------------------------------------------------------------------- */
int dmpnn_concat_bf16(const void* X1, int x1_dtype, int64_t ld1, const int32_t* idx1, int64_t K1,
                      const void* X2, int x2_dtype, int64_t ld2, const int32_t* idx2, int64_t K2,
                      void* OUT, int64_t ldo, int64_t width, int64_t R, void* stream);
/* the same gather-concatenate with an f32 result: the operands of the fp32 tier's tensor-core GEMMs (dmpnn_linear_x3) */
int dmpnn_concat_f32(const void* X1, int x1_dtype, int64_t ld1, const int32_t* idx1, int64_t K1,
                     const void* X2, int x2_dtype, int64_t ld2, const int32_t* idx2, int64_t K2,
                     float* OUT, int64_t ldo, int64_t width, int64_t R, void* stream);
int dmpnn_pack_weight_tc_bytes(int64_t N, int64_t K, size_t* bytes);
int dmpnn_pack_weight_tc(const float* W, int64_t ldw, int64_t N, int64_t K, int transpose, void* Wpk, void* stream);
int dmpnn_linear_tc_bf16(const void* A, int64_t lda, int64_t R, int64_t K, const void* Wpk, int64_t N,
                         const float* bias, const void* res, int64_t ldres, int act, float act_param,
                         void* C, int64_t ldc, void* stream);
/* The same kernel with the epilogues of the per-atom / per-edge read-outs (mol-atom-bond message passing), acc = A[r, 0:K] . B^T:
 *   forward mode (Y == NULL):  C[r, 0:N] = act(acc + bias), stored as out_dtype.  DMPNN_F32: columns [0, N) only,
 *                              ldc >= N and even, C 8-byte aligned; DMPNN_BF16: as dmpnn_linear_tc_bf16 (ldc >= pad16(N)).
 *                              out_row, res, res_row must be NULL and from_preact 0.
 *   mirror mode (Y != NULL):   with q = out_row[r] and s = res_row[r] (identity where the map is NULL),
 *                              C[q, 0:N] = (acc + res[s, 0:N]) * tau'(Y[q, 0:N]), bf16, columns [N, pad16(N)) zeroed;
 *                              tau' of `act` evaluated from the activation output Y, or from the pre-activation when
 *                              from_preact != 0.  res nullable.  Y, res, C bf16 with ld >= pad16(N), ld % 8 == 0, 16-byte
 *                              aligned; bias must be NULL; C may not alias A, Y or res.  out_row must not repeat a row
 *                              (rows of C not named by it are left as they are); res_row may.
 * A and Wpk as for dmpnn_linear_tc_bf16; K <= 448, N <= 304. */
int dmpnn_linear_tc_rows_bf16(const void* A, int64_t lda, int64_t R, int64_t K, const void* Wpk, int64_t N,
                              const float* bias, int act, float act_param, const void* Y, int64_t ldy, int from_preact,
                              const int32_t* out_row, const void* res, int64_t ldres, const int32_t* res_row,
                              void* C, int out_dtype, int64_t ldc, void* stream);

/* Autograd mirror of one depth step on the same fused kernel (gather-by-rev mode):
 *   dOut[e] = ( sum_{e'' : src(e'') = dst(e)} dM[e''] - dM[rev(e)] ) * tau'(Yact[e]),   dM = dZ . W_h
 * computed as ((S.P) dZ) . W_h with the row mixing done on the A operand; WpkT = dmpnn_pack_weight_bf16 of W_h^T.
 * Yact = the stored activation output H^{t-1} (tau' is evaluated from it); Yact == NULL -> no mask (dH^0).
 * y_is_preact != 0: Yact holds the PRE-activation (H_0) and tau' is evaluated from it -- the t = 1 step; then
 * add0 / add1 (nullable, bf16, same ld, 16-byte aligned, must not alias dOut) are summed into the output in f32
 * before the single rounding, so that step writes dH_0 = dZ^{T-1} + .. + dZ^1 + dH^0 * tau'(H_0) directly.
 * G_out (nullable, bf16, same ld, 32-byte aligned, ld % 16 == 0): also writes the gathered operand G = (S.P) dZ, so
 * that the W_h gradient of this step is the plain GEMM dW_h += G^T . H^{t-1} (dZ^T . M^t == ((S.P) dZ)^T . H^{t-1}).
 * Same size / layout / tile requirements as dmpnn_bond_step_fused_bf16 (tiles of more than 128 rows or atoms only through
 * the work table), and the same precondition: columns [h, pad16(h)) of every
 * hidden input (dZ, Yact, add0, add1) are zero (finite).  Columns [h, pad16(h)) of dOut are written as zeros. */
int dmpnn_bond_step_bwd_fused_bf16(const void* dZ, const void* Yact, void* dOut, int64_t ld, int64_t n_rows_alloc,
                                   int64_t h, const void* WpkT, const int32_t* rowptr, const int32_t* rev_row,
                                   const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles,
                                   int act, float act_param, int y_is_preact, const void* add0, const void* add1,
                                   void* G_out, const int8_t* work_flag, const int32_t* n_work_dev, const int32_t* dst_row,
                                   void* stream);

/* Molecule-aligned tiles with caller-given limits (the packing rule of dmpnn_layout_build: greedy, restarted every 1024
 * molecules): tile_row_ptr / tile_atom_ptr [<= B + 1] receive the first edge row / first atom of every tile plus the end
 * sentinel, info[0..2] = tile count, max rows (edges) and max atoms of a tile.  Used for the ATOM tiles (<= 128 atoms) of
 * dmpnn_atom_step_fused_bf16.  Workspace from dmpnn_tiles_workspace_bytes; stream-ordered, no host sync. */
int dmpnn_tiles_workspace_bytes(int64_t B, size_t* bytes);
int dmpnn_tiles_build(const int32_t* mol_atom_ptr, const int32_t* mol_row_ptr, int64_t B, int row_limit, int atom_limit,
                      int32_t* tile_row_ptr, int32_t* tile_atom_ptr, int32_t* info, void* workspace, void* stream);

/* Atom-granular fused depth step -- AtomMessagePassing (chemprop/nn/message_passing/mixins.py:25-30 + base.py:135-141)
 * restated on atoms (the reference's edge state H[e] depends only on src(e)):
 *   H_next[v] = act( H_0[v] + bias + W . sum_{e in in(v)} g(H_prev[src(e)]) ),   g = act on the first step, identity after,
 * one launch: neighbour gather from the TMA-loaded atom tile + wgmma GEMM + epilogue, the kernel of
 * dmpnn_bond_step_fused_bf16 with its ATOM gather.  The loop-invariant bond term W_h[:, h:] . sum_in E of the reference's
 * update is folded into H_0 by the caller (engine.atom_forward_fused).  rowptr: dst-sorted CSR over atoms; nbr_row: source
 * atom of every edge row; tile_atom_ptr / tile_edge_ptr: first atom / first edge row of every atom tile (dmpnn_tiles_build
 * with atom_limit = 128) and *n_tiles_dev tiles (device scalar; n_tiles_max only sizes the checks).  Every molecule must
 * have <= 128 atoms.  N_out (first step only): the gathered operand, for the W_h gradient.  The mirror:
 *   dOut[v] = ( (sum_{e in in(v)} dZ[src(e)]) . W ) * act'(Yact[v])      (the adjacency is symmetric)
 * with the modes of dmpnn_bond_step_bwd_fused_bf16 (Yact null: no mask; y_is_preact + addends: the last step).
 * Both entry points have the precondition of dmpnn_bond_step_fused_bf16: columns [h, pad16(h)) of every hidden input
 * (H_prev, H_0; dZ, Yact, add0, add1) are zero (finite), else whole output rows come out NaN.
 * The unmasked mode (Yact null) once gave NaN gradients on condensed-reaction batches (~80-atom molecules, h = 300), not at
 * h = 64.  That is this precondition broken: on 40 such graphs at h = 300 it gives no NaN with zero padding and a NaN in
 * every row with NaN in columns [300, 304); h = 64 has no padding column.  All modes are tested (DESIGN.md section 9). */
int dmpnn_atom_step_fused_bf16(const void* H_prev, const void* H_0, void* H_next, int64_t ld, int64_t n_rows_alloc, int64_t h,
                               const void* Wpk, const float* bias, const int32_t* rowptr, const int32_t* nbr_row,
                               const int32_t* tile_atom_ptr, const int32_t* tile_edge_ptr, const int32_t* n_tiles_dev,
                               int64_t n_tiles_max, int act, float act_param, int first_step, void* N_out, void* stream);
int dmpnn_atom_step_bwd_fused_bf16(const void* dZ, const void* Yact, void* dOut, int64_t ld, int64_t n_rows_alloc, int64_t h,
                                   const void* WpkT, const int32_t* rowptr, const int32_t* nbr_row,
                                   const int32_t* tile_atom_ptr, const int32_t* tile_edge_ptr, const int32_t* n_tiles_dev,
                                   int64_t n_tiles_max, int act, float act_param, int y_is_preact, const void* add0,
                                   const void* add1, void* G_out, void* stream);

/* Tensor-core weight gradient (bf16 operands, f32 accumulate, deterministic two-pass reduction):
 *   dW[n, 0:K] (+)= sum_r dY[r, n] * X[r, 0:K]      dY: R x N (ld lddy), X: R x K (ld ldx), both bf16 row-major
 * N <= 384, K <= 448; lddy, ldx multiples of 8.  Workspace from dmpnn_wgrad_tc_workspace_bytes. */
int dmpnn_wgrad_tc_workspace_bytes(int64_t N, int64_t K, size_t* bytes);
int dmpnn_wgrad_tc_bf16(const void* dY, int64_t lddy, const void* X, int64_t ldx, int64_t R, int64_t N, int64_t K,
                        float* dW, int64_t lddw, int accumulate, void* workspace, void* stream);
/* The same with up to three dY terms sharing the launch:  dW (+)= sum_t dY_t^T X  (all terms R x N with one ld; X is read
 * once per stage).  2 * n_terms + ceil(K / 64) <= 9.  Used for the W_i gradient (mixins.py:8-9 under autograd), whose
 * upstream gradient dH_0 = sum_t dZ^t + dH^0 tau'(H_0) is a sum the mirror never forms. */
int dmpnn_wgrad_tc_multi_bf16(const void* const* dYs, int n_terms, int64_t lddy, const void* X, int64_t ldx, int64_t R,
                              int64_t N, int64_t K, float* dW, int64_t lddw, int accumulate, void* workspace, void* stream);
/* Column sums (bias gradient): out[n] (+)= sum_r Y[r, n].  Workspace: dmpnn_linear_wgrad_workspace_bytes(R, N, 1). */
int dmpnn_column_sum(const void* Y, int y_dtype, int64_t ldy, int64_t R, int64_t N, float* out, int accumulate,
                     void* workspace, void* stream);

/* Debug aid: when set (device pointer to n_tiles x 12 uint64, zero-filled), block 0 of the fused
 * kernel records %globaltimer stamps of its pipeline phases for its first n_tiles tiles. NULL = off. */
int dmpnn_set_trace_buffer(void* dev_ptr, int64_t n_tiles);
/* W (f32, N x K) -> the fused step's bf16 weight image.  Its layout (80-row chunks x 64-column k slabs, swizzled, rows
 * permuted inside each chunk so that the epilogue stores column runs) is internal: only the fused step kernels read it. */
int dmpnn_pack_weight_bf16_bytes(int64_t N, int64_t K, size_t* bytes);
int dmpnn_pack_weight_bf16(const float* W, int64_t ldw, int64_t N, int64_t K, void* Wpk, void* stream);
int dmpnn_bond_step_fused_bf16(const void* H_prev, const void* H_0, void* H_next, int64_t ld,
                               int64_t n_rows_alloc, int64_t h,
                               const void* Wpk, const float* bias,
                               const int32_t* rowptr, const int32_t* rev_row,
                               const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles,
                               int act, float act_param, int first_step, void* M_out,
                               const int8_t* work_flag, const int32_t* n_work_dev, const int32_t* dst_row,
                               const void* drop_bits, float drop_scale, void* stream);

/* Training-mode dropout of base.py:139 INSIDE the fused step: `drop_bits` (nullable) holds 16 keep bits per (row, 16-column
 * block) -- uint16 [n_rows][pad16(h) / 16], bit q of word j = column 16 j + q, 2-byte aligned -- and the epilogue writes
 * keep ? tau(z) * drop_scale : 0 with one rounding (drop_scale = 1 / (1 - p), finite and > 0); no mask pass over the E x h
 * matrix.  Every fused activation takes keep bits, on every work item (the windows of oversized molecules too).  The
 * autograd mirror reads the mask back out of tau' of the stored state, which holds for ReLU only: a training step uses
 * keep bits with ReLU, a forward-only call (Monte Carlo dropout) with any activation.
 * dmpnn_dropout_bits fills such an array from Philox4x32-10 (key = seed, counter = (word index, offset)): bit = [u16 >= round(p *
 * 65536)], i.e. P(drop) = p to 2^-16; the same (seed, offset) always gives the same bits. */
int dmpnn_dropout_bits(void* bits, int64_t n_rows, int64_t words_per_row, float p, uint64_t seed, uint64_t offset, void* stream);

/* Work table for batches with molecules of MORE than 128 directed edges (condensed reaction graphs, BASELINE config 4 with
 * BondMessagePassing) or MORE than 128 atoms: the layout's tiles, with every tile of > 128 rows (one oversized molecule) cut
 * into windows of <= 128 consecutive rows, and every tile of <= 128 rows but > 128 atoms (one molecule of many fragments)
 * kept as one window.  Outputs: work_row_ptr / work_atom_ptr (n_work + 1 entries; capacity n_tiles + E / 128 + 2), work_flag
 * (1 = window of an oversized molecule, 0 = a tile within both limits) and the device scalar n_work.  Pass work_row_ptr /
 * work_atom_ptr as the tile tables of the fused step together with work_flag, n_work and the layout's dst_row (all three
 * NULL for batches whose tiles all hold <= 128 rows and <= 128 atoms): a flagged window gathers its sibling / reverse-edge
 * rows from global memory instead of its shared-memory tile.  n_tiles == 0 gives n_work = 0 and zero sentinels. */
int dmpnn_work_table_build(const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles,
                           int32_t* work_row_ptr, int32_t* work_atom_ptr, int8_t* work_flag, int32_t* n_work, void* stream);

/* ---------------------------------------------------------------------------------------
 * fp32-ACCURATE tensor-core GEMMs of the fp32 tier (csrc/gemm_x3.cu): every product is three
 * tf32 wgmma passes over an error-free hi / lo split of both operands, f32 accumulation in registers --
 * the accuracy of an f32 FMA chain (the reference's ATen sgemm on base.py:135-141, 180-182) at tensor-core
 * speed; hidden size up to 4096 (BASELINE config 3: h = 600, depth 6).
 *   dmpnn_pack_weight_x3  nn.Linear weight W (N x K f32, row stride ldw; transpose != 0: B[n][k] = W[k][n]) ->
 *                         pre-split {hi, lo} shared-memory images per (128-column pass, 32-wide k slab)
 *   dmpnn_linear_x3       C[r, 0:N] = act(A[row_idx ? row_idx[r] : r, 0:K] . B^T + bias + res[r, 0:N]);  A, C, res f32
 *                         row-major; K % 4 == 0, lda / ldc / ldres % 4 == 0, 16-byte aligned bases;
 *                         C columns [N, min(ldc_pad, pad16(N))) are written as zeros.
 *   dmpnn_wgrad_x3        dW[n, 0:K] (+)= sum_r dY[r, n] * X[r, 0:K];  dY: R x N, X: R x K f32 row-major, N, K, lddy,
 *                         ldx % 4 == 0; deterministic two-pass reduction; workspace from dmpnn_wgrad_x3_workspace_bytes.
 * ------------------------------------------------------------------------------------- */
int dmpnn_pack_weight_x3_bytes(int64_t N, int64_t K, size_t* bytes);
int dmpnn_pack_weight_x3(const float* W, int64_t ldw, int64_t N, int64_t K, int transpose, void* Wpk, void* stream);
int dmpnn_linear_x3(const float* A, int64_t lda, const int32_t* row_idx, int64_t R, int64_t K, const void* Wpk,
                    int64_t N, const float* bias, const float* res, int64_t ldres, int act, float act_param,
                    float* C, int64_t ldc, int64_t ldc_pad, void* stream);
int dmpnn_wgrad_x3_workspace_bytes(int64_t N, int64_t K, size_t* bytes);
int dmpnn_wgrad_x3(const float* dY, int64_t lddy, const float* X, int64_t ldx, int64_t R, int64_t N, int64_t K,
                   float* dW, int64_t lddw, int accumulate, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------
 * Molecule-level head of the training step (csrc/head.cu; chemprop/models/model.py:126-161):
 *   dmpnn_bn_train_fwd  nn.BatchNorm1d in training mode on X (B x d f32): Y = (X - mean) * invstd * gamma + beta with the
 *                       batch mean / biased variance; running_mean / running_var (nullable) are updated in place with
 *                       `momentum` and the unbiased variance; Xhat, save_mean, save_invstd are kept for the mirror.
 *   dmpnn_bn_bwd        dX (and dgamma, dbeta when non-null) from dY, Xhat, invstd.
 *   dmpnn_mse_loss      chemprop's MSE criterion (nn/metrics.py:78-123, 139-141): loss[0] = sum_{b,t} w[b] tw[t] m (P - Y)^2
 *                       / sum m with m = isfinite(Y) (NaN target = masked, model.py:140-141); dP (nullable) = dloss/dP.
 *   dmpnn_bce_loss      chemprop's BCELoss (nn/metrics.py:291-294) under the same reduction: loss[0] = sum_{b,t} w[b] tw[t] m
 *                       L / sum m, L = binary_cross_entropy_with_logits(P, Y) in torch's stable form
 *                       (1 - y) x + mx + log(e^{-mx} + e^{-x-mx}), mx = max(-x, 0); dP = (sigmoid(P) - Y) w tw m / sum m.
 *                       Y may hold soft labels in [0, 1].  P, Y, dP: B x T.
 *   dmpnn_ce_loss       chemprop's CrossEntropyLoss (nn/metrics.py:297-303): P is B x (T*C), task t owning columns
 *                       [t*C, (t+1)*C) (the layout of ffn(Z).reshape(B, T, C)); Y is B x T.  L = logsumexp(row) -
 *                       row[label] with label = trunc(Y) as torch's `.long()`; dP row = (softmax(row) - onehot) w tw m /
 *                       sum m.  A finite label whose truncation lies outside [0, C) makes loss[0] NaN and that row of dP
 *                       NaN: the reference raises there, which a kernel cannot do without synchronising with the host.
 *                       C = 1 is legal (loss and gradient 0).
 *   dmpnn_class_probs   eval-mode outputs of the classification predictors on P (B x (T*C)): softmax == 0 gives the
 *                       sigmoid of every entry (binary, C = 1), softmax == 1 the softmax of every group of C columns.
 * The three losses mask like dmpnn_mse_loss: m = isfinite(Y); with every target masked, loss[0] = 0 and dP = 0 (the
 * reference's 0 / 0 would be NaN).  dP is written for every element, masked ones as zeros.  B = 0 is accepted; weights
 * and task_weights are nullable (all ones).  One block per loss call.
 * All reductions run in a fixed order (deterministic); no host synchronisation.
 * ------------------------------------------------------------------------------------- */
int dmpnn_bn_train_fwd(const float* X, int64_t ldx, int64_t B, int64_t d, const float* gamma, const float* beta,
                       float eps, float momentum, float* running_mean, float* running_var, float* Y, int64_t ldy,
                       float* Xhat, int64_t ldh, float* save_mean, float* save_invstd, void* stream);
int dmpnn_bn_bwd(const float* dY, int64_t lddy, const float* Xhat, int64_t ldh, int64_t B, int64_t d,
                 const float* gamma, const float* invstd, float* dX, int64_t lddx, float* dgamma, float* dbeta,
                 void* stream);
int dmpnn_mse_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                   const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp, void* stream);
int dmpnn_bce_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                   const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp, void* stream);
int dmpnn_ce_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                  const float* task_weights, int64_t B, int64_t T, int64_t C, float* loss, float* dP, int64_t lddp,
                  void* stream);
int dmpnn_class_probs(const float* P, int64_t ldp, int64_t B, int64_t T, int64_t C, int softmax, float* out, int64_t ldo,
                      void* stream);

/* ---------------------------------------------------------------------------------------
 * Uncertainty predictors and target unscaling (csrc/head.cu; chemprop/nn/predictors.py:160-228, 250-270, 319-336,
 * nn/transforms.py:45-55, nn/metrics.py:202-257, 502-544, 588-613):
 *   dmpnn_pred_transform      X (B x (T*u), the raw MLP output) -> out (B x T x u, row stride ldo >= T*u), one thread per
 *                             (b, t).  kind / u:
 *                               0 regression (u = 1)       out = x
 *                               1 MVE (u = 2)              (mean, softplus(var))
 *                               2 evidential (u = 4)       (mean, softplus(v), softplus(alpha) + 1, softplus(beta))
 *                               3 quantile (u = 2)         (lo + hi) / 2, hi - lo
 *                               4 Dirichlet (u = C >= 1)   alpha = softplus(x) + 1
 *                               5 Dirichlet probabilities  alpha / sum(alpha)
 *                               6 binary Dirichlet (u = 2) (alpha_1 / S, 2 / S), S = alpha_0 + alpha_1
 *                               7 softplus (u = 1)         softplus(x): RegressionFFN's nn.Softplus() output transform
 *                                                          (beta 1, threshold 20), in training and eval mode
 *                             Kinds 0-3 read target j of task t from column j*T + t (torch.chunk of the MLP output);
 *                             kinds 4-6 read class c of task t from column t*u + c (reshape(B, T, u)).  softplus is
 *                             F.softplus with threshold 20.  mean and scale (T entries each, both or neither, kinds 0-3
 *                             only) apply UnscaleTransform's eval mode: x*scale + mean to the mean / bounds, var*scale^2
 *                             to MVE's var and evidential's beta, each product and sum rounded as torch rounds it.
 *   dmpnn_pred_transform_bwd  the mirror for kinds 0-4 and 7: dX (B x (T*u)) from dOut (B x T x u) and the forward's X; scale
 *                             (nullable) as in the forward.  Every column of dX in [0, T*u) is written.
 *   dmpnn_mve_loss            MVELoss on P (B x T x 2: mean, var): L = (mean - y)^2 / (2 var) + log(2 pi var) / 2
 *   dmpnn_evidential_loss     EvidentialLoss on P (B x T x 4: mean, v, alpha, beta) with v_kl and eps; d|r|/dr = 0 at r = 0
 *   dmpnn_quantile_loss       QuantileLoss on P (B x T x 2: mean, interval) at `alpha`: pinball losses of the bounds
 *                             mean -/+ interval / 2; where the two candidates of a bound's amax tie (target exactly on the
 *                             bound) the gradient is split evenly between them, as torch's amax does
 *   dmpnn_dirichlet_loss      DirichletLoss on P (B x T x C: alpha >= 1) with v_kl; its digamma / trigamma are written for
 *                             arguments >= 1 (recurrence below 6, asymptotic series above)
 * The four losses reduce like dmpnn_mse_loss: loss[0] = sum_{b,t} w[b] tw[t] m L / sum m with m = isfinite(Y), dP (nullable,
 * B x T x u, written for every element, masked ones as zeros) = dloss/dP; with every target masked loss[0] = 0 and dP = 0
 * (the reference's 0 / 0 would be NaN).  One block per call; fixed reduction order; no host synchronisation.
 * Dirichlet labels follow torch.eye(C)[Y.long()]: trunc(Y) in [0, C) is the class, in [-C, 0) it counts from the end
 * (class trunc(Y) + C); outside [-C, C) the reference raises, and the kernel makes loss[0] NaN and that row of dP NaN.
 * ------------------------------------------------------------------------------------- */
int dmpnn_pred_transform(const float* X, int64_t ldx, int64_t B, int64_t T, int kind, int64_t u, const float* mean,
                         const float* scale, float* out, int64_t ldo, void* stream);
int dmpnn_pred_transform_bwd(const float* X, int64_t ldx, const float* dOut, int64_t lddo, int64_t B, int64_t T, int kind,
                             int64_t u, const float* scale, float* dX, int64_t lddx, void* stream);
int dmpnn_mve_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                   const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp, void* stream);
int dmpnn_evidential_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                          const float* task_weights, int64_t B, int64_t T, float v_kl, float eps, float* loss, float* dP,
                          int64_t lddp, void* stream);
int dmpnn_quantile_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                        const float* task_weights, int64_t B, int64_t T, float alpha, float* loss, float* dP, int64_t lddp,
                        void* stream);
int dmpnn_dirichlet_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                         const float* task_weights, int64_t B, int64_t T, int64_t C, float v_kl, float* loss, float* dP,
                         int64_t lddp, void* stream);

/* ---------------------------------------------------------------------------------------
 * Count-data regression (csrc/head.cu; chemprop/nn/metrics.py:616-692, the loss of DNA-encoded-library screens):
 *   dmpnn_enrichment_loss     NLogProbEnrichment on R (B x 1, row stride ldr: the predicted enrichment, softplus output)
 *                             and Y (B x 2, row stride ldy: counts k1 in the positive and k2 in the negative sample).
 *                             Per molecule, with k = Y where finite and 0 where not (training_step's nan_to_num) and
 *                             Rd = R / d (d = n2 / n1):
 *                               method 0 sqrt   z = 2 (sqrt(k1 + 3/8) - sqrt((k2 + 3/8) Rd)) / sqrt(1 + Rd)
 *                               method 1 score  z = (k1 - k2 Rd) / sqrt((k1 + k2) Rd)
 *                               method 2 wald   z = (k1 - k2 Rd) / sqrt(k1 + k2 Rd^2)
 *                             c = clamp(z / zscale, -zinterval, zinterval), L = -log(1 - erf(|c| / sqrt 2)), computed as
 *                             x^2 - log(erfcx(x)) with x = |c| / sqrt 2 (no cancellation, no underflow).  loss[0] =
 *                             sum_b L_b w[b] (tw[0] m_b0 + tw[1] m_b1) / sum m with m = isfinite(Y): the reference's b x 1
 *                             loss broadcast against its b x 2 mask.  task_weights (nullable) has exactly 2 entries.
 *                             dR (nullable, row stride lddr) = dloss/dR for every row, masked ones 0; the clamp passes
 *                             the gradient at its bounds (inclusive) and not outside, d|c|/dc = 0 at c = 0, as torch's
 *                             autograd.  Where the reference raises ("Got nan loss", any NaN z, masked rows included:
 *                             score / wald with a row of zero counts, a NaN prediction) loss[0] is NaN, and so is that
 *                             row's dR.  Every target masked: loss[0] = 0 and dR = 0.  One block; fixed reduction order;
 *                             no atomics; no host synchronisation.  Refused: an unknown method, d not finite and > 0,
 *                             zscale not finite and nonzero, zinterval not finite and >= 0.
 * ------------------------------------------------------------------------------------- */
int dmpnn_enrichment_loss(const float* R, int64_t ldr, const float* Y, int64_t ldy, const float* weights,
                          const float* task_weights, int64_t B, float d, int method, float zscale, float zinterval,
                          float* loss, float* dR, int64_t lddr, void* stream);

/* ---------------------------------------------------------------------------------------
 * Regression-loss family and the spectral predictor (csrc/head.cu; chemprop/nn/metrics.py:128-183, 547-585,
 * nn/predictors.py:339-376):
 *   dmpnn_regression_loss     kind 0 MSE, 1 MAE, 2 RMSE under dmpnn_mse_loss's reduction and masking (dmpnn_mse_loss is
 *                             kind 0 without bounds, bit for bit).  MAE: L = |P - Y|, d|e|/de = 0 at e = 0 as torch's
 *                             abs.  RMSE: loss[0] = sqrt(the MSE value), dP = the MSE's dP / (2 loss[0]); where the loss
 *                             is 0 (every residual exactly 0) dP = 0 (the reference's sqrt backward gives 0 * inf = NaN).
 *                             lt_mask / gt_mask (nullable uint8, B x T, row stride ldm) give the bounded variants: where
 *                             lt_mask is set and P < Y, or gt_mask is set and P > Y, the residual is 0 and so are the term
 *                             and its gradient (BoundedMixin's torch.where).  One block.
 *   dmpnn_spectral_transform  SpectralFFN's output from the raw MLP output X (B x T): y = a(a(x)) (the reference applies
 *                             its activation twice), out = y / sum_j y_j per row over every bin.  act 0 = softplus
 *                             (dmpnn_pred_transform's, threshold 20), 1 = exp.  T = 1 gives exactly 1.
 *   dmpnn_spectral_transform_bwd  the mirror: dX from dOut and the forward's X.
 *   dmpnn_sid_loss            SID on P (B x T, the spectra) and Y (B x T): c = clamp(P, min = threshold) (threshold NaN:
 *                             none; the gradient passes where P >= threshold, as torch's clamp), pn = c / sum_j m_j c_j
 *                             per row, L = pn log(pn / y) + y log(y / pn) on the masked-in bins.
 *   dmpnn_wasserstein_loss    L_j = |cumsum(y0)_j - cumsum(pn)_j| with y0 = Y where finite and 0 where masked, pn (as in
 *                             SID) over every bin, masked or not; d|D|/dD = 0 at D = 0 (a cumsum tie), as torch's abs.
 *   Both spectral losses reduce like dmpnn_mse_loss: loss[0] = sum_{b,j} w[b] tw[j] m L / sum m, m = isfinite(Y), dP
 *   (nullable) = dloss/dP, every entry written.  Conventions where the reference gives NaN:
 *     - a row with every bin masked adds 0 to the loss and has dP = 0 (SID's reference: NaN gradient; Wasserstein's:
 *       NaN loss), and every target masked gives loss[0] = 0;
 *     - SID with a masked-in target of exactly 0 keeps the reference's NaN: loss[0] is NaN and so is that row's dP at its
 *       masked-in bins (its masked bins stay 0).
 *   One CTA of 256 threads per row, bins in chunks of 256 (any T); Wasserstein's cumsums are chunked block scans, forward
 *   for the loss and in reverse for the gradient.  The 1 / sum m of the gradient comes from a count prepass on the device,
 *   and a one-block launch sums the per-row losses: three launches, fixed summation order (bitwise repeatable), no
 *   floating-point atomics, no host synchronisation.  workspace: dmpnn_spectral_loss_workspace_bytes(B) bytes, any
 *   contents (every byte read is written first by the same call).
 * ------------------------------------------------------------------------------------- */
int dmpnn_regression_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                          const float* task_weights, const uint8_t* lt_mask, const uint8_t* gt_mask, int64_t ldm, int64_t B,
                          int64_t T, int kind, float* loss, float* dP, int64_t lddp, void* stream);
int dmpnn_spectral_transform(const float* X, int64_t ldx, int64_t B, int64_t T, int act, float* out, int64_t ldo,
                             void* stream);
int dmpnn_spectral_transform_bwd(const float* X, int64_t ldx, const float* dOut, int64_t lddo, int64_t B, int64_t T, int act,
                                 float* dX, int64_t lddx, void* stream);
int dmpnn_spectral_loss_workspace_bytes(int64_t B, size_t* bytes);
int dmpnn_sid_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                   const float* task_weights, int64_t B, int64_t T, float threshold, float* loss, float* dP, int64_t lddp,
                   void* workspace, void* stream);
int dmpnn_wasserstein_loss(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                           const float* task_weights, int64_t B, int64_t T, float threshold, float* loss, float* dP,
                           int64_t lddp, void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------
 * Atom- and bond-level heads (csrc/row_head.cu; chemprop/models/mol_atom_bond.py:140-151, 237-339):
 *   dmpnn_edge_pair_mean      the bond predictor's average over each reverse-edge pair: out[i, 0:C] = (P[2i] + P[2i+1]) / 2
 *                             for i in [0, E/2), P an E x C f32 matrix (row stride ldp), out E/2 x C (row stride ldo).
 *                             Chemprop's edge order is assumed, in which edge 2i+1 is the reverse of edge 2i; the kernel
 *                             reads rev (int32, E) and writes NaN across every output row i with rev[2i] != 2i+1 instead
 *                             of a silently wrong average (the reference's wrapper does not check; a kernel cannot raise
 *                             without synchronising with the host).  E must be even (refused otherwise); E = 0 launches
 *                             nothing.
 *   dmpnn_edge_pair_mean_bwd  its mirror: dP[2i] = dP[2i+1] = G[i] / 2.
 *   dmpnn_pinball_loss_rows   PointQuantileLoss (chemprop/nn/metrics.py:264-288) at `alpha`, under the _rows reduction
 *                             below and at every level (molecules included: it has no single-block twin): L =
 *                             alpha (y - p) where y - p > 0, (1 - alpha)(p - y) otherwise; dL/dp at y == p is 1 - alpha
 *                             (torch.where's second branch).
 *   dmpnn_regression_loss_rows, dmpnn_bce_loss_rows, dmpnn_ce_loss_rows
 *                             dmpnn_regression_loss, dmpnn_bce_loss and dmpnn_ce_loss with the same arguments, conventions
 *                             and outputs (NaN targets masked, w and tw nullable, division by the mask count, loss 0 and
 *                             dP 0 when every target is masked, NaN for a class label outside [0, C)), for B in the
 *                             hundreds of thousands of atom or bond rows: the terms are spread over a grid of up to 1024
 *                             CTAs (at least 2048 terms each), each CTA writing one partial sum to `workspace`, and a
 *                             second launch sums the partials in a fixed order and writes loss[0] and dP.  The grid depends
 *                             on B * T only: bitwise repeatable, no floating-point atomics, no host synchronisation, and
 *                             graph-capturable.  The summation order differs from the single-block kernels', so the two
 *                             agree to rounding, not bit for bit.  The mask count is an exact 64-bit integer.
 *                             workspace: *_rows_workspace_bytes(B, T) bytes, any contents (every byte read is written
 *                             first by the same call).
 * ------------------------------------------------------------------------------------- */
int dmpnn_edge_pair_mean(const float* P, int64_t ldp, const int32_t* rev, int64_t E, int64_t C, float* out, int64_t ldo,
                         void* stream);
int dmpnn_edge_pair_mean_bwd(const float* G, int64_t ldg, int64_t E, int64_t C, float* dP, int64_t lddp, void* stream);
int dmpnn_regression_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes);
int dmpnn_regression_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                               const float* task_weights, const uint8_t* lt_mask, const uint8_t* gt_mask, int64_t ldm,
                               int64_t B, int64_t T, int kind, float* loss, float* dP, int64_t lddp, void* workspace,
                               void* stream);
int dmpnn_bce_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes);
int dmpnn_bce_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                        const float* task_weights, int64_t B, int64_t T, float* loss, float* dP, int64_t lddp,
                        void* workspace, void* stream);
int dmpnn_pinball_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes);
int dmpnn_pinball_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                            const float* task_weights, int64_t B, int64_t T, float alpha, float* loss, float* dP, int64_t lddp,
                            void* workspace, void* stream);
int dmpnn_ce_loss_rows_workspace_bytes(int64_t B, int64_t T, size_t* bytes);
int dmpnn_ce_loss_rows(const float* P, int64_t ldp, const float* Y, int64_t ldy, const float* weights,
                       const float* task_weights, int64_t B, int64_t T, int64_t C, float* loss, float* dP, int64_t lddp,
                       void* workspace, void* stream);

/* ---------------------------------------------------------------------------------------
 * ConstrainerFFN's segmented part (csrc/constrain.cu; chemprop/nn/ffn.py:119-141).  Molecule s owns rows
 * [ptr[s], ptr[s+1]) of R = ptr[m] rows (int32 ptr, m + 1 entries, ptr[0] = 0; empty molecules allowed anywhere).
 * Kl is R x n_c f32 (the constrainer MLP's output), P R x t f32, C m x t f32 (the constraints), all with row strides.
 *   dmpnn_constrain_fwd   out[r, j] = P[r, j] + w[r, i] * (C[s, j] - sum_{r' in s} P[r', j]) for every constrained
 *                         column j, w[r, i] = exp(Kl[r, i]) / sum_{r' in s} exp(Kl[r', i]) (no max-subtraction, as the
 *                         reference); every other column is copied bit for bit.  Column j is constrained iff C[0, j] is
 *                         not NaN (row 0 only, as the reference), and i is its rank among the constrained columns when n_c
 *                         equals their number nq, 0 when n_c == 1.  Any other (n_c, nq >= 1) is a shape the reference
 *                         rejects: every constrained column of out is NaN.  *status (1 int32, device) is written by every
 *                         call with m > 0: 0, or nq for a rejected shape.  No constrained column: out = P.
 *   dmpnn_constrain_bwd   given G = dL/dout: dP[r, j] = G[r, j] - a_j and dKl[r, i] = sum over the constrained j paired
 *                         with i of D_j * w[r, i] * (G[r, j] - a_j), with D_j = C[s, j] - sum_s P[., j] and
 *                         a_j = sum_s G[., j] * w[., i]; unconstrained columns dP = G.  No constrained column: dKl = 0;
 *                         a rejected shape: NaN in dKl and in the constrained columns of dP.  No gradient to C.
 * One warp per molecule, sums in a fixed order: bitwise repeatable, no atomics, no workspace, no host synchronisation.
 * ------------------------------------------------------------------------------------- */
int dmpnn_constrain_fwd(const float* Kl, int64_t ldk, int64_t n_c, const float* P, int64_t ldp, const int32_t* ptr,
                        int64_t m, const float* C, int64_t ldc, int64_t t, float* out, int64_t ldo, int32_t* status,
                        void* stream);
int dmpnn_constrain_bwd(const float* G, int64_t ldg, const float* Kl, int64_t ldk, int64_t n_c, const float* P, int64_t ldp,
                        const int32_t* ptr, int64_t m, const float* C, int64_t ldc, int64_t t, float* dP, int64_t lddp,
                        float* dKl, int64_t lddk, void* stream);

/* ---------------------------------------------------------------------------------------
 * Validation and test metrics (csrc/metrics.cu; chemprop/nn/metrics.py:59-499 and the torchmetrics classes it wraps).
 * P, Y are B x T f32 (row strides ldp, ldy); `mask`, lt_mask, gt_mask are nullable B x T uint8 with row stride ldm, and a
 * null mask means m = isfinite(Y).  Each call ADDS into caller-owned state: f64 sums (fstate) and int64 counts (istate),
 * zeroed by the caller to start.  `status` (1 int32, device) is set to 1 by a call that meets a masked-in target its
 * metric cannot take (a binary label outside {0, 1} after truncation, a class outside [-C, C)) and is otherwise left
 * alone.  Classification inputs follow torchmetrics' per-update formatting: where any considered prediction of the call
 * lies outside [0, 1] (or is NaN) the call reads sigmoid(P) (softmax over the classes for the multiclass MCC); the
 * considered predictions are the masked-in ones for accuracy / F1 / AUROC / AUPRC (chemprop passes preds[mask]) and all of
 * them for the MCCs (the reference tests preds.min() / preds.max()).
 *   dmpnn_metric_accumulate   kind 0 squared error, 1 absolute error (MSE / MAE / RMSE; lt_mask / gt_mask give the bounded
 *                             variants as in dmpnn_regression_loss): fstate[0] += sum w tw m L, istate[0] += sum m;
 *                             kind 2 (R2, pooled over tasks): fstate[0..2] += sum y, sum y^2, sum (y - p)^2, istate[0] +=
 *                             sum m; kind 3 (accuracy / F1, pooled, threshold p > 0.5): istate[0..3] += TP, FP, TN, FN;
 *                             kind 4 (binary MCC, per task, soft): fstate[j * T + t] += the TP, FP, TN, FN (j = 0..3) of
 *                             task t weighted by w m.  weights (B) / task_weights (T) nullable; kinds 2 and 3 ignore them.
 *   dmpnn_metric_multiclass_mcc  P is B x T x C (row stride ldp >= T C, C >= 2); per task t, fstate[t (2C + 2) + j] += p_j
 *                             (j < C), t_j (C + j), c (2C), s (2C + 1) of MulticlassMCCLoss._calc_unreduced_loss, weighted
 *                             by w m; argmax takes the first maximum.
 *   dmpnn_metric_rank_format  one update of AUROC / AUPRC: for element e = b T + t, score[e] = the formatted prediction,
 *                             label[e] = its 0 / 1 target, keep[e] = m (masked-out elements: 0, 0, 0).
 *   Workspace of the three: dmpnn_metric_workspace_bytes(B, T, C) bytes (C = 1 except for the multiclass MCC), any
 *   contents.  Two-phase fixed-order reductions over a grid that depends on the shape only: bitwise repeatable, no
 *   floating-point atomics, no host synchronisation.
 *   dmpnn_rank_curve          AUROC and AUPRC of the n formatted elements kept: out[0] = AUROC (torchmetrics' binary_auroc:
 *                             trapezoids over (fpr, tpr) from the origin, summed exactly in int64 and divided once by
 *                             2 P N; 0 when either class is absent), out[1] = AUPRC (auc(recall, precision) of
 *                             binary_precision_recall_curve with the point (0, 1) appended, trapezoids summed in f64 in a
 *                             fixed order; NaN without positives).  Masked elements sort below every score instead of
 *                             being compacted, so the sort needs no device count on the host: one key pass, one
 *                             cub::DeviceRadixSort (descending, stable), one scan of (positives, run start), a fixed-order
 *                             reduction.  n <= 2^31 - 1; workspace: dmpnn_rank_curve_workspace_bytes(n) bytes, any
 *                             contents, `workspace_bytes` its size.  n = 0 writes (0, NaN).
 * ------------------------------------------------------------------------------------- */
int dmpnn_metric_workspace_bytes(int64_t B, int64_t T, int64_t C, size_t* bytes);
int dmpnn_metric_accumulate(int kind, const float* P, int64_t ldp, const float* Y, int64_t ldy, const uint8_t* mask,
                            const float* weights, const float* task_weights, const uint8_t* lt_mask,
                            const uint8_t* gt_mask, int64_t ldm, int64_t B, int64_t T, double* fstate, int64_t* istate,
                            int32_t* status, void* workspace, void* stream);
int dmpnn_metric_multiclass_mcc(const float* P, int64_t ldp, const float* Y, int64_t ldy, const uint8_t* mask, int64_t ldm,
                                const float* weights, int64_t B, int64_t T, int64_t C, double* fstate, int32_t* status,
                                void* workspace, void* stream);
int dmpnn_metric_rank_format(const float* P, int64_t ldp, const float* Y, int64_t ldy, const uint8_t* mask, int64_t ldm,
                             int64_t B, int64_t T, float* score, uint8_t* label, uint8_t* keep, int32_t* status,
                             void* workspace, void* stream);
int dmpnn_rank_curve_workspace_bytes(int64_t n, size_t* bytes);
int dmpnn_rank_curve(const float* score, const uint8_t* label, const uint8_t* keep, int64_t n, double* out,
                     void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DMPNN_H_ */
