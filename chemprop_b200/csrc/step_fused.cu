// Fused Hopper depth step of BondMessagePassing (bf16 hidden states), one launch per step:
//
//   H_next[rev(e')] = tau( H_0[rev(e')] + b + W_h . ( sum_{e'' in in(v)} g(H[e'']) - g(H[e']) ) ),  e' in in(v)
//
// = message (chemprop/nn/message_passing/mixins.py:11-18) + update (base.py:135-141).  g = tau when
// first_step (H^0 = tau(H_0), base.py:200, recomputed on load) else identity.
//
// Persistent, warp-specialised, one CTA per SM, molecule-aligned tiles of <=128 dst-sorted edge rows:
//   warp 0      TMA producer: H tile (5 boxes of 128 rows x 64 cols, SWIZZLE_128B) -> one shared-memory tile, handed
//               over slab by slab (box s of the next tile is loaded when the message warps have left slab s)
//   warp 1      TMA producer: W_h stages (pre-packed smem images, cp.async.bulk): an 80-column output chunk x one
//               k pass (slabs {0,1,2} | {3,4}), 2-stage ring of 30 KB
//   warps 2, 3  no role (warpgroup 0 runs at a reduced register budget, step_fused_kernel.cuh)
//   warps 4-11  two warpgroups, tile rows [0, 64) / [64, 128): wgmma m64n80k16, D (registers, fp32) = A (smem, bf16)
//               . W_h^T (smem), chunk by chunk, then the epilogue from registers: + H_0 + bias -> tau -> bf16 -> HBM
//               (the H_0 words of the next chunk are requested before each epilogue)
//   warps 12-19 message: thread = row e': sums the sibling rows of e' (same destination atom) out of the
//               shared-memory tile and writes the bf16 result row into the shared-memory A operand tile;
//               optionally also to HBM (M_out / G_out, one 32-byte sector per thread) for the W_h gradient
//
// The same kernel runs the autograd mirror of the step (MODE_BWD_*, dmpnn_bond_step_bwd_fused_bf16):
//   dOut = ((S.P) dZ) . W_h [* tau'(Y)]  -- the message warps read the sibling rows through a tile-local rev() table,
//   W is the packed W_h^T, the epilogue writes row e' itself and multiplies by tau' of Y.
//
// Algorithmic HBM bytes per step: read H_prev + H_0, write H_next = 3*E*h*2 (2*E*h*2 when first_step,
// H_prev == H_0 comes from L2 the second time); W_h (<=190 KB) is L2-resident.
#include "step_fused_kernel.cuh"

namespace dmpnn {
namespace fused {

// ---- weight packing: W (f32, N x K) -> bf16 stage images in consumption order ----------------
// image = for each 80-row output chunk c, for each 64-wide k slab s: a (rows_c x 128 B) block in the
// K-major SWIZZLE_128B layout the tensor core reads; one cp.async.bulk per block lands it in smem.  Inside a chunk, image
// row j holds W row 80 c + acc_out_col(j, rows_c) (tc_common.cuh), so that the epilogue's fragments are column runs.
struct PackGeom {
  int N, K, hpN, hpK, nslab, nchunks;
};
__host__ __device__ inline PackGeom pack_geom(int64_t N, int64_t K) {
  PackGeom g;
  g.N = (int)N; g.K = (int)K;
  g.hpN = (int)((N + 15) / 16 * 16);
  g.hpK = (int)((K + 15) / 16 * 16);
  g.nslab = (g.hpK + 63) / 64;
  g.nchunks = (g.hpN + kChunkN - 1) / kChunkN;
  return g;
}

__global__ void k_pack_weight(const float* __restrict__ W, int64_t ldw, PackGeom g, __nv_bfloat16* __restrict__ out) {
  const int c = blockIdx.x / kChunkN;              // image row blockIdx.x (0 .. hpN-1) = row nl of chunk c
  const int nl = blockIdx.x - c * kChunkN;
  const int rows = min(kChunkN, g.hpN - c * kChunkN);
  const int n = c * kChunkN + tc::acc_out_col(nl, rows);   // the W row (output column) it holds; zero at n >= N
  for (int k = threadIdx.x; k < g.nslab * 64; k += blockDim.x) {
    const int s = k >> 6, kl = k & 63;
    const size_t blk = (size_t)c * kChunkN * g.nslab * 128 + (size_t)s * rows * 128;
    const size_t off = blk + (size_t)(nl >> 3) * 1024 + (nl & 7) * 128 + (((kl >> 3) ^ (nl & 7)) << 4) + (kl & 7) * 2;
    const float v = (n < g.N && k < g.K) ? W[(int64_t)n * ldw + k] : 0.f;
    out[off >> 1] = __float2bfloat16_rn(v);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static bool encode_rows_map(EncodeTiledFn enc, CUtensorMap* tmap, const void* base, int hp, int64_t rows, int64_t ld) {
  cuuint64_t gdim[2] = {(cuuint64_t)hp, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)kTileM};
  cuuint32_t estr[2] = {1, 1};
  return enc(tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace fused
}  // namespace dmpnn

using namespace dmpnn;
using namespace dmpnn::fused;

static unsigned long long* g_trace = nullptr;
static int g_trace_tiles = 0;
extern "C" int dmpnn_set_trace_buffer(void* dev_ptr, int64_t n_tiles) {
  g_trace = (unsigned long long*)dev_ptr;
  g_trace_tiles = dev_ptr ? (int)n_tiles : 0;
  return 0;
}

extern "C" int dmpnn_pack_weight_bf16_bytes(int64_t N, int64_t K, size_t* bytes) {
  DMPNN_CHECK_ARG(bytes && N > 0 && K > 0 && N <= kMaxHp && K <= kMaxHp, "pack_weight_bf16: need 0 < N,K <= %d", kMaxHp);
  PackGeom g = pack_geom(N, K);
  *bytes = (size_t)g.nslab * g.hpN * 128;
  return 0;
}

extern "C" int dmpnn_pack_weight_bf16(const float* W, int64_t ldw, int64_t N, int64_t K, void* Wpk, void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  DMPNN_CHECK_ARG(W && Wpk && N > 0 && K > 0 && N <= kMaxHp && K <= kMaxHp, "pack_weight_bf16: bad args");
  PackGeom g = pack_geom(N, K);
  k_pack_weight<<<g.hpN, 128, 0, st>>>(W, ldw, g, (__nv_bfloat16*)Wpk);
  DMPNN_CHECK_LAUNCH("pack_weight_bf16", 1);
  return 0;
}

static int launch_step(const char* what, const void* H_prev, const void* H_0, void* H_next, int64_t ld, int64_t n_rows_alloc,
                       int64_t h, const void* Wpk, const float* bias, const int32_t* rowptr, const int32_t* rev_row,
                       const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles, int act, float act_param,
                       int first_step, int mode, void* gather_out, const void* add0, const void* add1,
                       const int8_t* work_flag, const int32_t* n_work_dev, const int32_t* dst_row, const uint16_t* drop_bits,
                       float drop_scale, cudaStream_t st, const int32_t* nbr_row = nullptr) {
  const bool atom = nbr_row != nullptr;     // atom-granular step: rows are atoms, tile_row_ptr / tile_atom_ptr = atom / edge offsets
  DMPNN_CHECK_ARG(drop_bits == nullptr || mode == MODE_FWD, "%s: keep bits apply to the forward step", what);
  DMPNN_CHECK_ARG(atom || ((work_flag == nullptr) == (n_work_dev == nullptr) && (work_flag == nullptr || dst_row != nullptr)),
                  "%s: work_flag, n_work_dev and dst_row come together (dmpnn_work_table_build)", what);
  DMPNN_CHECK_ARG(!atom || (work_flag == nullptr && drop_bits == nullptr), "%s: no windows / keep bits in the atom step", what);
  DMPNN_CHECK_ARG(drop_bits == nullptr || (drop_scale > 0.f && isfinite(drop_scale) &&
                                           (reinterpret_cast<uintptr_t>(drop_bits) & 1) == 0),
                  "%s: keep bits need a finite drop_scale > 0 and a 2-byte aligned array", what);
  DMPNN_CHECK_ARG((add0 == nullptr && add1 == nullptr) || (mode == MODE_BWD_LAST && add0 != nullptr),
                  "%s: addends need y_is_preact (and add0 before add1)", what);
  DMPNN_CHECK_ARG(((reinterpret_cast<uintptr_t>(add0) | reinterpret_cast<uintptr_t>(add1)) & 15) == 0,
                  "%s: addends must be 16-byte aligned", what);
  DMPNN_CHECK_ARG(add0 != H_next && add1 != H_next, "%s: an addend may not alias the output", what);
  DMPNN_CHECK_ARG(gather_out == nullptr || mode != MODE_FWD || first_step,
                  "%s: the gathered operand can only be written by the first forward step", what);
  DMPNN_CHECK_ARG(gather_out == nullptr || ((reinterpret_cast<uintptr_t>(gather_out) & 31) == 0 && ld % 16 == 0),
                  "%s: gather output needs a 32-byte aligned base and ld %% 16 == 0", what);
  DMPNN_CHECK_ARG(H_prev && H_next && Wpk && rowptr && (rev_row || atom) && tile_row_ptr && tile_atom_ptr && (H_0 || mode == MODE_BWD_COPY),
                  "%s: null pointer", what);
  DMPNN_CHECK_ARG(h > 0 && h <= kMaxHp, "%s: h=%lld unsupported (max %d)", what, (long long)h, kMaxHp);
  const int hp = (int)((h + 15) / 16 * 16);
  DMPNN_CHECK_ARG(ld >= hp && ld % 16 == 0, "%s: ld=%lld must be >= %d and a multiple of 16 (rows are written as 32-byte sectors)", what, (long long)ld, hp);
  DMPNN_CHECK_ARG(n_rows_alloc > 0 && n_tiles >= 0, "%s: bad sizes", what);
  DMPNN_CHECK_ARG(act >= DMPNN_ACT_NONE && act <= DMPNN_ACT_ELU, "%s: bad activation %d", what, act);
  DMPNN_CHECK_ARG((reinterpret_cast<uintptr_t>(H_prev) & 15) == 0 && (reinterpret_cast<uintptr_t>(H_0) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(H_next) & 31) == 0 && (reinterpret_cast<uintptr_t>(Wpk) & 15) == 0,
                  "%s: inputs must be 16-byte aligned, the output 32-byte aligned", what);
  DMPNN_CHECK_ARG(H_next != H_prev && H_next != H_0, "%s: in-place update not supported", what);
  if (n_tiles == 0) return 0;
  EncodeTiledFn enc = get_encode_fn();
  DMPNN_CHECK_ARG(enc != nullptr, "%s: cuTensorMapEncodeTiled not available from the driver", what);
  CUtensorMap mH;
  DMPNN_CHECK_ARG(encode_rows_map(enc, &mH, H_prev, hp, n_rows_alloc, ld), "%s: cuTensorMapEncodeTiled failed", what);

  PackGeom g = pack_geom(h, h);
  Params p;
  p.H0 = (const __nv_bfloat16*)H_0;
  p.Hn = (__nv_bfloat16*)H_next;
  p.G = (__nv_bfloat16*)gather_out;
  p.add0 = (const __nv_bfloat16*)add0;
  p.add1 = (const __nv_bfloat16*)add1;
  p.ld = ld;
  p.Wpk = (const uint8_t*)Wpk;
  p.bias = bias;
  p.rowptr = rowptr;
  p.rev_row = rev_row;
  p.tile_row_ptr = tile_row_ptr;
  p.tile_atom_ptr = tile_atom_ptr;
  p.work_flag = work_flag;
  p.n_work_dev = n_work_dev;
  p.dst_row = dst_row;
  p.Hprev = (const __nv_bfloat16*)H_prev;
  p.nbr_row = nbr_row;
  p.drop_bits = drop_bits;
  p.drop_scale = drop_scale;
  p.n_tiles = (int)n_tiles;
  p.h = (int)h;
  p.hp = hp;
  p.nslab = g.nslab;
  p.nchunks = g.nchunks;
  p.act_param = act_param;
  {
    static int exp_flags = -1;
    if (exp_flags < 0) { const char* e = getenv("DMPNN_EXP"); exp_flags = e ? atoi(e) : 0; }
    p.exp_flags = exp_flags;
  }
  p.trace = g_trace;
  p.trace_tiles = g_trace_tiles;
  {
    const char* tb = g_trace ? getenv("DMPNN_TRACE_BLOCK") : nullptr;
    p.trace_block = tb ? atoi(tb) : 0;
  }

  static int sm_count = 0;
  if (!sm_count) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
  }
  const int grid = (work_flag != nullptr || n_work_dev != nullptr || n_tiles >= sm_count) ? sm_count : (int)n_tiles;
  const bool far = work_flag != nullptr;
  cudaError_t e;
  if (atom)
    e = mode == MODE_FWD ? dispatch_fwd<false, true>(act, first_step != 0, bias != nullptr, false, grid, st, mH, p)
                         : dispatch_bwd<false, true>(mode, act, grid, st, mH, p);
  else if (mode == MODE_FWD)
    e = far ? dispatch_fwd<true>(act, first_step != 0, bias != nullptr, drop_bits != nullptr, grid, st, mH, p)
            : dispatch_fwd<false>(act, first_step != 0, bias != nullptr, drop_bits != nullptr, grid, st, mH, p);
  else
    e = far ? dispatch_bwd<true>(mode, act, grid, st, mH, p) : dispatch_bwd<false>(mode, act, grid, st, mH, p);
  DMPNN_CHECK_ARG(e == cudaSuccess, "%s: cannot configure %d B dynamic smem: %s", what, kSmemAlloc, cudaGetErrorString(e));
  DMPNN_CHECK_LAUNCH(what, 1);
  return 0;
}

extern "C" int dmpnn_bond_step_fused_bf16(const void* H_prev, const void* H_0, void* H_next, int64_t ld,
                                          int64_t n_rows_alloc, int64_t h, const void* Wpk, const float* bias,
                                          const int32_t* rowptr, const int32_t* rev_row, const int32_t* tile_row_ptr,
                                          const int32_t* tile_atom_ptr, int64_t n_tiles, int act, float act_param,
                                          int first_step, void* M_out, const int8_t* work_flag, const int32_t* n_work_dev,
                                          const int32_t* dst_row, const void* drop_bits, float drop_scale, void* stream_) {
  return launch_step("bond_step_fused", H_prev, H_0, H_next, ld, n_rows_alloc, h, Wpk, bias, rowptr, rev_row, tile_row_ptr,
                     tile_atom_ptr, n_tiles, act, act_param, first_step, MODE_FWD, M_out, nullptr, nullptr, work_flag, n_work_dev,
                     dst_row, (const uint16_t*)drop_bits, drop_scale, (cudaStream_t)stream_);
}

extern "C" int dmpnn_bond_step_bwd_fused_bf16(const void* dZ, const void* Yact, void* dOut, int64_t ld, int64_t n_rows_alloc,
                                              int64_t h, const void* WpkT, const int32_t* rowptr, const int32_t* rev_row,
                                              const int32_t* tile_row_ptr, const int32_t* tile_atom_ptr, int64_t n_tiles,
                                              int act, float act_param, int y_is_preact, const void* add0,
                                              const void* add1, void* G_out, const int8_t* work_flag,
                                              const int32_t* n_work_dev, const int32_t* dst_row, void* stream_) {
  DMPNN_CHECK_ARG(!y_is_preact || Yact, "bond_step_bwd_fused: y_is_preact needs Yact");
  return launch_step("bond_step_bwd_fused", dZ, Yact, dOut, ld, n_rows_alloc, h, WpkT, nullptr, rowptr, rev_row, tile_row_ptr,
                     tile_atom_ptr, n_tiles, act, act_param, 0,
                     Yact ? (y_is_preact ? MODE_BWD_LAST : MODE_BWD_MASK) : MODE_BWD_COPY, G_out, add0, add1, work_flag,
                     n_work_dev, dst_row, nullptr, 1.f, (cudaStream_t)stream_);
}

// ---- atom-granular step (AtomMessagePassing restated on atoms; ATOM instantiations of the same kernel) -------------------
extern "C" int dmpnn_atom_step_fused_bf16(const void* H_prev, const void* H_0, void* H_next, int64_t ld, int64_t n_rows_alloc,
                                          int64_t h, const void* Wpk, const float* bias, const int32_t* rowptr,
                                          const int32_t* nbr_row, const int32_t* tile_atom_ptr, const int32_t* tile_edge_ptr,
                                          const int32_t* n_tiles_dev, int64_t n_tiles_max, int act, float act_param,
                                          int first_step, void* N_out, void* stream_) {
  DMPNN_CHECK_ARG(nbr_row && n_tiles_dev, "atom_step_fused: null pointer");
  return launch_step("atom_step_fused", H_prev, H_0, H_next, ld, n_rows_alloc, h, Wpk, bias, rowptr, nullptr, tile_atom_ptr,
                     tile_edge_ptr, n_tiles_max, act, act_param, first_step, MODE_FWD, N_out, nullptr, nullptr, nullptr, n_tiles_dev,
                     nullptr, nullptr, 1.f, (cudaStream_t)stream_, nbr_row);
}

extern "C" int dmpnn_atom_step_bwd_fused_bf16(const void* dZ, const void* Yact, void* dOut, int64_t ld, int64_t n_rows_alloc,
                                              int64_t h, const void* WpkT, const int32_t* rowptr, const int32_t* nbr_row,
                                              const int32_t* tile_atom_ptr, const int32_t* tile_edge_ptr,
                                              const int32_t* n_tiles_dev, int64_t n_tiles_max, int act, float act_param,
                                              int y_is_preact, const void* add0, const void* add1, void* G_out, void* stream_) {
  DMPNN_CHECK_ARG(nbr_row && n_tiles_dev, "atom_step_bwd_fused: null pointer");
  DMPNN_CHECK_ARG(!y_is_preact || Yact, "atom_step_bwd_fused: y_is_preact needs Yact");
  return launch_step("atom_step_bwd_fused", dZ, Yact, dOut, ld, n_rows_alloc, h, WpkT, nullptr, rowptr, nullptr, tile_atom_ptr,
                     tile_edge_ptr, n_tiles_max, act, act_param, 0,
                     Yact ? (y_is_preact ? MODE_BWD_LAST : MODE_BWD_MASK) : MODE_BWD_COPY, G_out, add0, add1, nullptr, n_tiles_dev,
                     nullptr, nullptr, 1.f, (cudaStream_t)stream_, nbr_row);
}
