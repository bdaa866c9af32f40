// The fused depth-step kernel of csrc/step_fused.cu (see there for the description), as a template: its ~100 instantiations
// (activation x first step x bias x autograd-mirror mode x {windows of oversized molecules} x {dropout in the epilogue}) are
// compiled in six translation units in parallel (step_fused_{fwd,bwd,far_fwd,far_bwd,atom_fwd,atom_bwd}.cu).
#pragma once
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace dmpnn {
namespace fused {

constexpr int kTileM = 128;
constexpr int kSlabBytes = kTileM * 128;        // one 64-column K slab of a 128-row tile: 16 KB
constexpr int kMaxSlabs = 5;                    // hp <= 320
constexpr int kABufBytes = kMaxSlabs * kSlabBytes;
constexpr int kChunkN = 80;                     // W stage / accumulator chunk = 80 output features (the wgmma N)
constexpr int kMaxChunks = 4;
// A W stage = an 80-column chunk x up to kWHalfSlabs k slabs; the A operand tile is handed over in k passes of that many
// slabs ({0,1,2} | {3,4}).
constexpr int kWHalfSlabs = 3;
constexpr int kMaxPasses = (kMaxSlabs + kWHalfSlabs - 1) / kWHalfSlabs;   // 2
constexpr int kWStageBytes = kWHalfSlabs * kChunkN * 128;   // 30 KB
constexpr int kWStages = 2;
// Timing experiments (tc::kExp builds; DMPNN_EXP selects at run time; results are wrong by construction): 32768 epilogue
// skips its global stores, 65536 message warps skip their shared-memory gathers, 131072 message warps skip the A operand
// stores, 262144 the MMA warpgroups issue no MMA.
constexpr int kThreads = 640;
constexpr int kSWarps = 8;          // message warps (12..19)
constexpr int kMmaThreads = 256;    // two MMA + epilogue warpgroups (warps 4..7, 8..11)
// Registers per thread of each role (setmaxnreg at the top of its branch).  640 threads at one CTA per SM are launched with
// 96 each; the single-lane producer warps (warpgroup 0) and the message warps (warpgroups 3, 4) hand theirs to the MMA
// warpgroups, whose epilogue holds the next chunk's operand words next to the accumulator (up to 125 registers; at 96 it
// spills, DESIGN.md 4.1).  The budgets fill the launch's 640 x 96: kRegsProducer + 2 kRegsMsg + 2 kRegsMma = 5 x 96.
constexpr int kRegsProducer = 32;
constexpr int kRegsMsg = 88;
constexpr int kRegsMma = 136;
static_assert(kRegsProducer + 2 * kRegsMsg + 2 * kRegsMma <= 5 * 96, "register budgets exceed the launch's 640 x 96");
constexpr int kMaxHp = 304;

struct Params {
  const __nv_bfloat16* H0;
  __nv_bfloat16* Hn;
  const __nv_bfloat16* add0;   // MODE_BWD_LAST: optional addends (same ld), summed in the copy-out
  const __nv_bfloat16* add1;
  __nv_bfloat16* G;   // optional: the gathered A operand rows (M^1 forward / (S.P)dZ backward) for the W_h gradient
  int64_t ld;
  const uint8_t* Wpk;
  const float* bias;
  const int32_t* rowptr;
  const int32_t* rev_row;
  const int32_t* tile_row_ptr;   // work items: the layout's tiles, or (work_flag != nullptr) the work table in which
  const int32_t* tile_atom_ptr;  // every tile of more than 128 rows is cut into 128-row windows
  const int8_t* work_flag;       // nullable; 1 = window of a molecule of more than 128 rows or atoms: siblings / rev() partners
                                 // may lie outside, and its row-pointer slice would not fit s_rowptr's 132 words
  const int32_t* n_work_dev;     // nullable; number of work items when the work table is in use (device scalar)
  const int32_t* dst_row;        // destination atom of every row (needed by the non-local windows only)
  const __nv_bfloat16* Hprev;    // the H tile's matrix again, for the non-local windows' global gathers
  const int32_t* nbr_row;        // ATOM kernels: source atom of every dst-sorted edge row (the layout's src_row); rows are
                                 // ATOMS there, `tile_row_ptr` / `tile_atom_ptr` hold the atom / edge offsets of the atom tiles
  const uint16_t* drop_bits;     // nullable (forward): 16 keep bits per (row, 16-column block), dmpnn_dropout_bits
  float drop_scale;              // 1 / (1 - p)
  int n_tiles, h, hp, nslab, nchunks;
  float act_param;
  int exp_flags;  // timing experiments only (DMPNN_EXP env var); 0 in production
  unsigned long long* trace;  // optional per-tile phase timestamps of block 0 (dmpnn_set_trace_buffer)
  int trace_tiles;
  int trace_block;   // which CTA records (DMPNN_TRACE_BLOCK, default 0)
};

// shared memory carve-up (after 1024 B alignment)
constexpr int kOffA = 0;                                     // raw H tile (single buffer, read-only for the SMs)
constexpr int kOffAop = kABufBytes;                          // A operand tile written by the message warps: 81920
constexpr int kOffW = kOffAop + kABufBytes;                  // 163840
constexpr int kOffBar = kOffW + kWStages * kWStageBytes;     // 225280
constexpr int kNumBars = 24;
constexpr int kOffRowptr = kOffBar + kNumBars * 8;           // int32 [2][132]
constexpr int kOffRevl = kOffRowptr + 2 * 132 * 4;           // int16 [2][128]: tile-local rev() (backward mode)
constexpr int kOffBias = kOffRevl + 2 * 128 * 2;             // float [304]
constexpr int kNbCap = 512;                                  // ATOM kernels: staged neighbour entries per tile (else global look-ups)
constexpr int kOffNb = kOffBias + kMaxHp * 4;                // int16 [2][kNbCap]: tile-local neighbour rows of the atom tile
constexpr int kSmemBytes = kOffNb + 2 * kNbCap * 2;
constexpr int kSmemAlloc = kSmemBytes + 1024;
static_assert(kOffAop % 1024 == 0 && kOffW % 1024 == 0, "operand tiles must be 1024-byte aligned for SWIZZLE_128B");
static_assert(kSmemAlloc <= 232448, "exceeds the 227 KB per-CTA shared memory limit");

enum {
  B_AFULL = 0, B_AFREE = B_AFULL + kMaxSlabs,        // the H tile is handed over slab by slab (64 columns)
  B_AREADY = B_AFREE + kMaxSlabs, B_ATFREE = B_AREADY + kMaxPasses,
  B_WFULL = B_ATFREE + kMaxPasses, B_WFREE = B_WFULL + kWStages
};
static_assert(B_WFREE + kWStages <= kNumBars, "barrier table too small");
static_assert(kMaxSlabs == 5 && kMaxChunks <= 4, "barrier numbering assumes these");

using namespace dmpnn::tc;

// Every bounded wait of this kernel is tc::mbar_wait_trap: it makes no call, which would serialise the wgmmas (C7510).

constexpr int kTraceEvents = 16;
__device__ __forceinline__ void trace_ev(const Params& p, int it, int ev) {
  if (p.trace && blockIdx.x == p.trace_block && it < p.trace_tiles) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    p.trace[it * kTraceEvents + ev] = t;
  }
}

// ---------------------------------------------------------------------------------------------
// MODE 0: forward step (message of H, epilogue tau(H_0 + bias + acc) written to row e')
// MODE 1: autograd mirror, masked:  A row e' = sum of dZ[rev(x)] over the siblings x of e';  out[e'] = acc * tau'(Y[e'])
// MODE 2: autograd mirror, plain:   same gather;  out[e'] = acc
// MODE_BWD_LAST: mask from the PRE-activation (Y = H_0) and up to two row-aligned addends summed into the output:
// the t = 1 step then produces dH_0 = dZ^{T-1} + ... + dZ^1 + dH^0 * tau'(H_0) directly.
enum { MODE_FWD = 0, MODE_BWD_MASK = 1, MODE_BWD_COPY = 2, MODE_BWD_LAST = 3 };

// FAR: the launch's work table may hold windows of molecules larger than a tile (global gathers); DROP: keep bits in the
// forward epilogue.  Both are compile-time so that the common kernel (neither) carries none of their code.
// ATOM: the atom-granular step of AtomMessagePassing (mixins.py:25-30 restated on atoms, DESIGN.md 4.4): rows are atoms, a
// tile is a run of whole molecules with <= 128 atoms, and A row v = sum over the in-edges e of v of g(H[src(e)]) -- the neighbour
// rows are read from the same TMA-loaded tile through a staged tile-local neighbour table; the adjacency is symmetric (every bond
// is two directed edges), so the autograd mirror is the same gather applied to dZ.  Everything after the gather is shared.
template <int ACT, bool FIRST, bool HAS_BIAS, int MODE, bool FAR, bool DROP, bool ATOM = false>
__global__ void __launch_bounds__(kThreads, 1)
k_bond_step_fused(const __grid_constant__ CUtensorMap tmapH, Params p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment as an OFFSET from the shared-memory symbol (not through a uintptr_t round trip): the compiler keeps
  // the address space, so the row-pointer / rev() table look-ups of the message warps are LDS instead of generic LD.E
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t sA = sbase + kOffA, sAop = sbase + kOffAop, sW = sbase + kOffW, sBar = sbase + kOffBar;
  int32_t* s_rowptr = reinterpret_cast<int32_t*>(smem + kOffRowptr);
  int16_t* s_revl = reinterpret_cast<int16_t*>(smem + kOffRevl);
  float* s_bias = reinterpret_cast<float*>(smem + kOffBias);
  int16_t* s_nb = reinterpret_cast<int16_t*>(smem + kOffNb);
  // the role dispatch below branches on `warp`: broadcast from lane 0 so that ptxas sees a warp-uniform value (a role taken
  // from threadIdx.x directly is a divergent path to the compiler, and it serialises the wgmma instructions inside it)
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  auto bar = [&](int i) { return sBar + 8u * (uint32_t)i; };

  if (threadIdx.x == 0) {
    for (int i = 0; i < kMaxSlabs; ++i) {
      mbar_init(bar(B_AFULL + i), 1);
      mbar_init(bar(B_AFREE + i), kSWarps * 32);  // every message thread is done reading this slab of the tile
    }
    for (int i = 0; i < kMaxPasses; ++i) {      // the A operand tile is handed over k pass by k pass (slabs {0,1,2} | {3,4})
      mbar_init(bar(B_AREADY + i), kSWarps * 32);   // message threads have written this k pass of their row
      mbar_init(bar(B_ATFREE + i), kMmaThreads);    // both warpgroups' MMAs have finished reading this k pass
    }
    for (int i = 0; i < kWStages; ++i) {
      mbar_init(bar(B_WFULL + i), 1);
      mbar_init(bar(B_WFREE + i), kMmaThreads);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < kMaxHp; i += kThreads) s_bias[i] = (p.bias && i < p.h) ? p.bias[i] : 0.f;
  __syncthreads();
  const int n_items = p.n_work_dev ? __ldg(p.n_work_dev) : p.n_tiles;   // work items of this launch (uniform over the grid)
  const int npass = (p.nslab + kWHalfSlabs - 1) / kWHalfSlabs;

  if (warp < 4) {
    setmaxnreg_dec<kRegsProducer>();
    if (warp == 0) {
      // ===================== TMA producer: H_prev tile -> shared memory (single buffer) =====================
      // No L2 prefetch of the next tile's rows (nor of its H_0 rows): both made the step slower on an H100 at h = 300
      // (DESIGN.md 7).  The H_0 prefetch had no barrier to pace it, so it ran through all of a CTA's tiles at the start of
      // the launch, far more rows than L2 holds.  Warps 2 and 3 have no role: an L2 prefetch of MODE_BWD_LAST's addends there
      // kept ptxas from giving the MMA warpgroups more than 96 registers (their epilogue spilled).
      int it = 0;
      int row_carry = (int)blockIdx.x < n_items ? __ldg(p.tile_row_ptr + blockIdx.x) : 0;   // the next tile's first row, loaded a tile ahead
      for (int t = blockIdx.x; t < n_items; t += gridDim.x, ++it) {
        const int row0 = row_carry;
        const int t2 = t + gridDim.x;
        if (t2 < n_items) row_carry = __ldg(p.tile_row_ptr + t2);
        // slab s of this tile is loaded as soon as the message warps have left slab s of the previous tile: the load
        // of the leading slabs overlaps the gather of the trailing ones (one shared-memory tile, no exposed latency)
        for (int s = 0; s < p.nslab; ++s) {
          mbar_wait_trap(bar(B_AFREE + s), (it & 1) ^ 1);
          if (elect_one()) {
            if (s == 0) trace_ev(p, it, 0);
            mbar_expect_tx(bar(B_AFULL + s), kSlabBytes);
            tma_load_2d(sA + s * kSlabBytes, &tmapH, bar(B_AFULL + s), s * 64, row0);
          }
          __syncwarp();
        }
      }
    } else if (warp == 1) {
      // ===================== TMA producer: W_h stages (pre-packed smem images) =====================
      // a stage = the W_h rows of one 80-column output chunk for k slabs {0,1,2} or {3,4} (contiguous in the image), in the
      // MMA warpgroups' order: chunk by chunk, both k passes of a chunk back to back
      uint32_t ws = 0;
      for (int t = blockIdx.x; t < n_items; t += gridDim.x) {
        for (int c = 0; c < p.nchunks; ++c)
          for (int half = 0; half < npass; ++half, ++ws) {
            const int s0 = half * kWHalfSlabs;
            const int ns = min(kWHalfSlabs, p.nslab - s0);
            const int nc = min(kChunkN, p.hp - c * kChunkN);
            const uint8_t* src = p.Wpk + (size_t)c * kChunkN * p.nslab * 128 + (size_t)s0 * nc * 128;
            const uint32_t bytes = (uint32_t)(ns * nc * 128);
            const uint32_t st = ws % kWStages, use = ws / kWStages;
            mbar_wait_trap(bar(B_WFREE + st), (use & 1) ^ 1);
            if (elect_one()) {
              if (p.exp_flags & 4096) {              // timing experiment: no W stream at all (stale shared memory, wrong results)
                mbar_arrive(bar(B_WFULL + st));
              } else {
                mbar_expect_tx(bar(B_WFULL + st), bytes);
                bulk_load(sW + st * kWStageBytes, src, bytes, bar(B_WFULL + st));
              }
            }
            __syncwarp();
          }
      }
    }
  } else if (warp < 12) {
    setmaxnreg_inc<kRegsMma>();
    // ===================== MMA + epilogue: warpgroup wg owns tile rows [64 wg, 64 wg + 64) ==========
    // D[64 x 80] (registers, fp32) = A (shared memory, written by the message warps) . W_h^T (W stage) per 80-column chunk;
    // the epilogue of a chunk runs from registers right after its last k pass.  The message warps build A row r as the
    // message of edge r itself (they gather through the tile-local rev() table), so accumulator row r is the update of
    // edge r: it needs H_0 row r (global memory, requested one chunk ahead, below) and produces output row r.
    // W rows past a chunk's last column may hold the next slab's rows or stale data: they only reach accumulator columns
    // that the epilogue never stores.
    const int wg = (warp - 4) >> 2;
    const int tt = threadIdx.x - 128 - wg * 128;
    const int rA = wg * 64 + acc_row0(tt), cl = acc_col0(tt);
    const int nj = p.hp >> 4;
    // ---- epilogue operands of one chunk.  The packed W_h image permutes the columns of every chunk (tc::acc_out_col): in each
    // 32-column group G this thread's accumulator blocks 4 G .. 4 G + 3 hold the 8 contiguous output columns from
    // acc_out_col(32 G + cl, nc) on, in a 16-column tail its blocks 4 G, 4 G + 1 hold 4 (acc_run_cols).  So each row and group
    // is one 16-byte (tail: 8-byte) load, and hv[h][b] is the operand word of accumulator block b of row rA + 8 h.
    constexpr int kGroups = (kChunkN + 31) / 32;   // two 32-column groups and a 16-column tail
    auto load_ops = [&](uint32_t (&hv)[2][kChunkN / 8], int row0, int nrows, int c) {
      const int nc = min(kChunkN, p.hp - c * kChunkN);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = rA + 8 * h;
        const __nv_bfloat16* yrow = p.H0 + (int64_t)(row0 + r) * p.ld + c * kChunkN;
#pragma unroll
        for (int G = 0; G < kGroups; ++G) {
          const int run = acc_run_cols(32 * G + cl, nc);
          uint4 v = make_uint4(0u, 0u, 0u, 0u);
          if (MODE != MODE_BWD_COPY && r < nrows) {
            const __nv_bfloat16* src = yrow + acc_out_col(32 * G + cl, nc);
            if (32 * G + 32 <= kChunkN && run == 8) {
              v = __ldg(reinterpret_cast<const uint4*>(src));
            } else if (run == 4) {
              const uint2 u = __ldg(reinterpret_cast<const uint2*>(src));
              v.x = u.x; v.y = u.y;
            }
          }
          const uint32_t vw[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int w = 0; w < 4; ++w)
            if (4 * G + w < kChunkN / 8) hv[h][4 * G + w] = vw[w];
        }
      }
    };
    // The operands are requested one chunk ahead: those of chunk c + 1 (at the last chunk: chunk 0 of this CTA's next work
    // item) before chunk c's epilogue, so that their latency hides under a whole epilogue.  hwv holds the current chunk's.
    uint32_t hwv[2][kChunkN / 8], hwn[2][kChunkN / 8];
    int row0 = 0, nrows = 0;
    if ((int)blockIdx.x < n_items) {
      row0 = __ldg(p.tile_row_ptr + blockIdx.x);
      nrows = __ldg(p.tile_row_ptr + blockIdx.x + 1) - row0;
      load_ops(hwv, row0, nrows, 0);
    }
    uint32_t ws = 0;
    int it = 0;
    for (int t = blockIdx.x; t < n_items; t += gridDim.x, ++it) {
      const int tn = t + gridDim.x;
      int row0n = 0, nrowsn = 0;                                         // next work item (nrowsn = 0: none)
      if (tn < n_items) {
        row0n = __ldg(p.tile_row_ptr + tn);
        nrowsn = __ldg(p.tile_row_ptr + tn + 1) - row0n;
      }
      uint32_t a_waited = 0;                                             // k passes of this tile's A already waited for
      for (int c = 0; c < p.nchunks; ++c) {
        float acc[40];
#pragma unroll
        for (int i = 0; i < 40; ++i) acc[i] = 0.f;
        const int nc = min(kChunkN, p.hp - c * kChunkN);
        // A W stage (and, in the last chunk, its k pass of the A tile) is released once the wgmma group that read it has
        // retired: the group of pass k stays in flight while pass k + 1 waits for its operands and issues (wait<1>)
        auto release = [&](uint32_t st, int half) {
          mbar_arrive(bar(B_WFREE + st));
          if (c == p.nchunks - 1) mbar_arrive(bar(B_ATFREE + half));
        };
        uint32_t st_prev = 0;
        for (int half = 0; half < npass; ++half, ++ws) {
          const int s0 = half * kWHalfSlabs;
          const int ns = min(kWHalfSlabs, p.nslab - s0);
          if (!((a_waited >> half) & 1u)) {
            a_waited |= 1u << half;
            mbar_wait_trap(bar(B_AREADY + half), it & 1);           // the message warps have written this k pass
            if (half == 0 && wg == 0 && tt == 0) trace_ev(p, it, 3);
          }
          const uint32_t st = ws % kWStages, usew = ws / kWStages;
          mbar_wait_trap(bar(B_WFULL + st), usew & 1);
          if (!(kExp && (p.exp_flags & 262144))) {
#pragma unroll
            for (int si = 0; si < kWHalfSlabs; ++si) {
              if (si >= ns) break;
              const int s = s0 + si;
              const uint64_t adesc = desc_sw128(sAop + (uint32_t)s * kSlabBytes + (uint32_t)wg * 8192u);
              const uint64_t bdesc = desc_sw128(sW + st * kWStageBytes + (uint32_t)(si * nc * 128));
              // k step = 16 bf16 = 32 B of each operand row.  Every slab is four k steps, the last one too: its columns
              // past hp are zero in the A operand tile (written once by the message warps) and in the packed W_h image, so
              // they add exact zeros.  A slab is then one straight run of wgmmas behind one fence (a run-time k count would
              // put a branch between wgmmas, and ptxas inserts a warpgroup.arrive in front of each of them: C7519).
              wgmma_fence();
#pragma unroll
              for (int kk = 0; kk < 4; ++kk) wgmma_bf16_n80(acc, adesc + (uint64_t)(2 * kk), bdesc + (uint64_t)(2 * kk), 1u);
              wgmma_commit();   // one group per slab: a commit after the slab loop would sit at a join ptxas guards (C7519)
            }
          }
          if (half > 0) {   // the previous pass's groups have retired once at most this pass's ns groups are in flight
            if (ns >= 3) wgmma_wait<3>();
            else if (ns == 2) wgmma_wait<2>();
            else wgmma_wait<1>();
            release(st_prev, half - 1);
          }
          st_prev = st;
        }
        if (c + 1 < p.nchunks) load_ops(hwn, row0, nrows, c + 1);
        else load_ops(hwn, row0n, nrowsn, 0);
        wgmma_wait<0>();
        acc_fence(acc);
        release(st_prev, npass - 1);
        if (c == 0 && tt == 0) trace_ev(p, it, 6 + wg);
        // ---- epilogue of chunk c: rows rA, rA + 8; per group G the run of columns 80 c + acc_out_col(32 G + cl, nc) + [0, run),
        // word w of which (columns n, n + 1) comes from accumulator block 4 G + w
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = rA + 8 * h;
          if (r >= nrows) continue;
          const int64_t grow = (int64_t)(row0 + r);
          __nv_bfloat16* orow = p.Hn + grow * p.ld;
#pragma unroll
          for (int G = 0; G < kGroups; ++G) {
            const int run = acc_run_cols(32 * G + cl, nc);   // 8, 4 or 0 (nc is a multiple of 16)
            if (run == 0) continue;
            const bool full = 32 * G + 32 <= kChunkN && run == 8;
            const int n0 = c * kChunkN + acc_out_col(32 * G + cl, nc);
            // MODE_BWD_LAST addends: 8-byte loads, two words of each addend at a time (whole 16-byte runs of both addends
            // next to the preloaded operands spill at 96 registers)
            uint2 aw = make_uint2(0u, 0u), bw = make_uint2(0u, 0u);
            // keep bits of the run (it lies inside one 16-column block), shifted so that bit 2 w is column n0 + 2 w
            uint32_t kb = 0u;
            if constexpr (MODE == MODE_FWD && DROP) kb = (uint32_t)__ldg(p.drop_bits + grow * nj + (n0 >> 4)) >> (n0 & 15);
            uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int w = 0; w < 4; ++w) {
              const int b = 4 * G + w;
              if (b >= kChunkN / 8 || 2 * w >= run) break;
              const int n = n0 + 2 * w;
              const float v0 = acc[4 * b + 2 * h], v1 = acc[4 * b + 2 * h + 1];
              if constexpr (MODE == MODE_BWD_COPY) {          // dOut = (S.P)(dZ) . W_h
                o[w] = pack_bf2(v0, v1);
              } else {
                const uint32_t hw = hwv[h][b];
                if constexpr (MODE == MODE_BWD_MASK || MODE == MODE_BWD_LAST) {
                  // ... * tau'(.): from the activation output the row came from, or (LAST) from the pre-activation H_0
                  const float g0 = MODE == MODE_BWD_LAST ? act_grad_from_pre(ACT, p.act_param, bf_lo(hw))
                                                         : act_grad_from_out(ACT, p.act_param, bf_lo(hw));
                  const float g1 = MODE == MODE_BWD_LAST ? act_grad_from_pre(ACT, p.act_param, bf_hi(hw))
                                                         : act_grad_from_out(ACT, p.act_param, bf_hi(hw));
                  float z0 = v0 * g0, z1 = v1 * g1;
                  if (MODE == MODE_BWD_LAST && p.add0 != nullptr) {
                    // dH_0 = (this step's masked gradient) + the earlier steps' dZ rows
                    if ((w & 1) == 0) {
                      aw = __ldg(reinterpret_cast<const uint2*>(p.add0 + grow * p.ld + n));
                      bw = p.add1 != nullptr ? __ldg(reinterpret_cast<const uint2*>(p.add1 + grow * p.ld + n)) : make_uint2(0u, 0u);
                    }
                    const uint32_t a = (w & 1) ? aw.y : aw.x, bb = (w & 1) ? bw.y : bw.x;
                    z0 += bf_lo(a) + bf_lo(bb);
                    z1 += bf_hi(a) + bf_hi(bb);
                  }
                  o[w] = pack_bf2(z0, z1);
                } else {
                  float z0 = v0 + bf_lo(hw);
                  float z1 = v1 + bf_hi(hw);
                  if constexpr (HAS_BIAS) {
                    z0 += s_bias[n];
                    z1 += s_bias[n + 1];
                  }
                  if constexpr (MODE == MODE_FWD && DROP) {
                    // nn.Dropout of base.py:139 in the epilogue: tau in f32, keep bit, exact f32 scale 1 / (1 - p), one rounding
                    z0 = ((kb >> (2 * w)) & 1u) ? act_t<ACT>(p.act_param, z0) * p.drop_scale : 0.f;
                    z1 = ((kb >> (2 * w + 1)) & 1u) ? act_t<ACT>(p.act_param, z1) * p.drop_scale : 0.f;
                    o[w] = pack_bf2(z0, z1);
                  } else if constexpr (ACT == DMPNN_ACT_RELU) {
                    o[w] = act_word<ACT>(pack_bf2(z0, z1), 0.f);  // max after rounding == rounding after max
                  } else {
                    o[w] = pack_bf2(act_t<ACT>(p.act_param, z0), act_t<ACT>(p.act_param, z1));
                  }
                }
              }
            }
            if (!(kExp && (p.exp_flags & 32768))) {
              if (full) *reinterpret_cast<uint4*>(orow + n0) = make_uint4(o[0], o[1], o[2], o[3]);
              else *reinterpret_cast<uint2*>(orow + n0) = make_uint2(o[0], o[1]);
            }
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int b = 0; b < kChunkN / 8; ++b) hwv[h][b] = hwn[h][b];
      }
      if (tt == 0) trace_ev(p, it, 8 + wg);
      row0 = row0n;
      nrows = nrowsn;
    }
  } else {
    setmaxnreg_dec<kRegsMsg>();
    // ===================== message (warps 12..19): thread == tile row ==================
    // A row e' of the GEMM is M[rev(e')] = sum of the OTHER in-edge states of e's destination atom
    // (mixins.py:11-18).  Each thread reads the <= 3 sibling rows of its row from the TMA-loaded,
    // 128B-swizzled shared-memory tile (read-only), adds them in packed bf16x2 (<= 2 roundings; f32 for
    // in-degree > 4) and writes its bf16 row into the A operand tile (K-major SWIZZLE_128B, the layout wgmma reads).
    const int sq = warp & 3;                 // 32-row quarter of the tile
    const int shalf = (warp - 12) >> 2;      // two warps per quarter alternate over the 16-column blocks
    const int r = sq * 32 + lane;            // tile row
    const int tS = threadIdx.x - 384;        // 0..255
    const int nj = p.hp >> 4;
    constexpr bool kCanEmit = FIRST || MODE != MODE_FWD;   // variants that may also write the gathered operand out
    constexpr bool kNeedRev = !ATOM;   // every bond mode gathers through the tile-local rev() table
    int it = 0;
    int t = blockIdx.x;
    // ATOM kernels: `atom0` / `natoms` are the first EDGE row and the edge count of the atom tile (its CSR slice), rows are atoms
    int row0 = 0, atom0 = 0, natoms = 0, nr = 0;
    bool far = false;                        // this work item is a window of an oversized molecule (work_flag)
    if (t < n_items) {
      row0 = __ldg(p.tile_row_ptr + t);
      nr = __ldg(p.tile_row_ptr + t + 1) - row0;
      atom0 = __ldg(p.tile_atom_ptr + t);
      natoms = __ldg(p.tile_atom_ptr + t + 1) - atom0;
      far = FAR && p.work_flag != nullptr && __ldg(p.work_flag + t) != 0;
      if (far) natoms = 0;
      if (ATOM) {
        if (tS <= nr) s_rowptr[tS] = __ldg(p.rowptr + row0 + tS) - atom0;
#pragma unroll
        for (int k = 0; k < kNbCap / 256; ++k) {
          const int i = tS + 256 * k;
          if (i < natoms) s_nb[i] = (int16_t)(__ldg(p.nbr_row + atom0 + i) - row0);
        }
      } else if (tS <= natoms) s_rowptr[tS] = __ldg(p.rowptr + atom0 + tS) - row0;
      if (kNeedRev && tS < 128) {
        s_revl[tS] = (int16_t)(tS < nr ? __ldg(p.rev_row + row0 + tS) - row0 : tS);
      }
    }
    // scalars of the tile after the current one (see the metadata pipeline below)
    int nx_row0 = 0, nx_atom0 = 0, nx_natoms = 0, nx_nr = 0;
    bool nx_far = false;
    if (t + (int)gridDim.x < n_items) {
      const int t1 = t + gridDim.x;
      nx_row0 = __ldg(p.tile_row_ptr + t1);
      nx_nr = __ldg(p.tile_row_ptr + t1 + 1) - nx_row0;
      nx_atom0 = __ldg(p.tile_atom_ptr + t1);
      nx_natoms = __ldg(p.tile_atom_ptr + t1 + 1) - nx_atom0;
      nx_far = FAR && p.work_flag != nullptr && __ldg(p.work_flag + t1) != 0;
      if (nx_far) nx_natoms = 0;
    }
    // A operand columns [hp, 64 nslab) -- the last slab's k steps past hp, which the MMAs multiply with the zero columns of the
    // packed W_h image -- are zeroed once here and never written again (published with the first k pass below)
    for (int j = nj + shalf; j < p.nslab * 4; j += 2) {
      const uint32_t ab = sAop + (uint32_t)(j >> 2) * kSlabBytes;
      sts128(ab + sw128_off(r, 2 * (j & 3)), make_uint4(0, 0, 0, 0));
      sts128(ab + sw128_off(r, 2 * (j & 3) + 1), make_uint4(0, 0, 0, 0));
    }
    for (; t < n_items; t += gridDim.x, ++it) {
      const int b = it & 1;
      const int32_t* rp = s_rowptr + b * 132;
      const int16_t* rvl = s_revl + b * 128;
      const int16_t* nbl = s_nb + b * kNbCap;
      // Metadata pipeline, two tiles deep: the SCALARS of the next tile (row / atom offsets: first-level loads) were loaded
      // one iteration ago, so the dependent second-level loads (its row-pointer slice and rev() rows) issue here without
      // waiting for them; the scalars of the tile after that are requested now.  (One-deep, the address dependency stalled
      // every message warp for an L2 round trip at the top of every tile.)
      const int tn = t + gridDim.x;
      const int row0n = nx_row0, atom0n = nx_atom0, natomsn = nx_natoms, nrn = nx_nr;
      const bool farn = nx_far;
      int rpn = 0;
      int nbn[kNbCap / 256];
      if (ATOM) {
        if (tn < n_items && tS <= nrn) rpn = __ldg(p.rowptr + row0n + tS) - atom0n;
#pragma unroll
        for (int k = 0; k < kNbCap / 256; ++k) {
          const int i = tS + 256 * k;
          nbn[k] = (tn < n_items && i < natomsn) ? __ldg(p.nbr_row + atom0n + i) - row0n : 0;
        }
      } else if (tn < n_items && tS <= natomsn) rpn = __ldg(p.rowptr + atom0n + tS) - row0n;
      int rvn = tS;
      if (kNeedRev && tn < n_items && tS < 128 && tS < nrn) rvn = __ldg(p.rev_row + row0n + tS) - row0n;
      {
        const int tnn = tn + gridDim.x;
        if (tnn < n_items) {
          nx_row0 = __ldg(p.tile_row_ptr + tnn);
          nx_nr = __ldg(p.tile_row_ptr + tnn + 1) - nx_row0;
          nx_atom0 = __ldg(p.tile_atom_ptr + tnn);
          nx_natoms = __ldg(p.tile_atom_ptr + tnn + 1) - nx_atom0;
          nx_far = FAR && p.work_flag != nullptr && __ldg(p.work_flag + tnn) != 0;
          if (nx_far) nx_natoms = 0;
        }
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");   // rp[] and rvl[] of this tile are complete
      // Forward: A row r is the message of edge r ITSELF = sum over the in-edges of src(r) other than rev(r), i.e. the
      // siblings of rs = rev(r) inside rs's destination segment, read directly.  Autograd mirror: A row r = sum over the
      // siblings x of r of dZ[rev(x)].  Either way the row the epilogue produces from accumulator row r is output row r.
      // A window of a molecule with more than 128 rows ("far"): the segment of rs and the rows it needs may lie outside the
      // window, so everything is looked up in ABSOLUTE rows (rev_row / dst_row / rowptr) and gathered from global memory
      // (L2 hits: the molecule's other windows are in flight on neighbouring CTAs); the shared-memory tile is not read.
      const int wrows = (FAR && far) ? (__ldg(p.tile_row_ptr + t + 1) - row0) : 0;
      const bool rin = ATOM ? (r < nr) : ((FAR && far) ? (r < wrows) : (r < rp[natoms]));
      int rs = (!ATOM && MODE == MODE_FWD && rin && !(FAR && far)) ? (int)rvl[r] : r;
      // ATOM: neighbour k of row r = tile-local row nbl[rp[r] + k]; tiles with more edges than the staged table read the global one
      auto nb_at = [&](int i) -> int { return (natoms <= kNbCap) ? (int)nbl[i] : (int)(__ldg(p.nbr_row + atom0 + i) - row0); };
      // segment (atom) of row rs: largest a with rp[a] <= rs
      int g0 = 0, d = 0;
      const __nv_bfloat16* fsrc[3] = {p.Hprev, p.Hprev, p.Hprev};   // far: the (<= 3) sibling rows in global memory
      int g0a = 0, rsa = 0;                                          // far: absolute segment start / skipped row
      if (FAR && far && rin) {
        rsa = row0 + r;
        if (MODE == MODE_FWD) rsa = __ldg(p.rev_row + rsa);
        const int v = __ldg(p.dst_row + rsa);
        g0a = __ldg(p.rowptr + v);
        d = __ldg(p.rowptr + v + 1) - g0a;
      } else if (ATOM) {
        if (rin) { g0 = rp[r]; d = rp[r + 1] - g0; }
      } else if (rin) {
        int lo = 0, hi = natoms;          // invariant: rp[lo] <= rs < rp[hi]
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (rp[mid] <= rs) lo = mid; else hi = mid;
        }
        g0 = rp[lo];
        d = rp[lo + 1] - g0;
      }
      // up to three siblings (in-degree <= 4); slot k is row g0+k, skipping rs itself.  ATOM: up to three neighbours, all of them
      const int nsib = ATOM ? d : d - 1;  // rows summed into A row r
      uint32_t soff[3];
      int sxr[3];
      bool sval[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int x = g0 + k;
        if (!ATOM && x >= rs) ++x;
        sval[k] = (k < nsib) && nsib <= (ATOM ? 4 : 3);
        if (ATOM) x = sval[k] ? nb_at(x) : r;
        if (FAR && far) {
          int xa = g0a + k;
          if (xa >= rsa) ++xa;
          if (sval[k]) {
            if (MODE != MODE_FWD) xa = __ldg(p.rev_row + xa);
            fsrc[k] = p.Hprev + (int64_t)xa * p.ld;
          }
          x = r;
        }
        if (!sval[k]) x = r;               // harmless in-bounds address for the predicated-off slot
        if (!ATOM && MODE != MODE_FWD && !(FAR && far)) x = rvl[x];  // autograd mirror: the sibling contributes the row of its reverse edge
        soff[k] = (uint32_t)((x >> 3) * 1024 + (x & 7) * 128);
        sxr[k] = x & 7;
      }
      // ATOM: a fourth neighbour (sp3 centres) is added after the first three, into the same registers -- without it nearly every
      // warp holds one degree-4 atom and would run the f32 loop below next to the packed path
      uint32_t soff3 = 0;
      int sxr3 = 0;
      bool sval3 = false;
      if (ATOM && rin && d == 4) {
        const int x3 = nb_at(g0 + 3);
        sval3 = true;
        soff3 = (uint32_t)((x3 >> 3) * 1024 + (x3 & 7) * 128);
        sxr3 = x3 & 7;
      }
      __nv_bfloat16* gout = nullptr;
      if constexpr (kCanEmit) {
        if (p.G != nullptr && rin) gout = p.G + (int64_t)(row0 + r) * p.ld;
      }
      int cur_slab = -1;                              // slab whose AFULL this thread has waited for
      uint32_t left = (1u << p.nslab) - 1u;           // slabs this thread still has to release
      const int npass = (p.nslab + kWHalfSlabs - 1) / kWHalfSlabs;
      int cur_pass = 0;                               // k pass being written; earlier ones are published by this thread
      mbar_wait_trap(bar(B_ATFREE + 0), (it & 1) ^ 1);    // tensor core is done with the first k pass of the previous tile
      for (int j = shalf; j < nj; j += 2) {
        const int pj = (j >> 2) / kWHalfSlabs;
        if (pj != cur_pass) {                        // crossing into a later k pass: publish the finished ones, wait for the next
          fence_proxy_async();                       // A operand stores -> visible to wgmma (async proxy)
          for (int q = cur_pass; q < pj; ++q) mbar_arrive(bar(B_AREADY + q));
          cur_pass = pj;
          mbar_wait_trap(bar(B_ATFREE + pj), (it & 1) ^ 1);
        }
        if ((j >> 2) != cur_slab) {                   // entering a new 64-column slab of the H tile
          if (cur_slab >= 0) { mbar_arrive(bar(B_AFREE + cur_slab)); left &= ~(1u << cur_slab); }
          cur_slab = j >> 2;
          mbar_wait_trap(bar(B_AFULL + cur_slab), it & 1);
          if (tS == 0 && cur_slab == 0) trace_ev(p, it, 1);
        }
        const uint32_t sbase = sA + (uint32_t)(j >> 2) * kSlabBytes;
        const int c0 = 2 * (j & 3);
        uint32_t o[8];
        if (nsib <= (ATOM ? 4 : 3)) {
          uint4 u[3][2];
#pragma unroll
          for (int k = 0; k < 3; ++k) {
            // predicated: an absent sibling costs no shared-memory wavefront (tau(0) = 0 for every activation)
            u[k][0] = make_uint4(0, 0, 0, 0);
            u[k][1] = make_uint4(0, 0, 0, 0);
            if (sval[k] && !(kExp && (p.exp_flags & 65536))) {
              if (FAR && far) {
                const uint4* gp = reinterpret_cast<const uint4*>(fsrc[k] + j * 16);
                u[k][0] = g_load<ACT, FIRST>(gp, p.act_param);
                u[k][1] = g_load<ACT, FIRST>(gp + 1, p.act_param);
              } else {
                u[k][0] = s_load<ACT, FIRST>(sbase + soff[k] + (uint32_t)((c0 ^ sxr[k]) << 4), p.act_param);
                u[k][1] = s_load<ACT, FIRST>(sbase + soff[k] + (uint32_t)(((c0 + 1) ^ sxr[k]) << 4), p.act_param);
              }
            }
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const uint32_t w0[4] = {u[0][hh].x, u[0][hh].y, u[0][hh].z, u[0][hh].w};
            const uint32_t w1[4] = {u[1][hh].x, u[1][hh].y, u[1][hh].z, u[1][hh].w};
            const uint32_t w2[4] = {u[2][hh].x, u[2][hh].y, u[2][hh].z, u[2][hh].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const bf2 a0 = u2b(w0[q]), a1 = u2b(w1[q]), a2 = u2b(w2[q]);
              o[4 * hh + q] = b2u(__hadd2(__hadd2(a0, a1), a2));   // x + 0 is exact: <= 2 roundings for d <= 4
            }
          }
          if (ATOM && sval3) {
            const uint4 v0 = s_load<ACT, FIRST>(sbase + soff3 + (uint32_t)((c0 ^ sxr3) << 4), p.act_param);
            const uint4 v1 = s_load<ACT, FIRST>(sbase + soff3 + (uint32_t)(((c0 + 1) ^ sxr3) << 4), p.act_param);
            const uint32_t w3[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int q = 0; q < 8; ++q) o[q] = b2u(__hadd2(u2b(o[q]), u2b(w3[q])));
          }
        } else {
          float acc[16];
#pragma unroll
          for (int q = 0; q < 16; ++q) acc[q] = 0.f;
          for (int xx = ((FAR && far) ? g0a : g0); xx < ((FAR && far) ? g0a : g0) + d; ++xx) {
            if (!ATOM && xx == ((FAR && far) ? rsa : rs)) continue;
            uint4 u0, u1;
            if (FAR && far) {
              const int xa = (MODE != MODE_FWD) ? __ldg(p.rev_row + xx) : xx;
              const uint4* gp = reinterpret_cast<const uint4*>(p.Hprev + (int64_t)xa * p.ld + j * 16);
              u0 = g_load<ACT, FIRST>(gp, p.act_param);
              u1 = g_load<ACT, FIRST>(gp + 1, p.act_param);
            } else {
              const int x = ATOM ? nb_at(xx) : ((MODE != MODE_FWD) ? (int)rvl[xx] : xx);
              u0 = s_load<ACT, FIRST>(sbase + sw128_off(x, c0), p.act_param);
              u1 = s_load<ACT, FIRST>(sbase + sw128_off(x, c0 + 1), p.act_param);
            }
            const uint32_t w[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
            for (int q = 0; q < 8; ++q) { acc[2 * q] += bf_lo(w[q]); acc[2 * q + 1] += bf_hi(w[q]); }
          }
#pragma unroll
          for (int q = 0; q < 8; ++q) o[q] = pack_bf2(acc[2 * q], acc[2 * q + 1]);
        }
        if (!(kExp && (p.exp_flags & 131072))) {
          const uint32_t ab = sAop + (uint32_t)(j >> 2) * kSlabBytes;
          sts128(ab + sw128_off(r, c0), make_uint4(o[0], o[1], o[2], o[3]));
          sts128(ab + sw128_off(r, c0 + 1), make_uint4(o[4], o[5], o[6], o[7]));
        }
        if constexpr (kCanEmit) {
          // forward: A row r is M[r] (mixins.py:11-18); backward: A row r is ((S.P) dZ)[r].  One 32-byte
          // sector per thread and block, consumed by the W_h weight-gradient GEMM.
          if (gout != nullptr) st_global_2x128(gout + j * 16, o);
        }
      }
      // release the slabs not released inside the loop (the last one visited, and any this thread owned no block of)
      for (int sl = 0; sl < p.nslab; ++sl)
        if (left & (1u << sl)) mbar_arrive(bar(B_AFREE + sl));
      fence_proxy_async();
      for (int q = cur_pass; q < npass; ++q) mbar_arrive(bar(B_AREADY + q));   // every thread arrives once per pass
      if (tS == 0) trace_ev(p, it, 2);
      // publish the next tile's rowptr slice (other buffer; readers of it finished a tile ago)
      if (ATOM) {
        if (tn < n_items && tS <= nrn) s_rowptr[(b ^ 1) * 132 + tS] = rpn;
#pragma unroll
        for (int k = 0; k < kNbCap / 256; ++k) {
          const int i = tS + 256 * k;
          if (tn < n_items && i < natomsn) s_nb[(b ^ 1) * kNbCap + i] = (int16_t)nbn[k];
        }
      } else if (tn < n_items && tS <= natomsn) s_rowptr[(b ^ 1) * 132 + tS] = rpn;
      if (kNeedRev && tn < n_items && tS < 128) s_revl[(b ^ 1) * 128 + tS] = (int16_t)rvn;
      row0 = row0n; atom0 = atom0n; natoms = natomsn; far = farn; nr = nrn;
    }
  }

}


template <int ACT, bool FIRST, bool HAS_BIAS, int MODE, bool FAR, bool DROP, bool ATOM = false>
static cudaError_t launch_variant(int grid, cudaStream_t st, const CUtensorMap& mH, const Params& p) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_bond_step_fused<ACT, FIRST, HAS_BIAS, MODE, FAR, DROP, ATOM>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAlloc);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  k_bond_step_fused<ACT, FIRST, HAS_BIAS, MODE, FAR, DROP, ATOM><<<grid, kThreads, kSmemAlloc, st>>>(mH, p);
  return cudaSuccess;
}

// forward step: every fused activation x first x bias x {keep bits in the epilogue}.  Training steps take the keep bits
// with ReLU only (engine.plan's dropout_ok: the mirror reads the mask out of tau' of the stored state); a forward-only call
// (Monte Carlo dropout) takes them with every activation.  Bond steps only: the reference drops every directed edge's copy of
// an atom state independently, which an atom-row mask cannot express.
template <bool FAR, bool ATOM = false>
cudaError_t dispatch_fwd(int act, bool first, bool bias, bool drop, int grid, cudaStream_t st, const CUtensorMap& mH, const Params& p) {
#define DMPNN_FB(A, D)                                                                                              \
  (first ? (bias ? launch_variant<A, true, true, MODE_FWD, FAR, D, ATOM>(grid, st, mH, p)                             \
                 : launch_variant<A, true, false, MODE_FWD, FAR, D, ATOM>(grid, st, mH, p))                            \
         : (bias ? launch_variant<A, false, true, MODE_FWD, FAR, D, ATOM>(grid, st, mH, p)                            \
                 : launch_variant<A, false, false, MODE_FWD, FAR, D, ATOM>(grid, st, mH, p)))
#define DMPNN_FA(D)                                                  \
  switch (act) {                                                     \
    case DMPNN_ACT_NONE: return DMPNN_FB(DMPNN_ACT_NONE, D);           \
    case DMPNN_ACT_RELU: return DMPNN_FB(DMPNN_ACT_RELU, D);           \
    case DMPNN_ACT_LEAKYRELU: return DMPNN_FB(DMPNN_ACT_LEAKYRELU, D); \
    case DMPNN_ACT_TANH: return DMPNN_FB(DMPNN_ACT_TANH, D);           \
    case DMPNN_ACT_ELU: return DMPNN_FB(DMPNN_ACT_ELU, D);             \
  }
  if (drop) {
    if constexpr (ATOM) return cudaErrorInvalidValue;   // atom rows stand for every out-edge of the atom: no per-edge masks
    else { DMPNN_FA(true) }
  } else {
    DMPNN_FA(false)
  }
#undef DMPNN_FA
#undef DMPNN_FB
  return cudaErrorInvalidValue;
}

template <bool FAR, bool ATOM = false>
cudaError_t dispatch_bwd(int mode, int act, int grid, cudaStream_t st, const CUtensorMap& mH,
                         const Params& p) {
  if (mode == MODE_BWD_COPY) return launch_variant<DMPNN_ACT_NONE, false, false, MODE_BWD_COPY, FAR, false, ATOM>(grid, st, mH, p);
#define DMPNN_BM(A)                                                                                         \
  (mode == MODE_BWD_LAST ? launch_variant<A, false, false, MODE_BWD_LAST, FAR, false, ATOM>(grid, st, mH, p)   \
                         : launch_variant<A, false, false, MODE_BWD_MASK, FAR, false, ATOM>(grid, st, mH, p))
  switch (act) {
    case DMPNN_ACT_NONE: return DMPNN_BM(DMPNN_ACT_NONE);
    case DMPNN_ACT_RELU: return DMPNN_BM(DMPNN_ACT_RELU);
    case DMPNN_ACT_LEAKYRELU: return DMPNN_BM(DMPNN_ACT_LEAKYRELU);
    case DMPNN_ACT_TANH: return DMPNN_BM(DMPNN_ACT_TANH);
    case DMPNN_ACT_ELU: return DMPNN_BM(DMPNN_ACT_ELU);
  }
#undef DMPNN_BM
  return cudaErrorInvalidValue;
}

// explicit instantiations live in step_fused_{fwd,bwd,far_fwd,far_bwd,atom_fwd,atom_bwd}.cu
extern template cudaError_t dispatch_fwd<false, true>(int, bool, bool, bool, int, cudaStream_t, const CUtensorMap&, const Params&);
extern template cudaError_t dispatch_bwd<false, true>(int, int, int, cudaStream_t, const CUtensorMap&, const Params&);
extern template cudaError_t dispatch_fwd<false>(int, bool, bool, bool, int, cudaStream_t, const CUtensorMap&, const Params&);
extern template cudaError_t dispatch_fwd<true>(int, bool, bool, bool, int, cudaStream_t, const CUtensorMap&, const Params&);
extern template cudaError_t dispatch_bwd<false>(int, int, int, cudaStream_t, const CUtensorMap&, const Params&);
extern template cudaError_t dispatch_bwd<true>(int, int, int, cudaStream_t, const CUtensorMap&, const Params&);

}  // namespace fused
}  // namespace dmpnn
