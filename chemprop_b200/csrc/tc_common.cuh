// Hopper (sm_90a) PTX wrappers shared by the tensor-core kernels: mbarrier, TMA (tensor + bulk), wgmma
// (fence / commit / wait, shared-memory operand descriptors), packed-bf16 helpers.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "wgmma_ops.cuh"

// Timing experiments are compiled in only with -DDMPNN_EXPERIMENTS=1; the DMPNN_EXP environment variable then selects them
// at run time, one bit each (listed where each kernel tests them).  Their results are wrong by construction.
#ifndef DMPNN_EXPERIMENTS
#define DMPNN_EXPERIMENTS 0
#endif

namespace dmpnn {
namespace tc {

constexpr bool kExp = DMPNN_EXPERIMENTS != 0;

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  // suspend-time hint (ns): the thread sleeps in hardware until the phase completes (or the hint
  // expires) instead of burning issue slots in a spin loop
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(200000u)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must fail loudly (trap) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
      printf("dmpnn fused step: mbarrier wait timed out (block %d thread %d bar %u parity %u)\n", blockIdx.x,
             threadIdx.x, bar, parity);
      __trap();
    }
  }
}
// The bounded wait of the kernels that keep wgmma groups in flight (fused depth step, k_wgrad_tc): the timeout of mbar_wait
// without its printf.  A function call anywhere in a kernel makes ptxas serialise every wgmma (C7510), so on a timeout it
// only traps: a protocol bug still fails loudly (the launch ends in a sticky error that the next synchronising CUDA call
// reports) instead of hanging the GPU, but it no longer names the block, thread and barrier.  Swapping in mbar_wait, whose
// printf names them, brings that report back for debugging (at the cost of serialised wgmmas).
__device__ __forceinline__ void mbar_wait_trap(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) asm volatile("trap;");
  }
}
// one lane of a CONVERGED warp; keeps the warp on the uniform datapath (UTMALDG operands live
// in uniform registers -- issuing them from a divergent `lane == 0` branch makes ptxas emit a
// per-lane emulation loop around every instruction)
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tmap, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// bring a box into L2 only (no shared-memory destination): deepens the prefetch distance of the
// streams whose shared-memory staging is shallow
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
               "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}
// ---- warpgroup MMA (wgmma) ----------------------------------------------------------------------
// wgmma_fence orders the warpgroup's register / shared-memory accesses before the MMAs that follow; commit closes a group
// of issued MMAs, wait<N> blocks until at most N groups are still in flight (their accumulators are then readable).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Per-warpgroup register budget (sm_90a): every warp of a warpgroup executes the same one.  dec returns registers to the
// CTA's pool, inc blocks until the pool holds enough; N is a multiple of 8 in [24, 256].
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous MMA
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// K-major, SWIZZLE_128B operand descriptor (rows of 128 B, 8-row groups 1024 B apart); advancing the start address by
// 32 B steps one k16 (bf16) / k8 (tf32) slice along the row
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  uint64_t d = (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;             // leading byte offset (unused for swizzled K-major) = 16 B
  d |= (uint64_t)(1024 >> 4) << 32;   // stride byte offset: 8 rows x 128 B
  d |= (uint64_t)1 << 62;             // SWIZZLE_128B
  return d;
}
// MN-major SWIZZLE_128B operand (bf16): rows of the contraction index at 128 B pitch (64 MN elements), 8-row groups
// 1024 B apart (SBO), 64-element MN blocks `lbo` bytes apart (LBO)
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t saddr, uint32_t lbo) {
  uint64_t d = (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// 16-byte global store of 8 bf16 (two per 32-byte sector of a 16-column block)
__device__ __forceinline__ void st_global_2x128(void* ptr, const uint32_t (&v)[8]) {
  uint4* q = reinterpret_cast<uint4*>(ptr);
  q[0] = make_uint4(v[0], v[1], v[2], v[3]);
  q[1] = make_uint4(v[4], v[5], v[6], v[7]);
}
// Accumulator fragment of the calling thread inside its warpgroup (see wgmma_ops.cuh): rows acc_row0 and acc_row0 + 8,
// columns 8 * b + acc_col0 + {0, 1} of every 8-column block b
__device__ __forceinline__ int acc_row0(int t) { return ((t >> 5) << 4) + ((t & 31) >> 2); }
__device__ __forceinline__ int acc_col0(int t) { return (t & 3) << 1; }

// Output column held by accumulator column j (0 <= j < nc) of an nc-column chunk / work item (nc % 8 == 0).  The weight
// packers (k_pack_weight, k_pack_weight_tc) put W row `acc_out_col(j, nc)` at B row j, so that every thread's fragment covers
// contiguous output columns and the epilogues load and store whole runs:
// * in a 32-column group [32 g, 32 g + 32) (b and q swapped): accumulator column 32 g + 8 b + 2 q + e holds output column
//   32 g + 8 q + 2 b + e, so thread q (acc_col0 = 2 q) holds columns 32 g + 8 q + [0, 8): one 16-byte run per row;
// * in a 16-column tail (nc - 32 g in [16, 32)): 32 g + 8 b + 2 q + e holds 32 g + 4 q + 2 b + e, an 8-byte run per row;
// * an 8-column tail stays in place: thread q holds its 2 columns 2 q + {0, 1}.
// Every output column comes from the same products, summed in the same k order: only the register that holds it changes.
__host__ __device__ __forceinline__ int acc_out_col(int j, int nc) {
  const int base = j & ~31, rem = nc - base;
  if (rem >= 32) return base + (((j >> 1) & 3) << 3) + (((j >> 3) & 3) << 1) + (j & 1);
  if (rem >= 16 && j - base < 16) return base + (((j >> 1) & 3) << 2) + (((j >> 3) & 1) << 1) + (j & 1);
  return j;
}
// Width of the run of output columns whose first column is acc_out_col(j, nc), for the first accumulator column j of a
// thread in a group or tail (32 g + 2 q; 32 g + 16 + 2 q for an 8-column tail after a 16-column one): 8 in a full 32-column
// group, 4 in a 16-column tail, 2 in an 8-column tail, 0 past the chunk
__host__ __device__ __forceinline__ int acc_run_cols(int j, int nc) {
  const int base = j & ~31, rem = nc - base;
  if (rem >= 32) return 8;
  if (rem >= 16 && j - base < 16) return 4;
  return j < nc ? 2 : 0;
}
// A run of nw (4, 2 or 1) bf16x2 words: one 16-, 8- or 4-byte load / store (the address is aligned to its size)
__device__ __forceinline__ void ld_run(const __nv_bfloat16* p, int nw, uint32_t (&v)[4]) {
  if (nw == 4) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
    v[0] = u.x; v[1] = u.y; v[2] = u.z; v[3] = u.w;
  } else if (nw == 2) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    v[0] = u.x; v[1] = u.y;
  } else {
    v[0] = __ldg(reinterpret_cast<const unsigned int*>(p));
  }
}
__device__ __forceinline__ void st_run(__nv_bfloat16* p, int nw, const uint32_t (&v)[4]) {
  if (nw == 4) *reinterpret_cast<uint4*>(p) = make_uint4(v[0], v[1], v[2], v[3]);
  else if (nw == 2) *reinterpret_cast<uint2*>(p) = make_uint2(v[0], v[1]);
  else *reinterpret_cast<uint32_t*>(p) = v[0];
}

__device__ __forceinline__ uint4 lds128(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
// byte offset of 16-byte chunk `c` (0..7) of row `r` inside a 128-row, 128-byte-row SWIZZLE_128B slab
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4));
}

template <int ACT>
__device__ __forceinline__ float act_t(float p, float z) {
  if constexpr (ACT == DMPNN_ACT_RELU) return fmaxf(z, 0.f);
  else if constexpr (ACT == DMPNN_ACT_LEAKYRELU) return z > 0.f ? z : p * z;
  else if constexpr (ACT == DMPNN_ACT_TANH) return tanhf(z);
  else if constexpr (ACT == DMPNN_ACT_ELU) return z > 0.f ? z : p * expm1f(z);
  else return z;
}



// ---- packed bf16x2 helpers for the in-place message computation -------------------------------
using bf2 = __nv_bfloat162;
__device__ __forceinline__ bf2 u2b(uint32_t w) { return *reinterpret_cast<bf2*>(&w); }
__device__ __forceinline__ uint32_t b2u(bf2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ uint4 add4(uint4 a, uint4 b) {
  return make_uint4(b2u(__hadd2(u2b(a.x), u2b(b.x))), b2u(__hadd2(u2b(a.y), u2b(b.y))),
                    b2u(__hadd2(u2b(a.z), u2b(b.z))), b2u(__hadd2(u2b(a.w), u2b(b.w))));
}
template <int ACT>
__device__ __forceinline__ uint32_t act_word(uint32_t w, float ap) {
  if constexpr (ACT == DMPNN_ACT_NONE) return w;
  else if constexpr (ACT == DMPNN_ACT_RELU) return b2u(__hmax2(u2b(w), __float2bfloat162_rn(0.f)));
  else return pack_bf2(act_t<ACT>(ap, bf_lo(w)), act_t<ACT>(ap, bf_hi(w)));
}
template <int ACT, bool FIRST>
__device__ __forceinline__ uint4 s_load(uint32_t addr, float ap) {
  uint4 u = lds128(addr);
  if constexpr (FIRST) {
    u.x = act_word<ACT>(u.x, ap); u.y = act_word<ACT>(u.y, ap);
    u.z = act_word<ACT>(u.z, ap); u.w = act_word<ACT>(u.w, ap);
  }
  return u;
}


// the same 16-byte load from global memory (windows of molecules larger than a tile gather from L2)
template <int ACT, bool FIRST>
__device__ __forceinline__ uint4 g_load(const uint4* ptr, float ap) {
  uint4 u = __ldg(ptr);
  if constexpr (FIRST) {
    u.x = act_word<ACT>(u.x, ap); u.y = act_word<ACT>(u.y, ap);
    u.z = act_word<ACT>(u.z, ap); u.w = act_word<ACT>(u.w, ap);
  }
  return u;
}

}  // namespace tc
}  // namespace dmpnn
