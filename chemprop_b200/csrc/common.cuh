// Shared helpers for libdmpnn_sm90.so (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/dmpnn.h"

namespace dmpnn {

void set_error(const char* fmt, ...);
void count_launches(int n);  // bookkeeping for dmpnn_launch_count()

#define DMPNN_CHECK_ARG(cond, ...)        \
  do {                                    \
    if (!(cond)) {                        \
      ::dmpnn::set_error(__VA_ARGS__);    \
      return -1;                          \
    }                                     \
  } while (0)

#define DMPNN_CHECK_LAUNCH(name, n_kernels)                                           \
  do {                                                                                \
    ::dmpnn::count_launches(n_kernels);                                               \
    cudaError_t e__ = cudaGetLastError();                                             \
    if (e__ != cudaSuccess) {                                                         \
      ::dmpnn::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));     \
      return -2;                                                                      \
    }                                                                                 \
  } while (0)

// ---- element access ------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) { return *p; }
template <>
__device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}
template <typename T>
__device__ __forceinline__ void st_from_float(T* p, float v);
template <>
__device__ __forceinline__ void st_from_float<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void st_from_float<__nv_bfloat16>(__nv_bfloat16* p, float v) {
  *p = __float2bfloat16_rn(v);
}

// ---- 4-element vector access (8 B of bf16 / 16 B of f32); pointers must be aligned accordingly --------
__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const __nv_bfloat16* p, float (&v)[4]) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  v[0] = __uint_as_float(u.x << 16); v[1] = __uint_as_float(u.x & 0xffff0000u);
  v[2] = __uint_as_float(u.y << 16); v[3] = __uint_as_float(u.y & 0xffff0000u);
}
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4(__nv_bfloat16* p, const float (&v)[4]) {
  __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], v[3]);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
template <typename T>
static inline bool vec4_ok(const void* p, int64_t ld) {
  return p == nullptr || ((reinterpret_cast<uintptr_t>(p) % (4 * sizeof(T))) == 0 && ld % 4 == 0);
}
// VW-element vector access: VW = 4 or 8 (8 bf16 = one 16-byte access; 8 f32 = two)
template <int VW, typename T>
__device__ __forceinline__ void ldv(const T* p, float (&v)[VW]) {
  if constexpr (VW == 4) {
    ld4(p, v);
  } else if constexpr (sizeof(T) == 2) {
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = __uint_as_float(w[i] << 16); v[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u); }
  } else {
    float a[4], b[4];
    ld4(p, a); ld4(p + 4, b);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[i] = a[i]; v[4 + i] = b[i]; }
  }
}
template <int VW, typename T>
__device__ __forceinline__ void stv(T* p, const float (&v)[VW]) {
  if constexpr (VW == 4) {
    st4(p, v);
  } else if constexpr (sizeof(T) == 2) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { __nv_bfloat162 t = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]); w[i] = *reinterpret_cast<uint32_t*>(&t); }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  } else {
    const float a[4] = {v[0], v[1], v[2], v[3]}, b[4] = {v[4], v[5], v[6], v[7]};
    st4(p, a); st4(p + 4, b);
  }
}
template <typename T>
static inline bool vec8_ok(const void* p, int64_t ld) {
  return p == nullptr || ((reinterpret_cast<uintptr_t>(p) % (8 * sizeof(T) > 16 ? 16 : 8 * sizeof(T))) == 0 && ld % 8 == 0);
}

// ---- activations (chemprop/nn/utils.py:43-55) ------------------------------------------
__device__ __forceinline__ float act_apply(int act, float p, float z) {
  switch (act) {
    case DMPNN_ACT_RELU: return fmaxf(z, 0.f);
    case DMPNN_ACT_LEAKYRELU: return z > 0.f ? z : p * z;
    case DMPNN_ACT_TANH: return tanhf(z);
    case DMPNN_ACT_ELU: return z > 0.f ? z : p * expm1f(z);
    default: return z;
  }
}
// derivative expressed through the OUTPUT y = tau(z)
__device__ __forceinline__ float act_grad_from_out(int act, float p, float y) {
  switch (act) {
    case DMPNN_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case DMPNN_ACT_LEAKYRELU: return y > 0.f ? 1.f : p;
    case DMPNN_ACT_TANH: return 1.f - y * y;
    case DMPNN_ACT_ELU: return y > 0.f ? 1.f : y + p;
    default: return 1.f;
  }
}
// derivative expressed through the PRE-activation z
__device__ __forceinline__ float act_grad_from_pre(int act, float p, float z) {
  switch (act) {
    case DMPNN_ACT_RELU: return z > 0.f ? 1.f : 0.f;
    case DMPNN_ACT_LEAKYRELU: return z > 0.f ? 1.f : p;
    case DMPNN_ACT_TANH: { float t = tanhf(z); return 1.f - t * t; }
    case DMPNN_ACT_ELU: return z > 0.f ? 1.f : p * expf(z);
    default: return 1.f;
  }
}

// dtype dispatch over {f32, bf16}
#define DMPNN_DISPATCH_DTYPE(dt, T, ...)                              \
  if ((dt) == DMPNN_F32) { using T = float; __VA_ARGS__ }             \
  else if ((dt) == DMPNN_BF16) { using T = __nv_bfloat16; __VA_ARGS__ } \
  else { ::dmpnn::set_error("bad dtype %d", (int)(dt)); return -1; }

static inline int ceil_div_i64(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace dmpnn
