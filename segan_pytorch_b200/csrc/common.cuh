// Shared helpers for libsegan_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/segan_b200.h"

namespace sg {

void set_error(const char* fmt, ...);
// 16-bit format of every GRADIENT tensor the kernels read or write (sg_set_grad_dtype; default SG_F16)
extern int g_grad_dtype;

#define SG_CHECK_ARG(cond, ...)                                   \
  do {                                                            \
    if (!(cond)) {                                                \
      sg::set_error("%s:%d: %s: ", __FILE__, __LINE__, #cond);    \
      return SG_ERR_INVALID;                                      \
    }                                                             \
  } while (0)

#define SG_CHECK_LAUNCH()                                                         \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      sg::set_error("%s:%d: launch failed: %s", __FILE__, __LINE__,               \
                    cudaGetErrorString(e__));                                     \
      return SG_ERR_LAUNCH;                                                       \
    }                                                                             \
  } while (0)

#define SG_CHECK_CUDA(call)                                                       \
  do {                                                                            \
    cudaError_t e__ = (call);                                                     \
    if (e__ != cudaSuccess) {                                                     \
      sg::set_error("%s:%d: %s: %s", __FILE__, __LINE__, #call,                   \
                    cudaGetErrorString(e__));                                     \
      return SG_ERR_LAUNCH;                                                       \
    }                                                                             \
  } while (0)

constexpr int KW = 31;      // kernel width (train.opts gkwidth)
// served kernel widths of the stride-4 layers (engine.KW_MIN / KW_MAX): the waveform-end im2col holds 32 taps per
// input channel; below 4 a stride-4 transposed conv does not give 4x its input
constexpr int KW_MIN = 4, KW_MAX = 32;
__host__ __device__ __forceinline__ bool kw_served(int kw) { return kw >= KW_MIN && kw <= KW_MAX; }
constexpr int NTAP = 9;     // row taps d in [-4, 4] of the stride-1 "row" formulation
constexpr int NUM_SMS = 132;    // H100 SXM

__host__ __device__ inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// two fp32 -> packed fp16x2 (lo in the low half), round-to-nearest, saturating to +-65504 instead of inf: a
// loss-scaled fp16 gradient that overflows clips instead of poisoning the step (one F2FP.SATFINITE)
__device__ __forceinline__ uint32_t pack_half2_sat(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// ---- 16-bit element access, runtime dtype ------------------------------------------------
__device__ __forceinline__ float ld16(const void* p, int64_t i, int dtype) {
  if (dtype == SG_F16) return __half2float(reinterpret_cast<const __half*>(p)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
}
// fp16 stores saturate at +-65504 (a NaN stays NaN): a loss-scaled gradient that overflows clips instead of
// turning into inf; bf16 has fp32's range
__device__ __forceinline__ void st16(void* p, int64_t i, float v, int dtype) {
  if (dtype == SG_F16) reinterpret_cast<uint16_t*>(p)[i] = (uint16_t)pack_half2_sat(v, 0.f);
  else reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
}
__device__ __forceinline__ uint16_t cvt16(float v, int dtype) {
  if (dtype == SG_F16) return __half_as_ushort(__float2half_rn(v));
  return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
__device__ __forceinline__ float up16(uint16_t u, int dtype) {
  if (dtype == SG_F16) return __half2float(__ushort_as_half(u));
  return __bfloat162float(__ushort_as_bfloat16(u));
}
// 8 x 16-bit vector (16 bytes)
struct __align__(16) V8 { uint16_t v[8]; };

// reflect index for a position q in [-(L-1), 2L-2] onto [0, L)   (F.pad mode='reflect')
__device__ __forceinline__ int reflect_idx(int q, int L) {
  if (q < 0) q = -q;
  if (q >= L) q = 2 * (L - 1) - q;
  return q;
}
// circular: rolled[l] = src[(l - s) mod L]   (discriminator.py:165-172; s > 0 = right)
__device__ __forceinline__ int unroll_idx(int l, int s, int L) {
  int i = l - s;
  if (i < 0) i += L;
  if (i >= L) i -= L;
  return i;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace sg
