// Shared device helpers for the esvit_b200 sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define ESVIT_API extern "C" __attribute__((visibility("default")))

// every entry point returns a cudaError_t cast to int (0 == ok)
#define ESVIT_LAUNCH_CHECK() return (int)cudaGetLastError()

#define ESVIT_ERR_BAD_ARG 1001  // unsupported shape / argument (host wrapper raises ValueError)

typedef __nv_bfloat16 bf16;
typedef __nv_bfloat162 bf162;

static __device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
static __device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// 8 bf16 <-> 8 floats through one 16-byte access
struct __align__(16) bf16x8 {
  bf162 v[4];
};
static __device__ __forceinline__ void unpack8(const bf16x8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
static __device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; i++) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
static __device__ __forceinline__ uint32_t pack_bf162(float lo, float hi) {
  bf162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

// erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below the bf16 output resolution): one ex2, one rcp and
// five FMAs instead of erff()'s ~30-instruction path - the GELU kernels are otherwise ALU-bound, not HBM-bound.
// e = exp(-x^2/2) is shared with the Gaussian pdf of the derivative.  Exact-erf GELU (nn.GELU()) and its derivative.
static __device__ __forceinline__ float erf_as(float z_abs, float e) {
  const float t = __fdividef(1.f, fmaf(0.3275911f, z_abs, 1.f));  // MUFU.RCP (the IEEE reciprocal costs ~8 instructions)
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  return 1.f - p * t * e;
}
static __device__ __forceinline__ float gelu_f(float x) {
  const float e = __expf(-0.5f * x * x);
  const float er = copysignf(erf_as(fabsf(x) * 0.70710678118654752f, e), x);
  return 0.5f * x * (1.f + er);
}
static __device__ __forceinline__ float gelu_grad_f(float x) {
  const float e = __expf(-0.5f * x * x);
  const float er = copysignf(erf_as(fabsf(x) * 0.70710678118654752f, e), x);
  return 0.5f * (1.f + er) + x * 0.3989422804014327f * e;
}

static inline int esvit_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;  // H100 SXM
  }
  return sms;
}
