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
