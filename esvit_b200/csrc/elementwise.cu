// Row L2-normalise and weight-norm kernels of DINOHead (HBM-bound, vectorised 16-byte accesses).
//
// Reference semantics:
//   DINOHead: F.normalize(x, dim=-1, p=2) (eps 1e-12) and
//   weight_norm(last_layer): w = g * v / ||v||_row          models/vision_transformer.py:403-417
#include "common.cuh"

namespace {

// one warp per row, D % 8 == 0, D <= 8*32*NV
template <int NV>
__global__ void __launch_bounds__(256) l2norm_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y,
                                                         float* __restrict__ inv_o, float eps, long long R, int D) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < R; r += nwarps) {
    float f[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 8;
      if (c < D) {
        unpack8(*reinterpret_cast<const bf16x8*>(x + r * D + c), f[i]);
#pragma unroll
        for (int j = 0; j < 8; j++) s += f[i][j] * f[i][j];
      }
    }
    const float inv = 1.f / fmaxf(sqrtf(warp_sum(s)), eps);
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 8;
      if (c < D) {
#pragma unroll
        for (int j = 0; j < 8; j++) f[i][j] *= inv;
        *reinterpret_cast<bf16x8*>(y + r * D + c) = pack8(f[i]);
      }
    }
    if (lane == 0) inv_o[r] = inv;
  }
}

// dx = inv * (dy - xn * <xn, dy>), xn = x * inv
template <int NV>
__global__ void __launch_bounds__(256) l2norm_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                         const float* __restrict__ inv_i, bf16* __restrict__ dx,
                                                         long long R, int D) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < R; r += nwarps) {
    const float inv = inv_i[r];
    float f[NV][8], g[NV][8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 8;
      if (c < D) {
        unpack8(*reinterpret_cast<const bf16x8*>(x + r * D + c), f[i]);
        unpack8(*reinterpret_cast<const bf16x8*>(dy + r * D + c), g[i]);
#pragma unroll
        for (int j = 0; j < 8; j++) { f[i][j] *= inv; s += f[i][j] * g[i][j]; }
      }
    }
    s = warp_sum(s);
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 8;
      if (c < D) {
#pragma unroll
        for (int j = 0; j < 8; j++) g[i][j] = inv * (g[i][j] - f[i][j] * s);
        *reinterpret_cast<bf16x8*>(dx + r * D + c) = pack8(g[i]);
      }
    }
  }
}

// w = v * (g / ||v||), one warp per row; D % 4 == 0
__global__ void __launch_bounds__(256) weight_norm_fwd_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                                              bf16* __restrict__ w, float* __restrict__ norm_o,
                                                              long long K, int D) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < K; r += nwarps) {
    float s = 0.f;
    for (int c = lane * 4; c < D; c += 128) {
      float4 a = *reinterpret_cast<const float4*>(v + r * D + c);
      s += (a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w);
    }
    const float n = sqrtf(warp_sum(s));
    const float sc = g[r] / n;
    for (int c = lane * 4; c < D; c += 128) {
      float4 a = *reinterpret_cast<const float4*>(v + r * D + c);
      uint2 u;
      u.x = pack_bf162(a.x * sc, a.y * sc);
      u.y = pack_bf162(a.z * sc, a.w * sc);
      *reinterpret_cast<uint2*>(w + r * D + c) = u;
    }
    if (lane == 0) norm_o[r] = n;
  }
}

// dv = (g/n) * (dw - v * <dw,v>/n^2) ; dg = <dw,v>/n.   dw bf16: autograd hands the gradient of w over in w's dtype
__device__ __forceinline__ float4 load4(const bf16* p) {
  uint2 u = *reinterpret_cast<const uint2*>(p);
  float2 d0 = __bfloat1622float2(*reinterpret_cast<bf162*>(&u.x));
  float2 d1 = __bfloat1622float2(*reinterpret_cast<bf162*>(&u.y));
  return make_float4(d0.x, d0.y, d1.x, d1.y);
}

__global__ void __launch_bounds__(256) weight_norm_bwd_kernel(const float* __restrict__ v, const float* __restrict__ g,
                                                              const float* __restrict__ norm_i,
                                                              const bf16* __restrict__ dw, float* __restrict__ dv,
                                                              float* __restrict__ dg, long long K, int D) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < K; r += nwarps) {
    float s = 0.f;
    for (int c = lane * 4; c < D; c += 128) {
      const float4 a = *reinterpret_cast<const float4*>(v + r * D + c);
      const float4 d = load4(dw + r * D + c);
      s += (a.x * d.x + a.y * d.y) + (a.z * d.z + a.w * d.w);
    }
    s = warp_sum(s);
    const float n = norm_i[r], gg = g[r];
    const float sc = gg / n, k2 = s / (n * n);
    for (int c = lane * 4; c < D; c += 128) {
      const float4 a = *reinterpret_cast<const float4*>(v + r * D + c);
      const float4 d = load4(dw + r * D + c);
      float4 o;
      o.x = sc * (d.x - a.x * k2);
      o.y = sc * (d.y - a.y * k2);
      o.z = sc * (d.z - a.z * k2);
      o.w = sc * (d.w - a.w * k2);
      *reinterpret_cast<float4*>(dv + r * D + c) = o;
    }
    if (lane == 0 && dg) dg[r] = s / n;
  }
}

int ew_grid(long long n, int per_block, int waves) {
  long long need = (n + per_block - 1) / per_block;
  long long cap = (long long)esvit_num_sms() * waves;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

}  // namespace

ESVIT_API int esvit_l2norm_fwd(const void* x, void* y, float* inv, float eps, long long R, int D, void* stream) {
  if (D % 8 != 0 || D > 1024 || R <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ew_grid(R, 8, 16);
  if (D <= 256)
    l2norm_fwd_kernel<1><<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)y, inv, eps, R, D);
  else
    l2norm_fwd_kernel<4><<<grid, 256, 0, st>>>((const bf16*)x, (bf16*)y, inv, eps, R, D);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_l2norm_bwd(const void* x, const void* dy, const float* inv, void* dx, long long R, int D,
                               void* stream) {
  if (D % 8 != 0 || D > 1024 || R <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ew_grid(R, 8, 16);
  if (D <= 256)
    l2norm_bwd_kernel<1><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)dy, inv, (bf16*)dx, R, D);
  else
    l2norm_bwd_kernel<4><<<grid, 256, 0, st>>>((const bf16*)x, (const bf16*)dy, inv, (bf16*)dx, R, D);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_weight_norm_fwd(const float* v, const float* g, void* w, float* norm, long long K, int D,
                                    void* stream) {
  if (D % 4 != 0 || K <= 0) return ESVIT_ERR_BAD_ARG;
  weight_norm_fwd_kernel<<<ew_grid(K, 8, 16), 256, 0, (cudaStream_t)stream>>>(v, g, (bf16*)w, norm, K, D);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_weight_norm_bwd(const float* v, const float* g, const float* norm, const void* dw, float* dv,
                                    float* dg, long long K, int D, void* stream) {
  if (D % 4 != 0 || K <= 0) return ESVIT_ERR_BAD_ARG;
  weight_norm_bwd_kernel<<<ew_grid(K, 8, 16), 256, 0, (cudaStream_t)stream>>>(v, g, norm, (const bf16*)dw, dv, dg, K, D);
  ESVIT_LAUNCH_CHECK();
}
