// ViT token embedding and the cls / region split of the final norm's output.
//
// Reference: models/vision_transformer.py
//   PatchEmbed.forward :136-139              Conv2d(3, D, p, stride p) -> flatten(2).transpose(1, 2)
//   VisionTransformer.forward_features :233-251   cat(cls_token, patches) + pos_embed ; ... ; x[:, 0], x[:, 1:]
//
// The p x p / stride p convolution is a GEMM over non-overlapping patches: esvit_vit_patches gathers the fp32 NCHW
// crops into bf16 rows [B*N, 3p^2] in the conv weight's (c, ky, kx) flatten order, esvit_gemm_bf16 adds the bias.
// esvit_vit_tokens_fwd writes the fp32 residual stream [B, 1+N, D]: row 0 = cls + pos[0], row 1+i = patch_i + pos[1+i].
// The backward sums over the batch in a fixed order (dpos, then dbias / dcls from dpos): no atomics.
#include "common.cuh"

namespace ve {

// one thread per bf16 pair (p even): patches[b*N + py*np + px][c*p*p + ky*p + kx] = img[b, c, py*p + ky, px*p + kx]
__global__ void __launch_bounds__(256) patches_kernel(const float* __restrict__ img, bf16* __restrict__ patches,
                                                      long long npairs, int S, int p) {
  const int np = S / p, N = np * np, K3 = 3 * p * p;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < npairs; e += (long long)gridDim.x * blockDim.x) {
    const long long idx = e * 2;
    const long long row = idx / K3;
    const int col = (int)(idx - row * K3);
    const int c = col / (p * p), rem = col - c * p * p, ky = rem / p, kx = rem - ky * p;
    const int b = (int)(row / N), i = (int)(row - (long long)b * N), py = i / np, px = i - py * np;
    const float2 v = *reinterpret_cast<const float2*>(img + (((long long)b * 3 + c) * S + py * p + ky) * S + px * p + kx);
    *reinterpret_cast<bf162*>(patches + idx) = __floats2bfloat162_rn(v.x, v.y);
  }
}

// x[b, j, d] = (j == 0 ? cls[d] : pe[b*N + j-1, d]) + pos[j, d]; four columns per thread
__global__ void __launch_bounds__(256) tokens_fwd_kernel(const bf16* __restrict__ pe, const float* __restrict__ cls,
                                                         const float* __restrict__ pos, float* __restrict__ x, int B,
                                                         int N, int D) {
  const int D4 = D / 4;
  const long long n = (long long)B * (N + 1) * D4;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / D4;
    const int d = (int)(e - r * D4) * 4;
    const int b = (int)(r / (N + 1)), j = (int)(r - (long long)b * (N + 1));
    float4 v;
    if (j == 0) {
      v = *reinterpret_cast<const float4*>(cls + d);
    } else {
      const uint2 u = *reinterpret_cast<const uint2*>(pe + ((long long)b * N + j - 1) * D + d);
      const float2 lo = __bfloat1622float2(*reinterpret_cast<const bf162*>(&u.x));
      const float2 hi = __bfloat1622float2(*reinterpret_cast<const bf162*>(&u.y));
      v = make_float4(lo.x, lo.y, hi.x, hi.y);
    }
    const float4 q = *reinterpret_cast<const float4*>(pos + (long long)j * D + d);
    v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    *reinterpret_cast<float4*>(x + r * D + d) = v;
  }
}

// dpos[j, d] = sum_b g[b, j, d] (b ascending); dpe[b*N + j-1, d] = bf16(g[b, j, d]) for j >= 1
__global__ void __launch_bounds__(256) tokens_bwd_kernel(const float* __restrict__ g, bf16* __restrict__ dpe,
                                                         float* __restrict__ dpos, int B, int N, int D) {
  const long long n = (long long)(N + 1) * D;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(e / D), d = (int)(e - (long long)j * D);
    float s = 0.f;
    for (int b = 0; b < B; b++) {
      const float v = g[((long long)b * (N + 1) + j) * D + d];
      s += v;
      if (j > 0) dpe[((long long)b * N + j - 1) * D + d] = __float2bfloat16_rn(v);
    }
    dpos[e] = s;
  }
}

// dbias[d] (+)= sum_{j >= 1} dpos[j, d] (j ascending); dcls[d] (+)= dpos[0, d]
__global__ void __launch_bounds__(128) tokens_bwd_fold_kernel(const float* __restrict__ dpos, float* __restrict__ dbias,
                                                              float* __restrict__ dcls, int N, int D, int accumulate) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  float s = 0.f;
  for (int j = 1; j <= N; j++) s += dpos[(long long)j * D + d];
  dbias[d] = accumulate ? dbias[d] + s : s;
  dcls[d] = accumulate ? dcls[d] + dpos[d] : dpos[d];
}

// dir 0: cls[b] = x[b, 0], region[b*N + i] = x[b, 1+i].  dir 1: x[b, j] = the gradient of whichever output row it
// went to (0 when that output has no gradient: cls or region null).
__global__ void __launch_bounds__(256) split_kernel(float* __restrict__ x, float* __restrict__ cls,
                                                    float* __restrict__ region, int B, int N, int D, int dir) {
  const int D4 = D / 4;
  const long long n = (long long)B * (N + 1) * D4;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long r = e / D4;
    const int d = (int)(e - r * D4) * 4;
    const int b = (int)(r / (N + 1)), j = (int)(r - (long long)b * (N + 1));
    float* o = j == 0 ? (cls ? cls + (long long)b * D + d : nullptr)
                      : (region ? region + ((long long)b * N + j - 1) * D + d : nullptr);
    float4* xp = reinterpret_cast<float4*>(x + r * D + d);
    if (dir == 0) {
      if (o) *reinterpret_cast<float4*>(o) = *xp;
    } else {
      *xp = o ? *reinterpret_cast<const float4*>(o) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

static unsigned grid_for(long long n) {
  const long long need = (n + 255) / 256, cap = (long long)esvit_num_sms() * 16;
  return (unsigned)(need < cap ? (need > 0 ? need : 1) : cap);
}

}  // namespace ve

ESVIT_API int esvit_vit_patches(const float* img, void* patches, int B, int S, int p, void* stream) {
  if (!img || !patches || B <= 0 || p <= 0 || p % 2 != 0 || S <= 0 || S % p != 0) return ESVIT_ERR_BAD_ARG;
  const long long npairs = (long long)B * S * S * 3 / 2;  // = B*N*3p^2 / 2
  ve::patches_kernel<<<ve::grid_for(npairs), 256, 0, (cudaStream_t)stream>>>(img, (bf16*)patches, npairs, S, p);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vit_tokens_fwd(const void* pe, const float* cls, const float* pos, float* x, int B, int N, int D,
                                   void* stream) {
  if (!pe || !cls || !pos || !x || B <= 0 || N <= 0 || D <= 0 || D % 4 != 0) return ESVIT_ERR_BAD_ARG;
  const long long n = (long long)B * (N + 1) * (D / 4);
  ve::tokens_fwd_kernel<<<ve::grid_for(n), 256, 0, (cudaStream_t)stream>>>((const bf16*)pe, cls, pos, x, B, N, D);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vit_tokens_bwd(const float* g, void* dpe, float* dpos, float* dbias, float* dcls, int accumulate,
                                   int B, int N, int D, void* stream) {
  if (!g || !dpe || !dpos || !dbias || !dcls || B <= 0 || N <= 0 || D <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  ve::tokens_bwd_kernel<<<ve::grid_for((long long)(N + 1) * D), 256, 0, st>>>(g, (bf16*)dpe, dpos, B, N, D);
  ve::tokens_bwd_fold_kernel<<<(D + 127) / 128, 128, 0, st>>>(dpos, dbias, dcls, N, D, accumulate);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vit_split(float* x, float* cls, float* region, int B, int N, int D, int dir, void* stream) {
  if (!x || B <= 0 || N <= 0 || D <= 0 || D % 4 != 0 || (dir != 0 && dir != 1)) return ESVIT_ERR_BAD_ARG;
  const long long n = (long long)B * (N + 1) * (D / 4);
  ve::split_kernel<<<ve::grid_for(n), 256, 0, (cudaStream_t)stream>>>(x, cls, region, B, N, D, dir);
  ESVIT_LAUNCH_CHECK();
}
