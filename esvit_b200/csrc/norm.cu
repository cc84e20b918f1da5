// Residual-add + LayerNorm, PatchMerging gather + LayerNorm, token mean.  HBM-bound row kernels:
// one warp per token row, the row lives in registers (float4 per lane), single pass over HBM.
//
// Reference semantics (all models/swin_transformer.py of the reference):
//   x = shortcut + drop_path(branch); y = norm(x)          :329-331 with :283 of the next block
//   PatchMerging: 2x2 gather-concat -> LN(4C)               :393-417
//   final norm + AdaptiveAvgPool1d                          :687-689
#include <cstdlib>
#include "common.cuh"

namespace {

template <typename T> struct Vec4IO;
template <> struct Vec4IO<float> {
  static __device__ __forceinline__ float4 ld(const float* p) { return *reinterpret_cast<const float4*>(p); }
  static __device__ __forceinline__ void st(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
};
template <> struct Vec4IO<bf16> {
  static __device__ __forceinline__ float4 ld(const bf16* p) {
    uint2 u = *reinterpret_cast<const uint2*>(p);
    float2 a = __bfloat1622float2(*reinterpret_cast<bf162*>(&u.x));
    float2 b = __bfloat1622float2(*reinterpret_cast<bf162*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  static __device__ __forceinline__ void st(bf16* p, float4 v) {
    uint2 u;
    u.x = pack_bf162(v.x, v.y);
    u.y = pack_bf162(v.z, v.w);
    *reinterpret_cast<uint2*>(p) = u;
  }
};

__device__ __forceinline__ float sum4(float4 v) { return (v.x + v.y) + (v.z + v.w); }

// ---------------------------------------------------------------------------------------------
// Row kernels.  LPR lanes share one row (8 / 16 / 32 by row width), so a warp streams 32/LPR rows at once: narrow rows
// (C = 96 is the largest token count of the model) keep all lanes busy and 4x the bytes in flight per warp.
// Lane l of its group owns float4 chunks (i*LPR + l), i < NV.
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// forward: xout = x + keep[b] * delta ; y = LN(xout) * gamma + beta   (x may be NULL = 0: xout = fp32(delta), the start
// of a residual stream - PatchMerging's reduction output - without a separate cast kernel)
template <int LPR, int NV, typename OutT>
__global__ void __launch_bounds__(256) add_ln_fwd_kernel(
    const float* __restrict__ x, const bf16* __restrict__ delta,
    const float* __restrict__ keep, int tokens_per_sample, const float* __restrict__ gamma,
    const float* __restrict__ beta, float eps, float* __restrict__ xout, OutT* __restrict__ y,
    float* __restrict__ mean_o, float* __restrict__ rstd_o, long long T, int C) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float invC = 1.f / (float)C;
  for (long long r0 = warp * RPW; r0 < T; r0 += nwarps * RPW) {
    const long long row = r0 + sub;
    const bool ok = row < T;
    float4 v[NV];
    const float ks = (keep && ok) ? keep[row / tokens_per_sample] : 1.f;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * LPR + l) * 4;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ok && c < C) {
        if (x) v[i] = Vec4IO<float>::ld(x + row * C + c);
        if (delta) {
          const float4 d = Vec4IO<bf16>::ld(delta + row * C + c);
          v[i].x += ks * d.x; v[i].y += ks * d.y; v[i].z += ks * d.z; v[i].w += ks * d.w;
          if (xout) Vec4IO<float>::st(xout + row * C + c, v[i]);
        }
        s += sum4(v[i]);
      }
    }
    if (!y) continue;
    const float mean = group_sum<LPR>(s) * invC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * LPR + l) * 4;
      if (c < C) {
        float a = v[i].x - mean, b = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (cc * cc + d * d);
      }
    }
    const float rstd = rsqrtf(group_sum<LPR>(q) * invC + eps);
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * LPR + l) * 4;
      if (ok && c < C) {
        float4 g = Vec4IO<float>::ld(gamma + c), b = Vec4IO<float>::ld(beta + c), o;
        o.x = (v[i].x - mean) * rstd * g.x + b.x;
        o.y = (v[i].y - mean) * rstd * g.y + b.y;
        o.z = (v[i].z - mean) * rstd * g.z + b.z;
        o.w = (v[i].w - mean) * rstd * g.w + b.w;
        Vec4IO<OutT>::st(y + row * C + c, o);
      }
    }
    if (ok && l == 0) { mean_o[row] = mean; rstd_o[row] = rstd; }
  }
}

// backward: G = dxo + LNbwd(dy) ; dx = G ; ddelta = keep * G ; dgamma += dy*xhat ; dbeta += dy ; ddbias += keep*G
template <int LPR, int NV, typename DyT, int OCC>
// NV <= 3 (C <= 384 at 8/16/32 lanes per row: every stage-0..2 launch, 85 % of this kernel's bytes): OCC = 3 CTAs/SM at 80
// registers (some spill) or 2 at 128 - the kernel is latency-bound on bytes in flight, not on ALU (ESVIT_ADDLN_OCC)
__global__ void __launch_bounds__(NV <= 4 ? 256 : 128, NV <= 3 ? OCC : 1) add_ln_bwd_kernel(
    const DyT* __restrict__ dy, const float* __restrict__ dxo, const float* __restrict__ xs,
    const float* __restrict__ mean_i, const float* __restrict__ rstd_i, const float* __restrict__ gamma,
    const float* __restrict__ keep, int tokens_per_sample, float* __restrict__ dx, bf16* __restrict__ ddelta,
    float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ ddbias, long long T, int C) {
  extern __shared__ float sred[];  // [3*C]
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float invC = 1.f / (float)C;
  float4 ag[NV], ab[NV], ad[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) {
    ag[i] = make_float4(0, 0, 0, 0); ab[i] = make_float4(0, 0, 0, 0); ad[i] = make_float4(0, 0, 0, 0);
  }
  for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  for (long long r0 = warp * RPW; r0 < T; r0 += nwarps * RPW) {
    const long long row = r0 + sub;
    const bool ok = row < T;
    const float ks = (keep && ok) ? keep[row / tokens_per_sample] : 1.f;
    // every global load of the row is issued before the first use (the incoming gradient of the residual stream too: it
    // used to be loaded after the two row reductions, a second exposed round trip per iteration of a latency-bound kernel)
    float4 G[NV], o[NV];
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * LPR + l) * 4;
      o[i] = make_float4(0, 0, 0, 0);
      if (dxo && ok && c < C) o[i] = Vec4IO<float>::ld(dxo + row * C + c);
    }
    if (dy) {
      const float mean = ok ? mean_i[row] : 0.f, rstd = ok ? rstd_i[row] : 0.f;
      float4 xh[NV], g[NV];
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NV; i++) {
        const int c = (i * LPR + l) * 4;
        xh[i] = make_float4(0, 0, 0, 0);
        g[i] = make_float4(0, 0, 0, 0);
        if (ok && c < C) {
          float4 xv = Vec4IO<float>::ld(xs + row * C + c);
          float4 d = Vec4IO<DyT>::ld(dy + row * C + c);
          float4 gm = Vec4IO<float>::ld(gamma + c);
          xh[i] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
          g[i] = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
          s1 += sum4(g[i]);
          s2 += (g[i].x * xh[i].x + g[i].y * xh[i].y) + (g[i].z * xh[i].z + g[i].w * xh[i].w);
          ag[i].x += d.x * xh[i].x; ag[i].y += d.y * xh[i].y; ag[i].z += d.z * xh[i].z; ag[i].w += d.w * xh[i].w;
          ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
        }
      }
      s1 = group_sum<LPR>(s1) * invC;
      s2 = group_sum<LPR>(s2) * invC;
#pragma unroll
      for (int i = 0; i < NV; i++) {
        G[i].x = fmaf(rstd, g[i].x - s1 - xh[i].x * s2, o[i].x);
        G[i].y = fmaf(rstd, g[i].y - s1 - xh[i].y * s2, o[i].y);
        G[i].z = fmaf(rstd, g[i].z - s1 - xh[i].z * s2, o[i].z);
        G[i].w = fmaf(rstd, g[i].w - s1 - xh[i].w * s2, o[i].w);
      }
    } else {
#pragma unroll
      for (int i = 0; i < NV; i++) G[i] = o[i];
    }
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * LPR + l) * 4;
      if (ok && c < C) {
        if (dx) Vec4IO<float>::st(dx + row * C + c, G[i]);
        if (ddelta)
          Vec4IO<bf16>::st(ddelta + row * C + c, make_float4(ks * G[i].x, ks * G[i].y, ks * G[i].z, ks * G[i].w));
        ad[i].x += ks * G[i].x; ad[i].y += ks * G[i].y; ad[i].z += ks * G[i].z; ad[i].w += ks * G[i].w;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int c = (i * LPR + l) * 4;
    if (c < C) {
      if (dy) {
        atomicAdd(&sred[c + 0], ag[i].x); atomicAdd(&sred[c + 1], ag[i].y);
        atomicAdd(&sred[c + 2], ag[i].z); atomicAdd(&sred[c + 3], ag[i].w);
        atomicAdd(&sred[C + c + 0], ab[i].x); atomicAdd(&sred[C + c + 1], ab[i].y);
        atomicAdd(&sred[C + c + 2], ab[i].z); atomicAdd(&sred[C + c + 3], ab[i].w);
      }
      if (ddbias) {
        atomicAdd(&sred[2 * C + c + 0], ad[i].x); atomicAdd(&sred[2 * C + c + 1], ad[i].y);
        atomicAdd(&sred[2 * C + c + 2], ad[i].z); atomicAdd(&sred[2 * C + c + 3], ad[i].w);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    if (dy) {
      atomicAdd(&dgamma[i], sred[i]);
      atomicAdd(&dbeta[i], sred[C + i]);
    }
    if (ddbias) atomicAdd(&ddbias[i], sred[2 * C + i]);
  }
}

// ---------------------------------------------------------------------------------------------
// PatchMerging gather (+ zero pad for odd H/W) + LN over 4C.  Output channel block q in 0..3 takes the
// source token (2*oy + q%2, 2*ox + q/2): x0=(even,even) x1=(odd,even) x2=(even,odd) x3=(odd,odd).
template <int NV>
__global__ void __launch_bounds__(256) merge_ln_fwd_kernel(
    const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
    bf16* __restrict__ y, float* __restrict__ mean_o, float* __restrict__ rstd_o, int B, int H, int W, int C) {
  const int Ho = (H + 1) >> 1, Wo = (W + 1) >> 1, C4 = 4 * C;
  const long long T = (long long)B * Ho * Wo;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float inv = 1.f / (float)C4;
  for (long long row = warp; row < T; row += nwarps) {
    const int ox = (int)(row % Wo), oy = (int)((row / Wo) % Ho), b = (int)(row / ((long long)Wo * Ho));
    float4 v[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 4;
      v[i] = make_float4(0, 0, 0, 0);
      if (c < C4) {
        const int q = c / C, cc = c - q * C;
        const int sy = 2 * oy + (q & 1), sx = 2 * ox + (q >> 1);
        if (sy < H && sx < W) v[i] = Vec4IO<float>::ld(x + (((long long)b * H + sy) * W + sx) * C + cc);
        s += sum4(v[i]);
      }
    }
    const float mean = warp_sum(s) * inv;
    float qq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 4;
      if (c < C4) {
        float a = v[i].x - mean, bb = v[i].y - mean, cc = v[i].z - mean, d = v[i].w - mean;
        qq += (a * a + bb * bb) + (cc * cc + d * d);
      }
    }
    const float rstd = rsqrtf(warp_sum(qq) * inv + eps);
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 4;
      if (c < C4) {
        float4 g = Vec4IO<float>::ld(gamma + c), be = Vec4IO<float>::ld(beta + c), o;
        o.x = (v[i].x - mean) * rstd * g.x + be.x;
        o.y = (v[i].y - mean) * rstd * g.y + be.y;
        o.z = (v[i].z - mean) * rstd * g.z + be.z;
        o.w = (v[i].w - mean) * rstd * g.w + be.w;
        Vec4IO<bf16>::st(y + row * C4 + c, o);
      }
    }
    if (lane == 0) { mean_o[row] = mean; rstd_o[row] = rstd; }
  }
}

template <int NV>
__global__ void __launch_bounds__(256) merge_ln_bwd_kernel(
    const bf16* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean_i,
    const float* __restrict__ rstd_i, const float* __restrict__ gamma, float* __restrict__ dx,
    float* __restrict__ dgamma, float* __restrict__ dbeta, int B, int H, int W, int C) {
  extern __shared__ float sred[];  // [2*4C]
  const int Ho = (H + 1) >> 1, Wo = (W + 1) >> 1, C4 = 4 * C;
  const long long T = (long long)B * Ho * Wo;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float inv = 1.f / (float)C4;
  float4 ag[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; i++) { ag[i] = make_float4(0, 0, 0, 0); ab[i] = make_float4(0, 0, 0, 0); }
  for (int i = threadIdx.x; i < 2 * C4; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  // Up to NV = 16 the row's xh and gamma * dy stay in registers from the statistics pass to the dx pass.  At NV = 24
  // (4C = 3072) the dgamma / dbeta accumulators alone take 192 registers, so the statistics pass keeps nothing and
  // the dx pass loads the row again (it was just read by this warp: an L1 / L2 hit).
  constexpr bool HOLD = NV <= 16;
  constexpr int NH = HOLD ? NV : 1;
  for (long long row = warp; row < T; row += nwarps) {
    const int ox = (int)(row % Wo), oy = (int)((row / Wo) % Ho), b = (int)(row / ((long long)Wo * Ho));
    const float mean = mean_i[row], rstd = rstd_i[row];
    float4 xh[NH], g[NH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 4;
      if (c < C4) {
        const int q = c / C, cc = c - q * C;
        const int sy = 2 * oy + (q & 1), sx = 2 * ox + (q >> 1);
        float4 xv = make_float4(0, 0, 0, 0);
        if (sy < H && sx < W) xv = Vec4IO<float>::ld(x + (((long long)b * H + sy) * W + sx) * C + cc);
        float4 d = Vec4IO<bf16>::ld(dy + row * C4 + c);
        float4 gm = Vec4IO<float>::ld(gamma + c);
        const int h = HOLD ? i : 0;
        xh[h] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
        g[h] = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
        s1 += sum4(g[h]);
        s2 += (g[h].x * xh[h].x + g[h].y * xh[h].y) + (g[h].z * xh[h].z + g[h].w * xh[h].w);
        if constexpr (HOLD) {
          ag[i].x += d.x * xh[i].x; ag[i].y += d.y * xh[i].y; ag[i].z += d.z * xh[i].z; ag[i].w += d.w * xh[i].w;
          ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
        }
      }
    }
    s1 = warp_sum(s1) * inv;
    s2 = warp_sum(s2) * inv;
#pragma unroll
    for (int i = 0; i < NV; i++) {
      const int c = (i * 32 + lane) * 4;
      if (c < C4) {
        const int q = c / C, cc = c - q * C;
        const int sy = 2 * oy + (q & 1), sx = 2 * ox + (q >> 1);
        if constexpr (!HOLD) {
          float4 xv = make_float4(0, 0, 0, 0);
          if (sy < H && sx < W) xv = Vec4IO<float>::ld(x + (((long long)b * H + sy) * W + sx) * C + cc);
          float4 d = Vec4IO<bf16>::ld(dy + row * C4 + c);
          float4 gm = Vec4IO<float>::ld(gamma + c);
          xh[0] = make_float4((xv.x - mean) * rstd, (xv.y - mean) * rstd, (xv.z - mean) * rstd, (xv.w - mean) * rstd);
          g[0] = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
          ag[i].x += d.x * xh[0].x; ag[i].y += d.y * xh[0].y; ag[i].z += d.z * xh[0].z; ag[i].w += d.w * xh[0].w;
          ab[i].x += d.x; ab[i].y += d.y; ab[i].z += d.z; ab[i].w += d.w;
        }
        const int h = HOLD ? i : 0;
        if (sy < H && sx < W) {
          float4 o;
          o.x = rstd * (g[h].x - s1 - xh[h].x * s2);
          o.y = rstd * (g[h].y - s1 - xh[h].y * s2);
          o.z = rstd * (g[h].z - s1 - xh[h].z * s2);
          o.w = rstd * (g[h].w - s1 - xh[h].w * s2);
          Vec4IO<float>::st(dx + (((long long)b * H + sy) * W + sx) * C + cc, o);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; i++) {
    const int c = (i * 32 + lane) * 4;
    if (c < C4) {
      atomicAdd(&sred[c + 0], ag[i].x); atomicAdd(&sred[c + 1], ag[i].y);
      atomicAdd(&sred[c + 2], ag[i].z); atomicAdd(&sred[c + 3], ag[i].w);
      atomicAdd(&sred[C4 + c + 0], ab[i].x); atomicAdd(&sred[C4 + c + 1], ab[i].y);
      atomicAdd(&sred[C4 + c + 2], ab[i].z); atomicAdd(&sred[C4 + c + 3], ab[i].w);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C4; i += blockDim.x) {
    atomicAdd(&dgamma[i], sred[i]);
    atomicAdd(&dbeta[i], sred[C4 + i]);
  }
}

// pooled[b][c] = mean_t region[b][t][c]
__global__ void token_mean_fwd_kernel(const float* __restrict__ region, float* __restrict__ pooled, int N, int C) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int t = 0; t < N; t++) s += region[((long long)b * N + t) * C + c];
    pooled[(long long)b * C + c] = s / (float)N;
  }
}
// dregion[b][t][c] = (dregion_in ? dregion_in : 0) + dpooled[b][c] / N
__global__ void token_mean_bwd_kernel(const float* __restrict__ dpooled, const float* __restrict__ din,
                                      float* __restrict__ dout, int N, int C) {
  const int b = blockIdx.x;
  const float inv = 1.f / (float)N;
  for (int i = threadIdx.x; i < N * C; i += blockDim.x) {
    const int c = i % C;
    const long long o = (long long)b * N * C + i;
    dout[o] = (din ? din[o] : 0.f) + dpooled[(long long)b * C + c] * inv;
  }
}

int row_grid(long long T, int warps_per_block, int waves) {
  long long need = (T + warps_per_block - 1) / warps_per_block;
  long long cap = (long long)esvit_num_sms() * waves;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

}  // namespace

#define DISPATCH_NV(C_, CALL)                  \
  if ((C_) <= 128) { CALL(1) }                 \
  else if ((C_) <= 256) { CALL(2) }            \
  else if ((C_) <= 512) { CALL(4) }            \
  else if ((C_) <= 1024) { CALL(8) }           \
  else if ((C_) <= 2048) { CALL(16) }          \
  else if ((C_) <= 3072) { CALL(24) }          \
  else return ESVIT_ERR_BAD_ARG;

// (lanes per row, float4 chunks per lane) for a row of C floats
static bool addln_shape(int C, int& lpr, int& nv) {
  if (C % 4 != 0 || C <= 0 || C > 2048) return false;
  const int c4 = C / 4;
  lpr = c4 <= 32 ? 8 : (c4 <= 64 ? 16 : 32);
  nv = (c4 + lpr - 1) / lpr;
  if (nv == 5) nv = 6;
  else if (nv == 7) nv = 8;
  else if (nv > 8 && nv <= 12) nv = 12;
  else if (nv > 12) nv = 16;
  return true;
}

#define ADDLN_COMBOS(X) X(8, 1) X(8, 2) X(8, 3) X(8, 4) X(16, 3) X(16, 4) X(32, 3) X(32, 4) X(32, 6) X(32, 8) X(32, 12) X(32, 16)

ESVIT_API int esvit_add_ln_fwd(const float* x, const void* delta, const float* keep, int tokens_per_sample,
                               const float* gamma, const float* beta, float eps, float* xout, void* y,
                               int y_is_bf16, float* mean, float* rstd, long long T, int C, void* stream) {
  int lpr, nv;
  if (T <= 0 || !addln_shape(C, lpr, nv)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = row_grid((T + 32 / lpr - 1) / (32 / lpr), 8, 8);
  bool done = false;
#define X(L, N)                                                                                                  \
  if (!done && lpr == L && nv == N) {                                                                            \
    done = true;                                                                                                 \
    if (y_is_bf16)                                                                                               \
      add_ln_fwd_kernel<L, N, bf16><<<grid, 256, 0, st>>>(x, (const bf16*)delta, keep, tokens_per_sample, gamma, \
                                                          beta, eps, xout, (bf16*)y, mean, rstd, T, C);          \
    else                                                                                                         \
      add_ln_fwd_kernel<L, N, float><<<grid, 256, 0, st>>>(x, (const bf16*)delta, keep, tokens_per_sample,      \
                                                           gamma, beta, eps, xout, (float*)y, mean, rstd, T, C); \
  }
  ADDLN_COMBOS(X)
#undef X
  if (!done) return ESVIT_ERR_BAD_ARG;
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_add_ln_bwd(const void* dy, int dy_is_bf16, const float* dxo, const float* xs, const float* mean,
                               const float* rstd, const float* gamma, const float* keep, int tokens_per_sample,
                               float* dx, void* ddelta, float* dgamma, float* dbeta, float* ddelta_bias, long long T,
                               int C, void* stream) {
  int lpr, nv;
  if (T <= 0 || !addln_shape(C, lpr, nv)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int threads = nv <= 4 ? 256 : 128;
  const long long warp_rows = (T + 32 / lpr - 1) / (32 / lpr);
  // every CTA ends with 3*C global atomics: keep the CTA count modest
  // persistent grid = resident CTAs x small integer (no partial last wave)
  static const int occ = [] { const char* ev = getenv("ESVIT_ADDLN_OCC"); return ev && atoi(ev) == 3 ? 3 : 2; }();   // 2 (no spills) measured 0.68 of HBM over a step, 3: 0.66
  const int grid = row_grid(warp_rows, threads / 32, nv <= 3 ? occ : (threads == 256 ? 4 : 8));
  const size_t smem = 3 * (size_t)C * sizeof(float);
  bool done = false;
#define X(L, N)                                                                                                      \
  if (!done && lpr == L && nv == N) {                                                                                \
    done = true;                                                                                                     \
    if (dy_is_bf16 && (N > 3 || occ == 3))                                                                           \
      add_ln_bwd_kernel<L, N, bf16, 3><<<grid, threads, smem, st>>>((const bf16*)dy, dxo, xs, mean, rstd, gamma, keep, \
                                                                    tokens_per_sample, dx, (bf16*)ddelta, dgamma,     \
                                                                    dbeta, ddelta_bias, T, C);                        \
    else if (dy_is_bf16)                                                                                             \
      add_ln_bwd_kernel<L, N, bf16, 2><<<grid, threads, smem, st>>>((const bf16*)dy, dxo, xs, mean, rstd, gamma, keep, \
                                                                    tokens_per_sample, dx, (bf16*)ddelta, dgamma,     \
                                                                    dbeta, ddelta_bias, T, C);                        \
    else                                                                                                             \
      add_ln_bwd_kernel<L, N, float, 3><<<grid, threads, smem, st>>>((const float*)dy, dxo, xs, mean, rstd, gamma,   \
                                                                     keep, tokens_per_sample, dx, (bf16*)ddelta,      \
                                                                     dgamma, dbeta, ddelta_bias, T, C);               \
  }
  ADDLN_COMBOS(X)
#undef X
  if (!done) return ESVIT_ERR_BAD_ARG;
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_patch_merge_ln_fwd(const float* x, const float* gamma, const float* beta, float eps, void* y,
                                       float* mean, float* rstd, int B, int H, int W, int C, void* stream) {
  if (C % 4 != 0 || B <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long T = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
  const int grid = row_grid(T, 8, 8);
#define CALL(NV) merge_ln_fwd_kernel<NV><<<grid, 256, 0, st>>>(x, gamma, beta, eps, (bf16*)y, mean, rstd, B, H, W, C);
  DISPATCH_NV(4 * C, CALL)
#undef CALL
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_patch_merge_ln_bwd(const void* dy, const float* x, const float* mean, const float* rstd,
                                       const float* gamma, float* dx, float* dgamma, float* dbeta, int B, int H,
                                       int W, int C, void* stream) {
  if (C % 4 != 0 || B <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long T = (long long)B * ((H + 1) / 2) * ((W + 1) / 2);
  const int grid = row_grid(T, 8, 4);
  const size_t smem = 8 * (size_t)C * sizeof(float);
#define CALL(NV) \
  merge_ln_bwd_kernel<NV><<<grid, 256, smem, st>>>((const bf16*)dy, x, mean, rstd, gamma, dx, dgamma, dbeta, B, H, W, C);
  DISPATCH_NV(4 * C, CALL)
#undef CALL
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_token_mean_fwd(const float* region, float* pooled, int B, int N, int C, void* stream) {
  if (B <= 0) return ESVIT_ERR_BAD_ARG;
  token_mean_fwd_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(region, pooled, N, C);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_token_mean_bwd(const float* dpooled, const float* dregion_in, float* dregion, int B, int N, int C,
                                   void* stream) {
  if (B <= 0) return ESVIT_ERR_BAD_ARG;
  token_mean_bwd_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(dpooled, dregion_in, dregion, N, C);
  ESVIT_LAUNCH_CHECK();
}
