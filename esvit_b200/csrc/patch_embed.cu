// PatchEmbed: 4x4/stride-4 conv (3 -> E) + LayerNorm as ONE coalesced gather + K=48 FMA + LN kernel.
// Reference: models/swin_transformer.py:537-547 (Conv2d(3,E,4,4) -> flatten(2).transpose(1,2) -> LN).
//
// HBM-bound (reads the fp32 NCHW crops once, writes the fp32 token stream once).  A warp owns 8 horizontally
// adjacent patches: each of the 12 (channel, dy) image rows of that strip is ONE 128-byte coalesced load
// (lane = pixel), the 48 taps of a patch are broadcast from registers with shuffles, lane l produces output
// channels l, l+32, ... from a transposed weight tile in shared memory, and the LN statistics are a warp
// reduction.  The backward recomputes the conv output instead of saving it.
#include "common.cuh"

namespace {

constexpr int PE_K = 48;

template <int EJ>
__device__ __forceinline__ void load_strip(const float* __restrict__ img, int b, int ty, int gx, int H, int W,
                                           int lane, float* px) {
  const int x = gx * 32 + lane;
#pragma unroll
  for (int c = 0; c < 3; c++)
#pragma unroll
    for (int dy = 0; dy < 4; dy++) {
      const int y = ty * 4 + dy;
      px[c * 4 + dy] = (x < W) ? img[(((long long)b * 3 + c) * H + y) * W + x] : 0.f;
    }
}

template <int EJ, int T>
__device__ __forceinline__ void conv_token(const float* px, const float* __restrict__ wsm, const float* bj, int E,
                                           int lane, float* acc) {
#pragma unroll
  for (int j = 0; j < EJ; j++) acc[j] = bj[j];
#pragma unroll
  for (int k = 0; k < PE_K; k++) {
    const float v = __shfl_sync(0xffffffffu, px[(k >> 4) * 4 + ((k >> 2) & 3)], 4 * T + (k & 3));
#pragma unroll
    for (int j = 0; j < EJ; j++) {
      const int c = lane + 32 * j;
      if (c < E) acc[j] += v * wsm[k * E + c];
    }
  }
}

template <int EJ>
__global__ void __launch_bounds__(128) patch_embed_fwd_kernel(
    const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ out,
    float* __restrict__ mean_o, float* __restrict__ rstd_o, int B, int H, int W, int E) {
  extern __shared__ float wsm[];  // [48][E]
  for (int i = threadIdx.x; i < PE_K * E; i += blockDim.x) {
    const int e = i / PE_K, k = i - e * PE_K;
    wsm[k * E + e] = w[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int Ht = H / 4, Wt = W / 4, G = (Wt + 7) / 8;
  const long long ngroups = (long long)B * Ht * G;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float bj[EJ], gj[EJ], bej[EJ];
#pragma unroll
  for (int j = 0; j < EJ; j++) {
    const int c = lane + 32 * j;
    bj[j] = c < E ? bias[c] : 0.f;
    gj[j] = c < E ? gamma[c] : 0.f;
    bej[j] = c < E ? beta[c] : 0.f;
  }
  const float invE = 1.f / (float)E;
  for (long long g = warp; g < ngroups; g += nwarps) {
    const int gx = (int)(g % G), ty = (int)((g / G) % Ht), b = (int)(g / ((long long)G * Ht));
    float px[12];
    load_strip<EJ>(img, b, ty, gx, H, W, lane, px);
#define PE_TOKEN(T)                                                                      \
  if (gx * 8 + T < Wt) {                                                                 \
    float acc[EJ];                                                                       \
    conv_token<EJ, T>(px, wsm, bj, E, lane, acc);                                        \
    float s = 0.f;                                                                       \
    _Pragma("unroll") for (int j = 0; j < EJ; j++) if (lane + 32 * j < E) s += acc[j];   \
    const float mean = warp_sum(s) * invE;                                               \
    float q = 0.f;                                                                       \
    _Pragma("unroll") for (int j = 0; j < EJ; j++) if (lane + 32 * j < E) {              \
      const float d = acc[j] - mean;                                                     \
      q += d * d;                                                                        \
    }                                                                                    \
    const float rstd = rsqrtf(warp_sum(q) * invE + eps);                                 \
    const long long tok = ((long long)b * Ht + ty) * Wt + gx * 8 + T;                    \
    _Pragma("unroll") for (int j = 0; j < EJ; j++) if (lane + 32 * j < E)                \
        out[tok * E + lane + 32 * j] = (acc[j] - mean) * rstd * gj[j] + bej[j];          \
    if (lane == 0) { mean_o[tok] = mean; rstd_o[tok] = rstd; }                           \
  }
    PE_TOKEN(0) PE_TOKEN(1) PE_TOKEN(2) PE_TOKEN(3) PE_TOKEN(4) PE_TOKEN(5) PE_TOKEN(6) PE_TOKEN(7)
#undef PE_TOKEN
  }
}

// backward: dW[e][k] += dconv[e] * patch[k], dbias += dconv, dgamma += dy*xhat, dbeta += dy
template <int EJ>
__global__ void __launch_bounds__(128, 1) patch_embed_bwd_kernel(
    const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ mean_i, const float* __restrict__ rstd_i,
    const float* __restrict__ dout, float* __restrict__ dw, float* __restrict__ dbias, float* __restrict__ dgamma,
    float* __restrict__ dbeta, int B, int H, int W, int E) {
  extern __shared__ float smem[];  // wsm [48][E] | dwsm [48][E] | dvec [3][E]
  float* wsm = smem;
  float* dwsm = smem + PE_K * E;
  float* dvec = dwsm + PE_K * E;
  for (int i = threadIdx.x; i < PE_K * E; i += blockDim.x) {
    const int e = i / PE_K, k = i - e * PE_K;
    wsm[k * E + e] = w[i];
    dwsm[i] = 0.f;
  }
  for (int i = threadIdx.x; i < 3 * E; i += blockDim.x) dvec[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int Ht = H / 4, Wt = W / 4, G = (Wt + 7) / 8;
  const long long ngroups = (long long)B * Ht * G;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float bj[EJ], gj[EJ], adw[EJ][PE_K], adb[EJ], adg[EJ], adbe[EJ];
#pragma unroll
  for (int j = 0; j < EJ; j++) {
    const int c = lane + 32 * j;
    bj[j] = c < E ? bias[c] : 0.f;
    gj[j] = c < E ? gamma[c] : 0.f;
    adb[j] = adg[j] = adbe[j] = 0.f;
#pragma unroll
    for (int k = 0; k < PE_K; k++) adw[j][k] = 0.f;
  }
  const float invE = 1.f / (float)E;
  for (long long g = warp; g < ngroups; g += nwarps) {
    const int gx = (int)(g % G), ty = (int)((g / G) % Ht), b = (int)(g / ((long long)G * Ht));
    float px[12];
    load_strip<EJ>(img, b, ty, gx, H, W, lane, px);
#define PE_TOKEN(T)                                                                               \
  if (gx * 8 + T < Wt) {                                                                          \
    float acc[EJ], gy[EJ], xh[EJ];                                                                \
    conv_token<EJ, T>(px, wsm, bj, E, lane, acc);                                                 \
    const long long tok = ((long long)b * Ht + ty) * Wt + gx * 8 + T;                             \
    const float mean = mean_i[tok], rstd = rstd_i[tok];                                           \
    float s1 = 0.f, s2 = 0.f;                                                                     \
    _Pragma("unroll") for (int j = 0; j < EJ; j++) {                                              \
      const int c = lane + 32 * j;                                                                \
      const float d = c < E ? dout[tok * E + c] : 0.f;                                            \
      xh[j] = c < E ? (acc[j] - mean) * rstd : 0.f;                                               \
      gy[j] = d * gj[j];                                                                          \
      s1 += gy[j];                                                                                \
      s2 += gy[j] * xh[j];                                                                        \
      adg[j] += d * xh[j];                                                                        \
      adbe[j] += d;                                                                               \
    }                                                                                             \
    s1 = warp_sum(s1) * invE;                                                                     \
    s2 = warp_sum(s2) * invE;                                                                     \
    float dc[EJ];                                                                                 \
    _Pragma("unroll") for (int j = 0; j < EJ; j++) {                                              \
      dc[j] = (lane + 32 * j < E) ? rstd * (gy[j] - s1 - xh[j] * s2) : 0.f;                       \
      adb[j] += dc[j];                                                                            \
    }                                                                                             \
    _Pragma("unroll") for (int k = 0; k < PE_K; k++) {                                            \
      const float v = __shfl_sync(0xffffffffu, px[(k >> 4) * 4 + ((k >> 2) & 3)], 4 * T + (k & 3)); \
      _Pragma("unroll") for (int j = 0; j < EJ; j++) adw[j][k] += dc[j] * v;                      \
    }                                                                                             \
  }
    PE_TOKEN(0) PE_TOKEN(1) PE_TOKEN(2) PE_TOKEN(3) PE_TOKEN(4) PE_TOKEN(5) PE_TOKEN(6) PE_TOKEN(7)
#undef PE_TOKEN
  }
#pragma unroll
  for (int j = 0; j < EJ; j++) {
    const int c = lane + 32 * j;
    if (c < E) {
#pragma unroll
      for (int k = 0; k < PE_K; k++) atomicAdd(&dwsm[c * PE_K + k], adw[j][k]);
      atomicAdd(&dvec[c], adb[j]);
      atomicAdd(&dvec[E + c], adg[j]);
      atomicAdd(&dvec[2 * E + c], adbe[j]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PE_K * E; i += blockDim.x) atomicAdd(&dw[i], dwsm[i]);
  for (int i = threadIdx.x; i < E; i += blockDim.x) {
    atomicAdd(&dbias[i], dvec[i]);
    atomicAdd(&dgamma[i], dvec[E + i]);
    atomicAdd(&dbeta[i], dvec[2 * E + i]);
  }
}


// ------------------------------------------------------------------------------------------------------------
// v2: register-tiled kernels.  The first version spent its time on shared-memory weight reads and shuffles (1 LDS per
// FMA); here a 256-thread CTA owns a 64-token x E tile with the gathered patches A[48][64] and the weights W[48][E]
// in shared memory, and every thread accumulates a 4-token x (E/16)-channel micro-tile: (1 + E/16) LDS per
// 4*E/16 FMAs.  LN statistics are 16-lane shuffles (a token's channels live in one half-warp).
constexpr int PE_TM = 64;        // tokens per tile
constexpr int PE_LDA = PE_TM + 4;  // padded row stride of A / dconv tiles (floats): 68 % 32 = 4 -> conflict-free float4

template <int EJ>
__device__ __forceinline__ void pe_gather_tile(const float* __restrict__ img, float* As, long long t0, long long T,
                                               int Ht, int Wt, int H, int W) {
  // 64 tokens x 12 (channel, dy) rows of 4 contiguous pixels = 768 float4 loads; lanes = consecutive tokens (coalesced)
#pragma unroll
  for (int it = 0; it < 3; it++) {
    const int f = threadIdx.x + it * 256;
    const int tok = f & 63, cdy = f >> 6;
    const long long gt = t0 + tok;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gt < T) {
      const int tx = (int)(gt % Wt), ty = (int)((gt / Wt) % Ht), b = (int)(gt / ((long long)Wt * Ht));
      const int c = cdy >> 2, dy = cdy & 3;
      v = *reinterpret_cast<const float4*>(img + (((long long)b * 3 + c) * H + ty * 4 + dy) * W + tx * 4);
    }
    As[(cdy * 4 + 0) * PE_LDA + tok] = v.x;
    As[(cdy * 4 + 1) * PE_LDA + tok] = v.y;
    As[(cdy * 4 + 2) * PE_LDA + tok] = v.z;
    As[(cdy * 4 + 3) * PE_LDA + tok] = v.w;
  }
}

template <int EJ>
__device__ __forceinline__ void pe_conv_tile(const float* As, const float* Ws, const float* bj, int E, int tg, int cg,
                                             float (&acc)[4][EJ]) {
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < EJ; j++) acc[i][j] = bj[j];
#pragma unroll 4
  for (int k = 0; k < PE_K; k++) {
    const float4 a = *reinterpret_cast<const float4*>(As + k * PE_LDA + tg * 4);
    float wv[EJ];
#pragma unroll
    for (int j = 0; j < EJ; j++) wv[j] = Ws[k * E + cg + 16 * j];
#pragma unroll
    for (int j = 0; j < EJ; j++) {
      acc[0][j] = fmaf(a.x, wv[j], acc[0][j]);
      acc[1][j] = fmaf(a.y, wv[j], acc[1][j]);
      acc[2][j] = fmaf(a.z, wv[j], acc[2][j]);
      acc[3][j] = fmaf(a.w, wv[j], acc[3][j]);
    }
  }
}

__device__ __forceinline__ float half_warp_sum(float v) {  // over the 16 lanes that share a token group
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int EJ>
__global__ void __launch_bounds__(256) patch_embed_fwd2_kernel(
    const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ out,
    float* __restrict__ mean_o, float* __restrict__ rstd_o, int B, int H, int W) {
  constexpr int E = 16 * EJ;
  extern __shared__ float smem[];
  float* Ws = smem;             // [48][E]
  float* As = Ws + PE_K * E;    // [48][PE_LDA]
  for (int i = threadIdx.x; i < PE_K * E; i += 256) {
    const int e = i / PE_K, k = i - e * PE_K;
    Ws[k * E + e] = w[i];
  }
  const int cg = threadIdx.x & 15, tg = threadIdx.x >> 4;
  const int Ht = H / 4, Wt = W / 4;
  const long long T = (long long)B * Ht * Wt;
  float bj[EJ], gj[EJ], bej[EJ];
#pragma unroll
  for (int j = 0; j < EJ; j++) { bj[j] = bias[cg + 16 * j]; gj[j] = gamma[cg + 16 * j]; bej[j] = beta[cg + 16 * j]; }
  const float invE = 1.f / (float)E;
  for (long long t0 = (long long)blockIdx.x * PE_TM; t0 < T; t0 += (long long)gridDim.x * PE_TM) {
    __syncthreads();
    pe_gather_tile<EJ>(img, As, t0, T, Ht, Wt, H, W);
    __syncthreads();
    float acc[4][EJ];
    pe_conv_tile<EJ>(As, Ws, bj, E, tg, cg, acc);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < EJ; j++) s += acc[i][j];
      const float mean = half_warp_sum(s) * invE;
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < EJ; j++) { const float d = acc[i][j] - mean; q += d * d; }
      const float rstd = rsqrtf(half_warp_sum(q) * invE + eps);
      const long long gt = t0 + tg * 4 + i;
      if (gt < T) {
#pragma unroll
        for (int j = 0; j < EJ; j++) out[gt * E + cg + 16 * j] = (acc[i][j] - mean) * rstd * gj[j] + bej[j];
        if (cg == 0) { mean_o[gt] = mean; rstd_o[gt] = rstd; }
      }
    }
  }
}

template <int EJ>
__global__ void __launch_bounds__(256) patch_embed_bwd2_kernel(
    const float* __restrict__ img, const float* __restrict__ w, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ mean_i, const float* __restrict__ rstd_i,
    const float* __restrict__ dout, float* __restrict__ dw, float* __restrict__ dbias, float* __restrict__ dgamma,
    float* __restrict__ dbeta, int B, int H, int W) {
  constexpr int E = 16 * EJ;
  extern __shared__ float smem[];
  float* Ws = smem;                    // [48][E]
  float* As = Ws + PE_K * E;           // [48][PE_LDA]   gathered patches, k-major
  float* Ds = As + PE_K * PE_LDA;      // [E][PE_LDA]    dconv, channel-major
  float* red = Ds + E * PE_LDA;        // [3][E]         dbias | dgamma | dbeta partial sums
  for (int i = threadIdx.x; i < PE_K * E; i += 256) {
    const int e = i / PE_K, k = i - e * PE_K;
    Ws[k * E + e] = w[i];
  }
  for (int i = threadIdx.x; i < 3 * E; i += 256) red[i] = 0.f;
  const int cg = threadIdx.x & 15, tg = threadIdx.x >> 4;
  const int Ht = H / 4, Wt = W / 4;
  const long long T = (long long)B * Ht * Wt;
  float bj[EJ], gj[EJ];
#pragma unroll
  for (int j = 0; j < EJ; j++) { bj[j] = bias[cg + 16 * j]; gj[j] = gamma[cg + 16 * j]; }
  const float invE = 1.f / (float)E;
  // this thread's dW[e = cg+16j][k = tg*3 + kk] (two partial sums each: even / odd tokens) and
  // per-channel sums
  float2 adw[3][EJ];
  float adb[EJ], adg[EJ], adbe[EJ];
#pragma unroll
  for (int j = 0; j < EJ; j++) {
    adb[j] = adg[j] = adbe[j] = 0.f;
    adw[0][j] = adw[1][j] = adw[2][j] = make_float2(0.f, 0.f);
  }
  for (long long t0 = (long long)blockIdx.x * PE_TM; t0 < T; t0 += (long long)gridDim.x * PE_TM) {
    __syncthreads();
    pe_gather_tile<EJ>(img, As, t0, T, Ht, Wt, H, W);
    __syncthreads();
    float acc[4][EJ];
    pe_conv_tile<EJ>(As, Ws, bj, E, tg, cg, acc);
    float dc[4][EJ];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const long long gt = t0 + tg * 4 + i;
      const bool ok = gt < T;
      const float mean = ok ? mean_i[gt] : 0.f, rstd = ok ? rstd_i[gt] : 0.f;
      float gy[EJ], xh[EJ], s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int j = 0; j < EJ; j++) {
        const float d = ok ? dout[gt * E + cg + 16 * j] : 0.f;
        xh[j] = (acc[i][j] - mean) * rstd;
        gy[j] = d * gj[j];
        s1 += gy[j];
        s2 += gy[j] * xh[j];
        adg[j] += d * xh[j];
        adbe[j] += d;
      }
      s1 = half_warp_sum(s1) * invE;
      s2 = half_warp_sum(s2) * invE;
#pragma unroll
      for (int j = 0; j < EJ; j++) {
        dc[i][j] = rstd * (gy[j] - s1 - xh[j] * s2);
        adb[j] += dc[i][j];
      }
    }
#pragma unroll
    for (int j = 0; j < EJ; j++)
      *reinterpret_cast<float4*>(Ds + (cg + 16 * j) * PE_LDA + tg * 4) = make_float4(dc[0][j], dc[1][j], dc[2][j], dc[3][j]);
    __syncthreads();
    // dW[e][k] += sum_tokens dconv[token][e] * A[token][k]   (thread: k = tg*3..+2, e = cg + 16 j)
#pragma unroll 4
    for (int t4 = 0; t4 < PE_TM / 4; t4++) {
      float4 a[3];
#pragma unroll
      for (int kk = 0; kk < 3; kk++) a[kk] = *reinterpret_cast<const float4*>(As + (tg * 3 + kk) * PE_LDA + t4 * 4);
#pragma unroll
      for (int j = 0; j < EJ; j++) {
        const float4 d = *reinterpret_cast<const float4*>(Ds + (cg + 16 * j) * PE_LDA + t4 * 4);
#pragma unroll
        for (int kk = 0; kk < 3; kk++) {
          adw[kk][j].x = fmaf(a[kk].x, d.x, adw[kk][j].x);
          adw[kk][j].y = fmaf(a[kk].y, d.y, adw[kk][j].y);
          adw[kk][j].x = fmaf(a[kk].z, d.z, adw[kk][j].x);
          adw[kk][j].y = fmaf(a[kk].w, d.w, adw[kk][j].y);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < EJ; j++) {
    const int e = cg + 16 * j;
#pragma unroll
    for (int kk = 0; kk < 3; kk++) atomicAdd(&dw[e * PE_K + tg * 3 + kk], adw[kk][j].x + adw[kk][j].y);
    atomicAdd(&red[e], adb[j]);
    atomicAdd(&red[E + e], adg[j]);
    atomicAdd(&red[2 * E + e], adbe[j]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < E; i += 256) {
    atomicAdd(&dbias[i], red[i]);
    atomicAdd(&dgamma[i], red[E + i]);
    atomicAdd(&dbeta[i], red[2 * E + i]);
  }
}

}  // namespace

#define PE_DISPATCH(E_, CALL)        \
  if ((E_) <= 32) { CALL(1) }        \
  else if ((E_) <= 64) { CALL(2) }   \
  else if ((E_) <= 96) { CALL(3) }   \
  else if ((E_) <= 128) { CALL(4) }  \
  else return ESVIT_ERR_BAD_ARG;

// img fp32 [B,3,H,W] (H,W multiples of 4); w fp32 [E,3,4,4]; out fp32 [B,(H/4)*(W/4),E]
ESVIT_API int esvit_patch_embed_fwd(const float* img, const float* w, const float* bias, const float* gamma,
                                    const float* beta, float eps, float* out, float* mean, float* rstd, int B, int H,
                                    int W, int E, void* stream) {
  if (H % 4 || W % 4 || B <= 0) return ESVIT_ERR_BAD_ARG;
  if (E % 16 == 0 && E <= 192 && E >= 32) {  // register-tiled v2
    const long long T = (long long)B * (H / 4) * (W / 4);
    long long need = (T + PE_TM - 1) / PE_TM, cap = (long long)esvit_num_sms() * 4;
    const int grid2 = (int)(need < cap ? need : cap);
    const size_t smem2 = (size_t)(PE_K * E + PE_K * PE_LDA) * sizeof(float);
#define CALL2(EJ)                                                                                                  \
  {                                                                                                                \
    if (smem2 > 48 * 1024) { /* E = 192 */                                                                        \
      cudaError_t e2 = cudaFuncSetAttribute(patch_embed_fwd2_kernel<EJ>,                                           \
                                            cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);              \
      if (e2 != cudaSuccess) return (int)e2;                                                                       \
    }                                                                                                              \
    patch_embed_fwd2_kernel<EJ><<<grid2, 256, smem2, (cudaStream_t)stream>>>(img, w, bias, gamma, beta, eps, out,  \
                                                                             mean, rstd, B, H, W);                 \
  }
    switch (E / 16) {
      case 2: CALL2(2) break;
      case 4: CALL2(4) break;
      case 6: CALL2(6) break;
      case 8: CALL2(8) break;
      case 12: CALL2(12) break;
      default: return ESVIT_ERR_BAD_ARG;
    }
#undef CALL2
    ESVIT_LAUNCH_CHECK();
  }
  const long long ngroups = (long long)B * (H / 4) * ((W / 4 + 7) / 8);
  long long need = (ngroups + 3) / 4, cap = (long long)esvit_num_sms() * 8;
  const int grid = (int)(need < cap ? need : cap);
  const size_t smem = (size_t)PE_K * E * sizeof(float);
#define CALL(EJ) \
  patch_embed_fwd_kernel<EJ><<<grid, 128, smem, (cudaStream_t)stream>>>(img, w, bias, gamma, beta, eps, out, mean, rstd, B, H, W, E);
  PE_DISPATCH(E, CALL)
#undef CALL
  ESVIT_LAUNCH_CHECK();
}

// dw [E,48], dbias/dgamma/dbeta [E] are ACCUMULATED into (caller zero-fills)
ESVIT_API int esvit_patch_embed_bwd(const float* img, const float* w, const float* bias, const float* gamma,
                                    const float* mean, const float* rstd, const float* dout, float* dw, float* dbias,
                                    float* dgamma, float* dbeta, int B, int H, int W, int E, void* stream) {
  if (H % 4 || W % 4 || B <= 0) return ESVIT_ERR_BAD_ARG;
  if (E % 16 == 0 && E <= 192 && E >= 32) {  // register-tiled v2
    const long long T = (long long)B * (H / 4) * (W / 4);
    long long need = (T + PE_TM - 1) / PE_TM, cap = (long long)esvit_num_sms() * 2;
    const int grid2 = (int)(need < cap ? need : cap);
    const size_t smem2 = (size_t)(PE_K * E + PE_K * PE_LDA + E * PE_LDA + 3 * E) * sizeof(float);
#define CALL2(EJ)                                                                                                  \
  {                                                                                                                \
    cudaError_t e2 = cudaFuncSetAttribute(patch_embed_bwd2_kernel<EJ>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                          (int)smem2);                                                             \
    if (e2 != cudaSuccess) return (int)e2;                                                                         \
    patch_embed_bwd2_kernel<EJ><<<grid2, 256, smem2, (cudaStream_t)stream>>>(img, w, bias, gamma, mean, rstd, dout, \
                                                                             dw, dbias, dgamma, dbeta, B, H, W);   \
  }
    switch (E / 16) {
      case 2: CALL2(2) break;
      case 4: CALL2(4) break;
      case 6: CALL2(6) break;
      case 8: CALL2(8) break;
      case 12: CALL2(12) break;
      default: return ESVIT_ERR_BAD_ARG;
    }
#undef CALL2
    ESVIT_LAUNCH_CHECK();
  }
  const long long ngroups = (long long)B * (H / 4) * ((W / 4 + 7) / 8);
  long long need = (ngroups + 3) / 4, cap = (long long)esvit_num_sms() * 2;
  const int grid = (int)(need < cap ? need : cap);
  const size_t smem = (size_t)(2 * PE_K + 3) * E * sizeof(float);
#define CALL(EJ)                                                                                                   \
  {                                                                                                                \
    cudaError_t e = cudaFuncSetAttribute(patch_embed_bwd_kernel<EJ>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                         (int)smem);                                                               \
    if (e != cudaSuccess) return (int)e;                                                                           \
    patch_embed_bwd_kernel<EJ><<<grid, 128, smem, (cudaStream_t)stream>>>(img, w, bias, gamma, mean, rstd, dout,   \
                                                                          dw, dbias, dgamma, dbeta, B, H, W, E);   \
  }
  PE_DISPATCH(E, CALL)
#undef CALL
  ESVIT_LAUNCH_CHECK();
}
