// CvT-specific kernels (models/cvt_v4_transformer.py): the convolutional token embedding's patch gather and its
// transpose, and the depthwise 3x3 conv + BatchNorm2d in front of the qkv projection, forward and backward.  The
// BatchNorm1d + GELU of a DINOHead(use_bn=True) (models/vision_transformer.py:389-397) shares their statistics, running-
// statistics and coefficient arithmetic (esvit_headbn_*, at the end of this file).
//
// Conv embed (ConvEmbed :349-382): Conv2d(k, stride, pad) = im2col rows bf16 [B*Ho*Wo, Kp] in the weight's (c, ky, kx)
// order (columns >= Cin*k*k are zero, Kp % 8 == 0 for the TMA row pitch) + the bias-epilogue GEMM.  The input is the fp32
// NCHW crop (stage 0) or the fp32 token-major residual stream [B*H*W, Cin] (later stages).  col2im is the input gradient
// as a gather: every input element sums its (at most k*k) row entries in (ky, kx) order, no atomics.
//
// Depthwise + BN (Attention :170-180, DepthWiseConv2d :101-105): y bf16 [B*H*W, C] (the PreNorm output) zero-padded
// right / bottom to Hp x Wp, dw 3x3 conv with pad 1 -> z bf16 [B*Hp*Wp, C] -> BatchNorm2d -> bf16 [B*Hp*Wp, C] for the pw
// GEMM.  Train mode: batch statistics over all B*Hp*Wp positions (padded ones included), the running statistics updated
// in place (momentum, unbiased variance, num_batches_tracked += 1).  Eval mode: the running statistics.
// Reductions: per 256-position chunk in registers + fixed-order block reduce -> fp32 partials [chunk][R][C] -> one
// fixed-order fold in fp64.  No floating-point atomics anywhere, so every result is bit-reproducible.  The folded sums
// (with the element count at [R*C]) are what a SyncBatchNorm all-reduces between the *_stats and *_apply calls.
#include "common.cuh"

namespace cvt {

constexpr int PCH = 256;   // positions per reduction chunk
constexpr int NT = 256;    // threads of the chunk kernels: 64 channels x 4 position lanes

__device__ __forceinline__ float ld(const bf16* p) { return __bfloat162float(*p); }

// NCHW source (the stage-0 crops): one element per thread, consecutive threads walk kx along a row of the image
__global__ void im2col_kernel(const float* __restrict__ x, bf16* __restrict__ rows, int C, int H, int W, int k, int s,
                              int pad, int Ho, int Wo, int Kp, long long total) {
  const int kk = k * k, K = C * kk;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % Kp);
    const long long row = i / Kp;
    float v = 0.f;
    if (col < K) {
      const int c = col / kk, t = col - c * kk, ky = t / k, kx = t - ky * k;
      const long long b = row / ((long long)Ho * Wo);
      const int r = (int)(row - b * Ho * Wo), oy = r / Wo, ox = r - oy * Wo;
      const int iy = oy * s - pad + ky, ix = ox * s - pad + kx;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W)
        v = x[((b * C + c) * H + iy) * W + ix];
    }
    rows[i] = __float2bfloat16(v);
  }
}

// token-major source: one output row per block iteration, staged in shared memory.  The gather reads each tap's C
// contiguous channels (coalesced), the row goes out contiguous in (c, ky, kx) order.
__global__ void __launch_bounds__(256) im2col_tokens_kernel(const float* __restrict__ x, bf16* __restrict__ rows, int C,
                                                            int H, int W, int k, int s, int pad, int Ho, int Wo, int Kp,
                                                            long long nrows) {
  extern __shared__ bf16 srow[];   // [Kp]
  const int kk = k * k, K = C * kk;
  for (long long row = blockIdx.x; row < nrows; row += gridDim.x) {
    const long long b = row / ((long long)Ho * Wo);
    const int r = (int)(row - b * Ho * Wo), oy = r / Wo, ox = r - oy * Wo;
    for (int e = threadIdx.x; e < K; e += blockDim.x) {
      const int t = e / C, c = e - t * C, ky = t / k, kx = t - ky * k;
      const int iy = oy * s - pad + ky, ix = ox * s - pad + kx;
      const float v = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? x[((b * H + iy) * W + ix) * C + c] : 0.f;
      srow[c * kk + t] = __float2bfloat16(v);
    }
    __syncthreads();
    for (int col = threadIdx.x; col < Kp; col += blockDim.x)
      rows[row * Kp + col] = col < K ? srow[col] : __float2bfloat16(0.f);
    __syncthreads();
  }
}

__global__ void col2im_kernel(const bf16* __restrict__ rows, float* __restrict__ dx, int C, int H, int W, int k, int s,
                              int pad, int Ho, int Wo, int Kp, long long total) {
  const int kk = k * k;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long pix = i / C;
    const long long b = pix / ((long long)H * W);
    const int r = (int)(pix - b * H * W), y = r / W, x = r - y * W;
    float sum = 0.f;
    for (int ky = 0; ky < k; ky++) {
      const int ty = y + pad - ky;
      if (ty < 0 || ty % s) continue;
      const int oy = ty / s;
      if (oy >= Ho) continue;
      for (int kx = 0; kx < k; kx++) {
        const int tx = x + pad - kx;
        if (tx < 0 || tx % s) continue;
        const int ox = tx / s;
        if (ox >= Wo) continue;
        sum += ld(rows + ((b * Ho + oy) * Wo + ox) * Kp + c * kk + ky * k + kx);
      }
    }
    dx[i] = sum;
  }
}

struct Geo {
  int H, W, Hp, Wp, C;
  long long N;   // B * Hp * Wp
};

// value of the zero-padded PreNorm output at padded-map coordinates (b, iy, ix): 0 outside [0, H) x [0, W)
__device__ __forceinline__ float ypad(const bf16* __restrict__ y, const Geo& g, long long b, int iy, int ix, int c) {
  return (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) ? ld(y + ((b * g.H + iy) * g.W + ix) * g.C + c) : 0.f;
}

// fixed-order reduction of v[R] over the 4 position lanes of the block -> part[chunk][R][C]
template <int R>
__device__ __forceinline__ void block_partials(const float (&v)[R], float* __restrict__ part, int C) {
  __shared__ float red[R][NT];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
#pragma unroll
  for (int r = 0; r < R; r++) red[r][threadIdx.x] = v[r];
  __syncthreads();
  if (ty == 0) {
#pragma unroll
    for (int r = 0; r < R; r++)
      part[((long long)blockIdx.x * R + r) * C + c] =
          ((red[r][tx] + red[r][64 + tx]) + red[r][128 + tx]) + red[r][192 + tx];
  }
}

__global__ void __launch_bounds__(NT, 4) dw_fwd_kernel(const bf16* __restrict__ y, const float* __restrict__ w,
                                                    bf16* __restrict__ z, float* __restrict__ part, Geo g) {
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
  float wr[9];
#pragma unroll
  for (int t = 0; t < 9; t++) wr[t] = w[c * 9 + t];
  float v[2] = {0.f, 0.f};
  const int p0 = blockIdx.x * PCH, hw = g.Hp * g.Wp;
  for (int i = ty; i < PCH; i += 4) {
    const int p = p0 + i;   // geo_ok: B * Hp * Wp < 2^31
    if (p >= g.N) break;
    const int b = p / hw, r = p - b * hw, py = r / g.Wp, px = r - py * g.Wp;
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 9; t++) acc = fmaf(wr[t], ypad(y, g, b, py + t / 3 - 1, px + t % 3 - 1, c), acc);
    const bf16 zb = __float2bfloat16(acc);
    z[(long long)p * g.C + c] = zb;
    const float zf = __bfloat162float(zb);   // statistics of the stored (bf16) conv output
    v[0] += zf;
    v[1] = fmaf(zf, zf, v[1]);
  }
  block_partials<2>(v, part, g.C);
}

// part [nchunk][R][C] -> sums fp64 [R][C] (+ count at [R*C]); acc0 / acc1 (fp32 [C]) += rows 0 / 1; acc_cr (fp32 [C][R])
// += the transpose.  Chunk j of element e is added by thread (e, j % 8) in increasing j; the 8 lanes combine in order.
__global__ void __launch_bounds__(256) fold_kernel(const float* __restrict__ part, int nchunk, int R, int C,
                                                   double* __restrict__ sums, double count, float* __restrict__ acc0,
                                                   float* __restrict__ acc1, float* __restrict__ acc_cr) {
  __shared__ double red[8][32];
  const int cl = threadIdx.x & 31, j = threadIdx.x >> 5;
  const int e = blockIdx.x * 32 + cl, RC = R * C;
  double a = 0.0;
  if (e < RC)
    for (int ch = j; ch < nchunk; ch += 8) a += (double)part[(long long)ch * RC + e];
  red[j][cl] = a;
  __syncthreads();
  if (j == 0 && e < RC) {
    double tot = red[0][cl];
#pragma unroll
    for (int q = 1; q < 8; q++) tot += red[q][cl];
    const int r = e / C, c = e - r * C;
    if (sums) sums[e] = tot;
    if (acc0 && r == 0) acc0[c] += (float)tot;
    if (acc1 && r == 1) acc1[c] += (float)tot;
    if (acc_cr) acc_cr[c * R + r] += (float)tot;
  }
  if (sums && blockIdx.x == 0 && threadIdx.x == 0) sums[RC] = count;
}

// stat fp32 [4][C] = (mean, rstd, scale = gamma rstd, shift = beta - mean scale)
__global__ void bn_finalize_kernel(const double* __restrict__ sums, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float* __restrict__ rm, float* __restrict__ rv,
                                   long long* __restrict__ nbt, float* __restrict__ stat, int C, int train, float momentum,
                                   float eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double mean, var;
  if (train) {
    const double n = sums[2 * C];
    mean = sums[c] / n;
    var = fmax(sums[C + c] / n - mean * mean, 0.0);
    if (rm) {
      const double unb = n > 1.0 ? var * n / (n - 1.0) : var;
      rm[c] = (1.f - momentum) * rm[c] + momentum * (float)mean;
      rv[c] = (1.f - momentum) * rv[c] + momentum * (float)unb;
    }
    if (nbt && c == 0) nbt[0] += 1;
  } else {
    mean = rm[c];
    var = rv[c];
  }
  const float rstd = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = gamma[c] * rstd;
  stat[c] = (float)mean;
  stat[C + c] = rstd;
  stat[2 * C + c] = sc;
  stat[3 * C + c] = beta[c] - (float)mean * sc;
}

template <bool GELU>
__global__ void bn_normalize_kernel(const bf16* __restrict__ z, const float* __restrict__ stat, bf16* __restrict__ out,
                                    int C, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)((i * 8) % C);
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(z)[i], f);
#pragma unroll
    for (int q = 0; q < 8; q++) {
      f[q] = fmaf(f[q], stat[2 * C + c0 + q], stat[3 * C + c0 + q]);
      if (GELU) f[q] = gelu_f(f[q]);
    }
    reinterpret_cast<bf16x8*>(out)[i] = pack8(f);
  }
}

// gradient at the BN output: dy, or (GELU) dy * gelu'(z scale + shift) for the BN + GELU of the DINO head
template <bool GELU>
__device__ __forceinline__ float bn_dout(float dy, float z, float sc, float sh) {
  return GELU ? dy * gelu_grad_f(fmaf(z, sc, sh)) : dy;
}

// partials of (sum dy, sum dy * xhat) per channel
template <bool GELU>
__global__ void __launch_bounds__(NT) bn_bwd_partials_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z,
                                                             const float* __restrict__ stat, float* __restrict__ part,
                                                             long long N, int C) {
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
  const float mean = stat[c], rstd = stat[C + c], sc = stat[2 * C + c], sh = stat[3 * C + c];
  float v[2] = {0.f, 0.f};
  const long long p0 = (long long)blockIdx.x * PCH;
  for (int i = ty; i < PCH; i += 4) {
    const long long p = p0 + i;
    if (p >= N) break;
    const float zv = ld(z + p * C + c);
    const float g = bn_dout<GELU>(ld(dy + p * C + c), zv, sc, sh), xh = (zv - mean) * rstd;
    v[0] += g;
    v[1] = fmaf(g, xh, v[1]);
  }
  block_partials<2>(v, part, C);
}

// dz = coef0 dy + coef1 z + coef2: train = gamma rstd (dy - mean(dy) - xhat mean(dy xhat)); eval = gamma rstd dy
__global__ void bn_bwd_coef_kernel(const double* __restrict__ sums, const float* __restrict__ stat, float* __restrict__ coef,
                                   int C, int train) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float mean = stat[c], rstd = stat[C + c], sc = stat[2 * C + c];
  if (train) {
    const double n = sums[2 * C];
    const float mdy = (float)(sums[c] / n), mdx = (float)(sums[C + c] / n);
    coef[c] = sc;
    coef[C + c] = -sc * rstd * mdx;
    coef[2 * C + c] = sc * (rstd * mdx * mean - mdy);
  } else {
    coef[c] = sc;
    coef[C + c] = 0.f;
    coef[2 * C + c] = 0.f;
  }
}

__device__ __forceinline__ float dz_at(const bf16* __restrict__ dy, const bf16* __restrict__ z, long long off, float c0,
                                       float c1, float c2) {
  return fmaf(c0, ld(dy + off), fmaf(c1, ld(z + off), c2));
}

// input gradient of the dw conv on the unpadded map: dx(q) = sum_t w[t] dz(q - t + 1), taps in order
__global__ void dw_bwd_dx_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z, const float* __restrict__ w,
                                 const float* __restrict__ coef, bf16* __restrict__ dx, Geo g, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % g.C);
    const long long pix = i / g.C;
    const long long b = pix / ((long long)g.H * g.W);
    const int r = (int)(pix - b * g.H * g.W), y = r / g.W, x = r - y * g.W;
    const float c0 = coef[c], c1 = coef[g.C + c], c2 = coef[2 * g.C + c];
    float sum = 0.f;
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const int py = y + 1 - t / 3, px = x + 1 - t % 3;
      if (py < 0 || py >= g.Hp || px < 0 || px >= g.Wp) continue;
      const long long off = ((b * g.Hp + py) * g.Wp + px) * g.C + c;
      sum = fmaf(w[c * 9 + t], dz_at(dy, z, off, c0, c1, c2), sum);
    }
    dx[i] = __float2bfloat16(sum);
  }
}

// filter-gradient partials: sum over the chunk's positions p of dz(p) * ypad(p + t - 1) for the 9 taps
__global__ void __launch_bounds__(NT) dw_bwd_w_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z,
                                                      const bf16* __restrict__ y, const float* __restrict__ coef,
                                                      float* __restrict__ part, Geo g) {
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
  const float c0 = coef[c], c1 = coef[g.C + c], c2 = coef[2 * g.C + c];
  float v[9];
#pragma unroll
  for (int t = 0; t < 9; t++) v[t] = 0.f;
  const int p0 = blockIdx.x * PCH, hw = g.Hp * g.Wp;
  for (int i = ty; i < PCH; i += 4) {
    const int p = p0 + i;   // geo_ok: B * Hp * Wp < 2^31
    if (p >= g.N) break;
    const int b = p / hw, r = p - b * hw, py = r / g.Wp, px = r - py * g.Wp;
    const float d = dz_at(dy, z, (long long)p * g.C + c, c0, c1, c2);
#pragma unroll
    for (int t = 0; t < 9; t++) v[t] = fmaf(d, ypad(y, g, b, py + t / 3 - 1, px + t % 3 - 1, c), v[t]);
  }
  block_partials<9>(v, part, g.C);
}

// DINO head BN: per-column sums of z bf16 [N, C] (the bias-GEMM output) and of z^2
__global__ void __launch_bounds__(NT) head_stats_kernel(const bf16* __restrict__ z, float* __restrict__ part, long long N,
                                                        int C) {
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
  float v[2] = {0.f, 0.f};
  const long long p0 = (long long)blockIdx.x * PCH;
  for (int i = ty; i < PCH; i += 4) {
    const long long p = p0 + i;
    if (p >= N) break;
    const float zv = ld(z + p * C + c);
    v[0] += zv;
    v[1] = fmaf(zv, zv, v[1]);
  }
  block_partials<2>(v, part, C);
}

// DINO head BN backward: dz = coef0 gelu'(u) dy + coef1 z + coef2 (bf16, the GEMM operand of dx / dW) and the partials
// of its column sums (the gradient of the Linear's bias)
__global__ void __launch_bounds__(NT) head_bwd_dz_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ z,
                                                         const float* __restrict__ stat, const float* __restrict__ coef,
                                                         bf16* __restrict__ dz, float* __restrict__ part, long long N,
                                                         int C) {
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6, c = blockIdx.y * 64 + tx;
  const float sc = stat[2 * C + c], sh = stat[3 * C + c];
  const float c0 = coef[c], c1 = coef[C + c], c2 = coef[2 * C + c];
  float v[1] = {0.f};
  const long long p0 = (long long)blockIdx.x * PCH;
  for (int i = ty; i < PCH; i += 4) {
    const long long p = p0 + i;
    if (p >= N) break;
    const float zv = ld(z + p * C + c);
    const float d = fmaf(c0, bn_dout<true>(ld(dy + p * C + c), zv, sc, sh), fmaf(c1, zv, c2));
    dz[p * C + c] = __float2bfloat16(d);
    v[0] += d;
  }
  block_partials<1>(v, part, C);
}

static unsigned grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)esvit_num_sms() * 32;
  return (unsigned)(b < cap ? (b > 0 ? b : 1) : cap);
}

static bool geo_ok(int B, int H, int W, int Hp, int Wp, int C, Geo* g) {
  if (B < 1 || H < 1 || W < 1 || Hp < H || Wp < W || Hp > H + 63 || Wp > W + 63 || C < 64 || C % 64) return false;
  g->H = H; g->W = W; g->Hp = Hp; g->Wp = Wp; g->C = C;
  g->N = (long long)B * Hp * Wp;
  return g->N < (1LL << 31) - PCH;
}

static cudaError_t fold(const float* part, long long nchunk, int R, int C, double* sums, double count, float* acc0,
                        float* acc1, float* acc_cr, cudaStream_t st) {
  fold_kernel<<<(R * C + 31) / 32, 256, 0, st>>>(part, (int)nchunk, R, C, sums, count, acc0, acc1, acc_cr);
  return cudaGetLastError();
}

}  // namespace cvt

ESVIT_API int esvit_conv_im2col(const float* x, void* rows, int nchw, int B, int C, int H, int W, int k, int stride,
                                int pad, int Kp, void* stream) {
  if (!x || !rows || B < 1 || C < 1 || H < 1 || W < 1 || k < 1 || stride < 1 || pad < 0 || Kp < C * k * k || Kp % 8)
    return ESVIT_ERR_BAD_ARG;
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  if (Ho < 1 || Wo < 1) return ESVIT_ERR_BAD_ARG;
  if (nchw) {
    const long long total = (long long)B * Ho * Wo * Kp;
    cvt::im2col_kernel<<<cvt::grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, (bf16*)rows, C, H, W, k, stride,
                                                                                     pad, Ho, Wo, Kp, total);
  } else {
    if ((size_t)Kp * sizeof(bf16) > 48 * 1024) return ESVIT_ERR_BAD_ARG;
    const long long nrows = (long long)B * Ho * Wo;
    const long long cap = (long long)esvit_num_sms() * 8;
    cvt::im2col_tokens_kernel<<<(unsigned)(nrows < cap ? nrows : cap), 256, Kp * sizeof(bf16), (cudaStream_t)stream>>>(
        x, (bf16*)rows, C, H, W, k, stride, pad, Ho, Wo, Kp, nrows);
  }
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_conv_col2im(const void* rows, float* dx, int B, int C, int H, int W, int k, int stride, int pad, int Kp,
                                void* stream) {
  if (!rows || !dx || B < 1 || C < 1 || H < 1 || W < 1 || k < 1 || stride < 1 || pad < 0 || Kp < C * k * k || Kp % 8)
    return ESVIT_ERR_BAD_ARG;
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  if (Ho < 1 || Wo < 1) return ESVIT_ERR_BAD_ARG;
  const long long total = (long long)B * H * W * C;
  cvt::col2im_kernel<<<cvt::grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)rows, dx, C, H, W, k, stride,
                                                                                   pad, Ho, Wo, Kp, total);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dwbn_fwd_stats(const void* y, const float* w, void* z, float* part, double* sums, int B, int H, int W,
                                   int Hp, int Wp, int C, void* stream) {
  cvt::Geo g;
  if (!y || !w || !z || !part || !sums || !cvt::geo_ok(B, H, W, Hp, Wp, C, &g)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long nchunk = (g.N + cvt::PCH - 1) / cvt::PCH;
  cvt::dw_fwd_kernel<<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)y, w, (bf16*)z, part, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 2, C, sums, (double)g.N, nullptr, nullptr, nullptr, st);
}

ESVIT_API int esvit_dwbn_fwd_apply(const void* z, const float* gamma, const float* beta, const double* sums,
                                   float* run_mean, float* run_var, long long* nbt, float* stat, void* out, long long N,
                                   int C, int train, float momentum, float eps, void* stream) {
  if (!z || !gamma || !beta || !stat || !out || N < 1 || C < 64 || C % 64 || (train && !sums) ||
      (!train && (!run_mean || !run_var)) || ((run_mean == nullptr) != (run_var == nullptr)))
    return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cvt::bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, gamma, beta, run_mean, run_var, nbt, stat, C, train,
                                                           momentum, eps);
  const long long n8 = N * C / 8;
  cvt::bn_normalize_kernel<false><<<cvt::grid_for(n8, 256), 256, 0, st>>>((const bf16*)z, stat, (bf16*)out, C, n8);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dwbn_bwd_stats(const void* dy, const void* z, const float* stat, float* part, double* sums,
                                   float* dgamma, float* dbeta, long long N, int C, void* stream) {
  if (!dy || !z || !stat || !part || !sums || N < 1 || C < 64 || C % 64) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long nchunk = (N + cvt::PCH - 1) / cvt::PCH;
  if (nchunk >= (1LL << 31)) return ESVIT_ERR_BAD_ARG;
  cvt::bn_bwd_partials_kernel<false><<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)dy, (const bf16*)z,
                                                                                        stat, part, N, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 2, C, sums, (double)N, dbeta, dgamma, nullptr, st);
}

ESVIT_API int esvit_dwbn_bwd_apply(const void* dy, const void* z, const void* y, const float* w, const float* stat,
                                   const double* sums, float* coef, void* dx, float* part, float* dw, int B, int H, int W,
                                   int Hp, int Wp, int C, int train, void* stream) {
  cvt::Geo g;
  if (!dy || !z || !y || !w || !stat || !coef || !dx || !part || !dw || (train && !sums) ||
      !cvt::geo_ok(B, H, W, Hp, Wp, C, &g))
    return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cvt::bn_bwd_coef_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, stat, coef, C, train);
  const long long total = (long long)B * H * W * C;
  cvt::dw_bwd_dx_kernel<<<cvt::grid_for(total, 256), 256, 0, st>>>((const bf16*)dy, (const bf16*)z, w, coef, (bf16*)dx, g,
                                                                   total);
  const long long nchunk = (g.N + cvt::PCH - 1) / cvt::PCH;
  cvt::dw_bwd_w_kernel<<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)dy, (const bf16*)z, (const bf16*)y,
                                                                          coef, part, g);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 9, C, nullptr, 0.0, nullptr, nullptr, dw, st);
}

// ---- DINOHead(use_bn=True): Linear -> BatchNorm1d -> GELU on rows z bf16 [N, C] (the bias-GEMM output) ----------------

static bool head_ok(long long N, int C) {
  return N >= 1 && C >= 64 && C % 64 == 0 && (N + cvt::PCH - 1) / cvt::PCH < (1LL << 31);
}

ESVIT_API int esvit_headbn_fwd_stats(const void* z, float* part, double* sums, long long N, int C, void* stream) {
  if (!z || !part || !sums || !head_ok(N, C)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long nchunk = (N + cvt::PCH - 1) / cvt::PCH;
  cvt::head_stats_kernel<<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)z, part, N, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 2, C, sums, (double)N, nullptr, nullptr, nullptr, st);
}

ESVIT_API int esvit_headbn_fwd_apply(const void* z, const float* gamma, const float* beta, const double* sums,
                                     float* run_mean, float* run_var, long long* nbt, float* stat, void* out, long long N,
                                     int C, int train, float momentum, float eps, void* stream) {
  if (!z || !gamma || !beta || !stat || !out || !head_ok(N, C) || (train && !sums) ||
      (!train && (!run_mean || !run_var)) || ((run_mean == nullptr) != (run_var == nullptr)))
    return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cvt::bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, gamma, beta, run_mean, run_var, nbt, stat, C, train,
                                                           momentum, eps);
  const long long n8 = N * C / 8;
  cvt::bn_normalize_kernel<true><<<cvt::grid_for(n8, 256), 256, 0, st>>>((const bf16*)z, stat, (bf16*)out, C, n8);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_headbn_bwd_stats(const void* dy, const void* z, const float* stat, float* part, double* sums,
                                     float* dgamma, float* dbeta, long long N, int C, void* stream) {
  if (!dy || !z || !stat || !part || !sums || !head_ok(N, C)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long nchunk = (N + cvt::PCH - 1) / cvt::PCH;
  cvt::bn_bwd_partials_kernel<true><<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)dy, (const bf16*)z,
                                                                                       stat, part, N, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 2, C, sums, (double)N, dbeta, dgamma, nullptr, st);
}

ESVIT_API int esvit_headbn_bwd_apply(const void* dy, const void* z, const float* stat, const double* sums, float* coef,
                                     void* dz, float* part, float* dbias, long long N, int C, int train, void* stream) {
  if (!dy || !z || !stat || !coef || !dz || !part || !dbias || (train && !sums) || !head_ok(N, C))
    return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  cvt::bn_bwd_coef_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums, stat, coef, C, train);
  const long long nchunk = (N + cvt::PCH - 1) / cvt::PCH;
  cvt::head_bwd_dz_kernel<<<dim3((unsigned)nchunk, C / 64), cvt::NT, 0, st>>>((const bf16*)dy, (const bf16*)z, stat, coef,
                                                                             (bf16*)dz, part, N, C);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  return (int)cvt::fold(part, nchunk, 1, C, nullptr, 0.0, dbias, nullptr, nullptr, st);
}
