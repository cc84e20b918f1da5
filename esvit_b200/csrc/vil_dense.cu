// Vision Longformer pieces around the sliding-chunk attention (vil_attn.cu): the dense stages' biased attention, the
// token-stream patch embedding, the global-token assembly and the relative-position bias assembly.
//
// Reference: models/vision_longformer.py  Attention.forward :86-131, PatchEmbed.forward :227-259, MsViT.forward_features
// :581-605 (the global row dropped before the next stage's conv).
//
// Dense attention at head dim 32 with an additive fp32 bias [nH, L, L] (L <= 256; the step runs L = 197 / 37 in stage 3
// and 49 / 9 in stage 4).  qkv bf16 [B*L, 3C] token-major as the qkv GEMM writes it (channel order [q|k|v][head][32]),
// out bf16 [B*L, C], lse fp32 [B, nH, L].  One thread owns one query row (forward, dq) or one key row (dk / dv); the
// K / V (or Q / dO) rows of one (image, head) sit in shared memory as fp32 and every thread streams through them.
// The scores are fp32 (scale * q.k + bias), softmax in fp32.
//
// Backward, without floating-point atomics:
//   dq    CTA = (64 query rows, head, part p): images b = p, p + P, ... in increasing order; writes D = rowsum(dO * O)
//         and dq, and sums dS over its images into a shared-memory row per thread, stored as part[p, h, i, :]
//   dkdv  CTA = (64 key rows, head, image): loops over every query of the image
//   dbias = sum_p part[p] in increasing p (esvit_vil_dense_bwd runs all three kernels)
// so dq / dk / dv / dbias are bit-identical from run to run.
#include "common.cuh"

namespace vd {

constexpr int HD = 32;
constexpr int ROWS = 64;     // threads per CTA = rows per CTA
constexpr int MAXL = 256;

__device__ __forceinline__ void load_row(float (&r)[HD], const bf16* __restrict__ p, float s) {
#pragma unroll
  for (int k = 0; k < HD / 8; k++) {
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(p)[k], f);
#pragma unroll
    for (int e = 0; e < 8; e++) r[k * 8 + e] = f[e] * s;
  }
}

// rows [0, L) of one head's 32 columns (source row stride ld) -> fp32 smem [L][32]
__device__ __forceinline__ void stage_rows(float* __restrict__ dst, const bf16* __restrict__ src, long long ld, int L) {
  for (int e = threadIdx.x; e < L * (HD / 8); e += blockDim.x) {
    const int r = e / (HD / 8), k = e % (HD / 8);
    float f[8];
    unpack8(reinterpret_cast<const bf16x8*>(src + (long long)r * ld)[k], f);
    float4* d = reinterpret_cast<float4*>(dst + r * HD + k * 8);
    d[0] = make_float4(f[0], f[1], f[2], f[3]);
    d[1] = make_float4(f[4], f[5], f[6], f[7]);
  }
}

__device__ __forceinline__ float dot_s(const float (&a)[HD], const float* __restrict__ row) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < HD; k += 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + k);
    s = fmaf(a[k], v.x, s);
    s = fmaf(a[k + 1], v.y, s);
    s = fmaf(a[k + 2], v.z, s);
    s = fmaf(a[k + 3], v.w, s);
  }
  return s;
}

__device__ __forceinline__ void axpy_s(float (&acc)[HD], float w, const float* __restrict__ row) {
#pragma unroll
  for (int k = 0; k < HD; k += 4) {
    const float4 v = *reinterpret_cast<const float4*>(row + k);
    acc[k] = fmaf(w, v.x, acc[k]);
    acc[k + 1] = fmaf(w, v.y, acc[k + 1]);
    acc[k + 2] = fmaf(w, v.z, acc[k + 2]);
    acc[k + 3] = fmaf(w, v.w, acc[k + 3]);
  }
}

__device__ __forceinline__ void store_row(bf16* __restrict__ p, const float (&r)[HD], float s) {
#pragma unroll
  for (int k = 0; k < HD / 8; k++) {
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; e++) f[e] = r[k * 8 + e] * s;
    reinterpret_cast<bf16x8*>(p)[k] = pack8(f);
  }
}

__global__ void __launch_bounds__(ROWS) dense_fwd_kernel(const bf16* __restrict__ qkv, const float* __restrict__ bias,
                                                         bf16* __restrict__ out, float* __restrict__ lse, int L, int C,
                                                         int nH, float scale) {
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;
  float* Vs = sm + L * HD;
  const int h = blockIdx.y, b = blockIdx.z, i = blockIdx.x * ROWS + threadIdx.x;
  const long long C3 = 3LL * C;
  const bf16* base = qkv + (long long)b * L * C3 + h * HD;
  stage_rows(Ks, base + C, C3, L);
  stage_rows(Vs, base + 2 * C, C3, L);
  __syncthreads();
  if (i >= L) return;
  float q[HD], o[HD];
  load_row(q, base + (long long)i * C3, scale);
#pragma unroll
  for (int k = 0; k < HD; k++) o[k] = 0.f;
  const float* brow = bias + ((long long)h * L + i) * L;
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < L; j0 += 8) {
    float s[8];
    float mx = m;
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int j = j0 + u;
      s[u] = j < L ? dot_s(q, Ks + j * HD) + brow[j] : -INFINITY;
      mx = fmaxf(mx, s[u]);
    }
    const float a = __expf(m - mx);  // m = -inf on the first chunk: a = 0
    l *= a;
#pragma unroll
    for (int k = 0; k < HD; k++) o[k] *= a;
#pragma unroll
    for (int u = 0; u < 8; u++) {
      const int j = j0 + u;
      if (j < L) {
        const float p = __expf(s[u] - mx);
        l += p;
        axpy_s(o, p, Vs + j * HD);
      }
    }
    m = mx;
  }
  store_row(out + ((long long)b * L + i) * C + h * HD, o, 1.f / l);
  lse[((long long)b * nH + h) * L + i] = m + __logf(l);
}

// dq of 64 query rows over the images b = part, part + nparts, ...; D = rowsum(dO * O) to dvec; sum_b dS to part rows
__global__ void __launch_bounds__(ROWS) dense_dq_kernel(const bf16* __restrict__ qkv, const float* __restrict__ bias,
                                                        const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                                        const float* __restrict__ lse, float* __restrict__ dvec,
                                                        bf16* __restrict__ dqkv, float* __restrict__ part, int B, int L,
                                                        int C, int nH, float scale, int nparts) {
  extern __shared__ __align__(16) float sm[];
  float* Ks = sm;
  float* Vs = sm + L * HD;
  float* acc = sm + 2 * L * HD + threadIdx.x * L;  // this thread's dS row sum (stride L is odd for every step geometry)
  const int h = blockIdx.y, p = blockIdx.z, i = blockIdx.x * ROWS + threadIdx.x;
  const long long C3 = 3LL * C;
  if (i < L)
    for (int j = 0; j < L; j++) acc[j] = 0.f;
  const float* brow = bias + ((long long)h * L + (i < L ? i : 0)) * L;
  for (int b = p; b < B; b += nparts) {
    const bf16* base = qkv + (long long)b * L * C3 + h * HD;
    __syncthreads();  // the previous image's rows are no longer read
    stage_rows(Ks, base + C, C3, L);
    stage_rows(Vs, base + 2 * C, C3, L);
    __syncthreads();
    if (i < L) {
      float q[HD], g[HD], dq[HD];
      load_row(q, base + (long long)i * C3, scale);
      const long long orow = ((long long)b * L + i) * C + h * HD;
      load_row(g, dout + orow, 1.f);
      load_row(dq, out + orow, 1.f);
      float D = 0.f;
#pragma unroll
      for (int k = 0; k < HD; k++) D = fmaf(g[k], dq[k], D);
#pragma unroll
      for (int k = 0; k < HD; k++) dq[k] = 0.f;
      const long long si = ((long long)b * nH + h) * L + i;
      dvec[si] = D;
      const float li = lse[si];
      for (int j = 0; j < L; j++) {
        const float pr = __expf(dot_s(q, Ks + j * HD) + brow[j] - li);
        const float ds = pr * (dot_s(g, Vs + j * HD) - D);
        acc[j] += ds;
        axpy_s(dq, ds, Ks + j * HD);
      }
      store_row(dqkv + ((long long)b * L + i) * C3 + h * HD, dq, scale);
    }
  }
  if (i < L) {
    float* dst = part + (((long long)p * nH + h) * L + i) * L;
    for (int j = 0; j < L; j++) dst[j] = acc[j];
  }
}

// dk, dv of 64 key rows of one image; D from dense_dq_kernel
__global__ void __launch_bounds__(ROWS) dense_dkdv_kernel(const bf16* __restrict__ qkv, const float* __restrict__ bias,
                                                          const bf16* __restrict__ dout, const float* __restrict__ lse,
                                                          const float* __restrict__ dvec, bf16* __restrict__ dqkv, int L,
                                                          int C, int nH, float scale) {
  extern __shared__ __align__(16) float sm[];
  float* Qs = sm;
  float* Gs = sm + L * HD;
  float* ls = sm + 2 * L * HD;
  float* Ds = ls + L;
  const int h = blockIdx.y, b = blockIdx.z, j = blockIdx.x * ROWS + threadIdx.x;
  const long long C3 = 3LL * C;
  const bf16* base = qkv + (long long)b * L * C3 + h * HD;
  stage_rows(Qs, base, C3, L);
  stage_rows(Gs, dout + (long long)b * L * C + h * HD, C, L);
  for (int e = threadIdx.x; e < L; e += blockDim.x) {
    const long long si = ((long long)b * nH + h) * L + e;
    ls[e] = lse[si];
    Ds[e] = dvec[si];
  }
  __syncthreads();
  if (j >= L) return;
  float k[HD], v[HD], dk[HD], dv[HD];
  load_row(k, base + C + (long long)j * C3, scale);  // q . (scale k) = scale q . k
  load_row(v, base + 2 * C + (long long)j * C3, 1.f);
#pragma unroll
  for (int e = 0; e < HD; e++) dk[e] = dv[e] = 0.f;
  const float* bcol = bias + (long long)h * L * L + j;
  for (int i = 0; i < L; i++) {
    const float pr = __expf(dot_s(k, Qs + i * HD) + bcol[(long long)i * L] - ls[i]);
    axpy_s(dv, pr, Gs + i * HD);
    const float ds = pr * (dot_s(v, Gs + i * HD) - Ds[i]);
    axpy_s(dk, ds, Qs + i * HD);
  }
  bf16* dst = dqkv + ((long long)b * L + j) * C3 + h * HD;
  store_row(dst + C, dk, scale);
  store_row(dst + 2 * C, dv, 1.f);
}

// dbias[e] = sum_p part[p][e], p increasing
__global__ void part_sum_kernel(const float* __restrict__ part, float* __restrict__ dbias, long long n, int nparts) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  float s = 0.f;
  for (int p = 0; p < nparts; p++) s += part[(long long)p * n + e];
  dbias[e] = s;
}

static size_t fwd_smem(int L) { return (size_t)2 * L * HD * sizeof(float); }
static size_t dq_smem(int L) { return (size_t)(2 * L * HD + ROWS * L) * sizeof(float); }
static size_t dkdv_smem(int L) { return (size_t)(2 * L * HD + 2 * L) * sizeof(float); }

template <typename K>
static cudaError_t opt_in(K kernel, size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                          : cudaSuccess;
}

static bool ok_args(int B, int L, int C, int nH) {
  return B >= 1 && B <= 65535 && L >= 1 && L <= MAXL && nH >= 1 && nH <= 65535 && C == nH * HD;
}
static bool al16(const void* p) { return p && ((uintptr_t)p & 15) == 0; }

// ---- stream patch embedding ----------------------------------------------------------------------------------------
// rows[(b, oy, ox), c*p*p + ky*p + kx] = x[b*N + off + (oy*p + ky)*W + ox*p + kx, c]; thread per (row, ky, kx, c)
__global__ void im2col_kernel(const float* __restrict__ x, bf16* __restrict__ rows, int N, int off, int Cin, int W,
                              int Ho, int Wo, int p, int Kp, long long total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % Cin);
  long long t = e / Cin;
  const int kk = (int)(t % (p * p));
  const long long r = t / (p * p);
  const int ky = kk / p, kx = kk % p;
  const int ox = (int)(r % Wo), oy = (int)((r / Wo) % Ho);
  const long long b = r / ((long long)Wo * Ho);
  const float v = x[(b * N + off + (long long)(oy * p + ky) * W + ox * p + kx) * Cin + c];
  rows[r * Kp + (long long)c * p * p + kk] = __float2bfloat16_rn(v);
}

// dx of the whole stream slice [B*N, Cin]: the patch rows' gradient at covered positions, 0 on global rows and at
// positions no patch covers (each position is covered at most once: stride = kernel)
__global__ void col2im_kernel(const bf16* __restrict__ drows, float* __restrict__ dx, int N, int off, int Cin, int W,
                              int Ho, int Wo, int p, int Kp, long long total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % Cin);
  const long long row = e / Cin;
  const int n = (int)(row % N);
  const long long b = row / N;
  float v = 0.f;
  if (n >= off) {
    const int y = (n - off) / W, xx = (n - off) % W;
    const int oy = y / p, ox = xx / p;
    if (oy < Ho && ox < Wo)
      v = __bfloat162float(drows[((b * Ho + oy) * Wo + ox) * Kp + (long long)c * p * p + (y % p) * p + xx % p]);
  }
  dx[e] = v;
}

// ---- global-token assembly -------------------------------------------------------------------------------------------
// out[b*(1+n) + 0] = cls, out[b*(1+n) + 1 + r] = y[b*n + r]
__global__ void cls_cat_fwd_kernel(const float4* __restrict__ y, const float4* __restrict__ cls, float4* __restrict__ out,
                                   int n, int C4, long long total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % C4);
  const long long row = e / C4;
  const int r = (int)(row % (n + 1));
  const long long b = row / (n + 1);
  out[e] = r == 0 ? cls[c] : y[(b * n + r - 1) * C4 + c];
}
__global__ void cls_cat_bwd_rows_kernel(const float4* __restrict__ g, float4* __restrict__ dy, int n, int C4,
                                        long long total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int c = (int)(e % C4);
  const long long row = e / C4;
  const long long b = row / n;
  dy[e] = g[(b * (n + 1) + 1 + row % n) * C4 + c];
}
// dcls[c] (+)= sum_b g[b*(1+n), c], b increasing
__global__ void cls_cat_bwd_cls_kernel(const float* __restrict__ g, float* __restrict__ dcls, int B, int n, int C,
                                       int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = accumulate ? dcls[c] : 0.f;
  for (int b = 0; b < B; b++) s += g[(long long)b * (n + 1) * C + c];
  dcls[c] = s;
}

// ---- relative-position bias assembly -----------------------------------------------------------------------------
// y[r] = sum_{k in [rowptr[r], rowptr[r+1])} val[k] * src(col[k]), k increasing; src(c) = s0[c] (c < n0),
// s1[c - n0] (c < n0 + n1), s2[c - n0 - n1]
__global__ void spmv_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const float* __restrict__ val,
                            const float* __restrict__ s0, const float* __restrict__ s1, const float* __restrict__ s2,
                            int n0, int n1, float* __restrict__ y, int nrows) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nrows) return;
  float s = 0.f;
  for (int k = rowptr[r]; k < rowptr[r + 1]; k++) {
    const int c = col[k];
    const float v = c < n0 ? s0[c] : (c < n0 + n1 ? s1[c - n0] : s2[c - n0 - n1]);
    s = fmaf(val[k], v, s);
  }
  y[r] = s;
}

static unsigned nblk(long long n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace vd

ESVIT_API int esvit_vil_dense_fwd(const void* qkv, const float* bias, void* out, float* lse, int B, int L, int C, int nH,
                                  float scale, void* stream) {
  if (!vd::ok_args(B, L, C, nH) || !vd::al16(qkv) || !vd::al16(out) || !bias || !lse) return ESVIT_ERR_BAD_ARG;
  const size_t smem = vd::fwd_smem(L);
  cudaError_t e = vd::opt_in(vd::dense_fwd_kernel, smem);
  if (e != cudaSuccess) return (int)e;
  const dim3 grid((L + vd::ROWS - 1) / vd::ROWS, nH, B);
  vd::dense_fwd_kernel<<<grid, vd::ROWS, smem, (cudaStream_t)stream>>>((const bf16*)qkv, bias, (bf16*)out, lse, L, C, nH,
                                                                       scale);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_dense_parts(int B) { return B < 16 ? B : 16; }

ESVIT_API int esvit_vil_dense_bwd(const void* qkv, const float* bias, const void* out, const void* dout, const float* lse,
                                  float* dvec, float* part, void* dqkv, float* dbias, int B, int L, int C, int nH,
                                  float scale, void* stream) {
  if (!vd::ok_args(B, L, C, nH) || !vd::al16(qkv) || !vd::al16(out) || !vd::al16(dout) || !vd::al16(dqkv) || !bias ||
      !lse || !dvec || !part || !dbias)
    return ESVIT_ERR_BAD_ARG;
  cudaError_t e = vd::opt_in(vd::dense_dq_kernel, vd::dq_smem(L));
  if (e == cudaSuccess) e = vd::opt_in(vd::dense_dkdv_kernel, vd::dkdv_smem(L));
  if (e != cudaSuccess) return (int)e;
  cudaStream_t st = (cudaStream_t)stream;
  const int P = esvit_vil_dense_parts(B);
  const int nb = (L + vd::ROWS - 1) / vd::ROWS;
  vd::dense_dq_kernel<<<dim3(nb, nH, P), vd::ROWS, vd::dq_smem(L), st>>>(
      (const bf16*)qkv, bias, (const bf16*)out, (const bf16*)dout, lse, dvec, (bf16*)dqkv, part, B, L, C, nH, scale, P);
  vd::dense_dkdv_kernel<<<dim3(nb, nH, B), vd::ROWS, vd::dkdv_smem(L), st>>>((const bf16*)qkv, bias, (const bf16*)dout,
                                                                            lse, dvec, (bf16*)dqkv, L, C, nH, scale);
  const long long n = (long long)nH * L * L;
  vd::part_sum_kernel<<<vd::nblk(n, 256), 256, 0, st>>>(part, dbias, n, P);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_im2col(const float* x, void* rows, int B, int N, int off, int Cin, int H, int W, int p, int Kp,
                               void* stream) {
  if (!x || !rows || B < 1 || Cin < 1 || p < 1 || H < p || W < p || off < 0 || N < off + H * W || Kp < Cin * p * p)
    return ESVIT_ERR_BAD_ARG;
  const int Ho = H / p, Wo = W / p;
  const long long total = (long long)B * Ho * Wo * p * p * Cin;
  vd::im2col_kernel<<<vd::nblk(total, 256), 256, 0, (cudaStream_t)stream>>>(x, (bf16*)rows, N, off, Cin, W, Ho, Wo, p,
                                                                             Kp, total);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_col2im(const void* drows, float* dx, int B, int N, int off, int Cin, int H, int W, int p, int Kp,
                               void* stream) {
  if (!drows || !dx || B < 1 || Cin < 1 || p < 1 || H < p || W < p || off < 0 || N < off + H * W || Kp < Cin * p * p)
    return ESVIT_ERR_BAD_ARG;
  const long long total = (long long)B * N * Cin;
  vd::col2im_kernel<<<vd::nblk(total, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)drows, dx, N, off, Cin, W, H / p,
                                                                             W / p, p, Kp, total);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_cls_cat_fwd(const float* y, const float* cls, float* out, int B, int n, int C, void* stream) {
  if (!vd::al16(y) || !vd::al16(cls) || !vd::al16(out) || B < 1 || n < 1 || C < 4 || C % 4) return ESVIT_ERR_BAD_ARG;
  const long long total = (long long)B * (n + 1) * (C / 4);
  vd::cls_cat_fwd_kernel<<<vd::nblk(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const float4*)y, (const float4*)cls, (float4*)out, n, C / 4, total);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_cls_cat_bwd(const float* g, float* dy, float* dcls, int B, int n, int C, int accumulate,
                                    void* stream) {
  if (!vd::al16(g) || !vd::al16(dy) || !dcls || B < 1 || n < 1 || C < 4 || C % 4) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)B * n * (C / 4);
  vd::cls_cat_bwd_rows_kernel<<<vd::nblk(total, 256), 256, 0, st>>>((const float4*)g, (float4*)dy, n, C / 4, total);
  vd::cls_cat_bwd_cls_kernel<<<vd::nblk(C, 128), 128, 0, st>>>(g, dcls, B, n, C, accumulate);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_bias_spmv(const int* rowptr, const int* col, const float* val, const float* s0, const float* s1,
                                  const float* s2, int n0, int n1, float* y, int nrows, void* stream) {
  if (!rowptr || !col || !val || !s0 || !y || nrows < 1 || n0 < 0 || n1 < 0) return ESVIT_ERR_BAD_ARG;
  vd::spmv_kernel<<<vd::nblk(nrows, 256), 256, 0, (cudaStream_t)stream>>>(rowptr, col, val, s0, s1, s2, n0, n1, y,
                                                                           nrows);
  ESVIT_LAUNCH_CHECK();
}
