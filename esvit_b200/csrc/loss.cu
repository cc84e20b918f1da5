// DINOLoss / DDINOLoss kernels: streaming (HBM-bound) passes over the [rows, K] bf16 logits.
//
// Reference: main_esvit.py
//   DINOLoss.forward  :620-648     DDINOLoss.forward :683-750     update_center :650-660, :752-770
//
// Formulation (DESIGN.md §loss).  With s~ = s / tau_s, t~ = (t - center) / temp and q = softmax(t~):
//   sum_k -q_k log_softmax(s~)_k = LSE(s~) - <q, s~>          (sum_k q_k = 1)
// so one student row r paired with its n_r <= 2 teacher rows costs ONE streaming pass:
//   row_loss[r] = n_r * LSE(s~_r) - sum_j <q_{t_j(r)}, s~_r>,   loss = sum_r w_r row_loss[r]
//   d loss / d s_{r,k} = w_r / tau_s * ( n_r softmax(s~_r)_k - sum_j q_{t_j(r),k} )
// The teacher rows of a region row are the cosine arg-max matches (region_match below); for a cls row
// they are the same image's other global view(s).  Nothing of size [B, T, K] is ever materialised.
#include <cuda_fp16.h>
#include "common.cuh"

namespace {

constexpr int LT = 256;  // threads per row CTA

__device__ __forceinline__ void block_reduce_ms(float& m, float& s) {
  // online-softmax (max, sum) pair reduction over the CTA
  __shared__ float sm[LT / 32], ss[LT / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    float nm = fmaxf(m, om);
    s = (m == -INFINITY ? 0.f : s * __expf(m - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
    m = nm;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { sm[w] = m; ss[w] = s; }
  __syncthreads();
  if (w == 0) {
    m = l < LT / 32 ? sm[l] : -INFINITY;
    s = l < LT / 32 ? ss[l] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      float nm = fmaxf(m, om);
      s = (m == -INFINITY ? 0.f : s * __expf(m - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
      m = nm;
    }
  }
}

__device__ __forceinline__ float block_sum(float v) {
  __shared__ float sb[LT / 32];
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sb[w] = v;
  __syncthreads();
  v = (threadIdx.x < LT / 32) ? sb[threadIdx.x] : 0.f;
  if (w == 0) v = warp_sum(v);
  return v;  // valid in warp 0
}

// lse[r] = log sum_k exp( (x[r,k] - center[k]) * inv_temp )      (center may be null)
__global__ void __launch_bounds__(LT) row_lse_kernel(const bf16* __restrict__ x, const float* __restrict__ center,
                                                     float inv_temp, float* __restrict__ lse, int K) {
  const long long r = blockIdx.x;
  const bf16x8* xr = reinterpret_cast<const bf16x8*>(x + r * K);
  float m = -INFINITY, s = 0.f;
  for (int i = threadIdx.x; i < K / 8; i += LT) {
    float f[8];
    unpack8(xr[i], f);
    if (center) {
      float4 c0 = *reinterpret_cast<const float4*>(center + i * 8), c1 = *reinterpret_cast<const float4*>(center + i * 8 + 4);
      f[0] -= c0.x; f[1] -= c0.y; f[2] -= c0.z; f[3] -= c0.w;
      f[4] -= c1.x; f[5] -= c1.y; f[6] -= c1.z; f[7] -= c1.w;
    }
    float lm = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; j++) { f[j] *= inv_temp; lm = fmaxf(lm, f[j]); }
    if (lm > m) { s *= __expf(m - lm); m = lm; }
#pragma unroll
    for (int j = 0; j < 8; j++) s += __expf(f[j] - m);
  }
  block_reduce_ms(m, s);
  if (threadIdx.x == 0) lse[r] = m + logf(s);
}

// row_loss[r] = n_r * lse_s[r] - sum_j sum_k exp(t~[tj,k] - lse_t[tj]) * s[r,k] * inv_tau_s
// The student log-sum-exp is accumulated (online max/sum) in the SAME pass over the row - the dot term does not depend
// on it - and written to lse_s for the backward: the student logits are read once, not twice.
__global__ void __launch_bounds__(LT) dino_ce_fwd_kernel(
    const bf16* __restrict__ s, const bf16* __restrict__ t, const float* __restrict__ center,
    float* __restrict__ lse_s, const float* __restrict__ lse_t, const int* __restrict__ trow,
    float inv_temp_t, float inv_tau_s, float* __restrict__ row_loss, int K, const int* __restrict__ order) {
  // CTA -> row through `order` (image-major): the CTAs resident together then stream the SAME image's teacher rows, which
  // stay in L2 across the ~3.5 student rows paired with each (row-major = crop-major order re-read them from DRAM)
  const long long r = order ? order[blockIdx.x] : blockIdx.x;
  const int t0 = trow[2 * r], t1 = trow[2 * r + 1];
  const bf16x8* sr = reinterpret_cast<const bf16x8*>(s + r * K);
  const bf16x8* tr0 = t0 >= 0 ? reinterpret_cast<const bf16x8*>(t + (long long)t0 * K) : nullptr;
  const bf16x8* tr1 = t1 >= 0 ? reinterpret_cast<const bf16x8*>(t + (long long)t1 * K) : nullptr;
  const float l0 = t0 >= 0 ? lse_t[t0] : 0.f, l1 = t1 >= 0 ? lse_t[t1] : 0.f;
  float acc = 0.f, m = -INFINITY, sm = 0.f;
  for (int i = threadIdx.x; i < K / 8; i += LT) {
    float fs[8];
    unpack8(sr[i], fs);
    const float4 c0 = *reinterpret_cast<const float4*>(center + i * 8);
    const float4 c1 = *reinterpret_cast<const float4*>(center + i * 8 + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    float q[8];
#pragma unroll
    for (int j = 0; j < 8; j++) q[j] = 0.f;
    if (tr0) {
      float ft[8];
      unpack8(tr0[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) q[j] += __expf((ft[j] - c[j]) * inv_temp_t - l0);
    }
    if (tr1) {
      float ft[8];
      unpack8(tr1[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) q[j] += __expf((ft[j] - c[j]) * inv_temp_t - l1);
    }
    float lm = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      acc += q[j] * fs[j];
      fs[j] *= inv_tau_s;
      lm = fmaxf(lm, fs[j]);
    }
    if (lm > m) { sm *= __expf(m - lm); m = lm; }
#pragma unroll
    for (int j = 0; j < 8; j++) sm += __expf(fs[j] - m);
  }
  block_reduce_ms(m, sm);
  __shared__ float lse_sh;
  if (threadIdx.x == 0) lse_sh = m + logf(sm);
  acc = block_sum(acc);  // (contains the __syncthreads that publishes lse_sh)
  if (threadIdx.x == 0) {
    const float n = (float)((t0 >= 0) + (t1 >= 0));
    lse_s[r] = lse_sh;
    row_loss[r] = n * lse_sh - acc * inv_tau_s;
  }
}

// ds[r,k] = gscale * w_r * inv_tau_s * ( n_r * exp(s~ - lse_s) - sum_j q_j )
__global__ void __launch_bounds__(LT) dino_ce_bwd_kernel(
    const bf16* __restrict__ s, const bf16* __restrict__ t, const float* __restrict__ center,
    const float* __restrict__ lse_s, const float* __restrict__ lse_t, const int* __restrict__ trow,
    const float* __restrict__ w, const float* __restrict__ gscale, float inv_temp_t, float inv_tau_s,
    bf16* __restrict__ ds, int K, const int* __restrict__ order) {
  const long long r = order ? order[blockIdx.x] : blockIdx.x;
  const int t0 = trow[2 * r], t1 = trow[2 * r + 1];
  const bf16x8* sr = reinterpret_cast<const bf16x8*>(s + r * K);
  bf16x8* dr = reinterpret_cast<bf16x8*>(ds + r * K);
  const bf16x8* tr0 = t0 >= 0 ? reinterpret_cast<const bf16x8*>(t + (long long)t0 * K) : nullptr;
  const bf16x8* tr1 = t1 >= 0 ? reinterpret_cast<const bf16x8*>(t + (long long)t1 * K) : nullptr;
  const float l0 = t0 >= 0 ? lse_t[t0] : 0.f, l1 = t1 >= 0 ? lse_t[t1] : 0.f;
  const float n = (float)((t0 >= 0) + (t1 >= 0));
  const float coef = gscale[0] * w[r] * inv_tau_s, ls = lse_s[r];
  for (int i = threadIdx.x; i < K / 8; i += LT) {
    float fs[8], g[8];
    unpack8(sr[i], fs);
    const float4 c0 = *reinterpret_cast<const float4*>(center + i * 8);
    const float4 c1 = *reinterpret_cast<const float4*>(center + i * 8 + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
    for (int j = 0; j < 8; j++) g[j] = n * __expf(fs[j] * inv_tau_s - ls);
    if (tr0) {
      float ft[8];
      unpack8(tr0[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) g[j] -= __expf((ft[j] - c[j]) * inv_temp_t - l0);
    }
    if (tr1) {
      float ft[8];
      unpack8(tr1[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) g[j] -= __expf((ft[j] - c[j]) * inv_temp_t - l1);
    }
#pragma unroll
    for (int j = 0; j < 8; j++) g[j] *= coef;
    dr[i] = pack8(g);
  }
}

// out[0] = sum_r w[r] * v[r]   (single CTA, fixed order => deterministic)
__global__ void __launch_bounds__(LT) weighted_sum_kernel(const float* __restrict__ v, const float* __restrict__ w,
                                                          int R, float* __restrict__ out) {
  float a = 0.f;
  for (int i = threadIdx.x; i < R; i += LT) a += v[i] * w[i];
  a = block_sum(a);
  if (threadIdx.x == 0) out[0] = a;
}

// ---- center: column sums (two deterministic stages) + EMA ------------------------------------
constexpr int CS_ROWS = 8;  // row lanes per CTA
__global__ void __launch_bounds__(32 * CS_ROWS) colsum_partial_kernel(const bf16* __restrict__ t, long long R, int K,
                                                                      float* __restrict__ partial) {
  // grid (K/256, GY); thread (x: 8 columns, y: row lane)
  __shared__ float sh[CS_ROWS][256 + 8];
  const int col = (blockIdx.x * 32 + threadIdx.x) * 8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (long long r = (long long)blockIdx.y * CS_ROWS + threadIdx.y; r < R && col < K;
       r += (long long)gridDim.y * CS_ROWS) {
    float f[8];
    unpack8(*reinterpret_cast<const bf16x8*>(t + r * K + col), f);
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] += f[j];
  }
#pragma unroll
  for (int j = 0; j < 8; j++) sh[threadIdx.y][threadIdx.x * 8 + j] = acc[j];
  __syncthreads();
  const int tid = threadIdx.y * 32 + threadIdx.x;  // 256 threads -> 256 columns
  float a = 0.f;
#pragma unroll
  for (int y = 0; y < CS_ROWS; y++) a += sh[y][tid];
  if (blockIdx.x * 256 + tid < K) partial[(long long)blockIdx.y * K + blockIdx.x * 256 + tid] = a;
}
__global__ void colsum_final_kernel(const float* __restrict__ partial, int GY, int K, float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float a = 0.f;
  for (int y = 0; y < GY; y++) a += partial[(long long)y * K + k];
  out[k] = a;
}
// center = center * m + (colsum / rows_total) * (1 - m); products/sum rounded separately like the reference's
// three ATen ops (main_esvit.py:657-660)
__global__ void center_ema_kernel(const float* __restrict__ center, const float* __restrict__ colsum,
                                  float rows_total, float m, float one_minus_m, float* __restrict__ out, int K) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const float bc = __fdiv_rn(colsum[k], rows_total);
  out[k] = __fadd_rn(__fmul_rn(center[k], m), __fmul_rn(bc, one_minus_m));
}

// ---- region match -----------------------------------------------------------------------------
// y = x / max(||x||, eps), fp32 rows (F.normalize, main_esvit.py:735)
__global__ void __launch_bounds__(256) normalize_rows_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                             long long R, int P, float eps) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < R; r += nwarps) {
    float s = 0.f;
    for (int c = lane * 4; c < P; c += 128) {
      float4 a = *reinterpret_cast<const float4*>(x + r * P + c);
      s += (a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w);
    }
    const float d = fmaxf(sqrtf(warp_sum(s)), eps);
    for (int c = lane * 4; c < P; c += 128) {
      float4 a = *reinterpret_cast<const float4*>(x + r * P + c);
      a.x = __fdiv_rn(a.x, d); a.y = __fdiv_rn(a.y, d); a.z = __fdiv_rn(a.z, d); a.w = __fdiv_rn(a.w, d);
      *reinterpret_cast<float4*>(y + r * P + c) = a;
    }
  }
}

// CTA (b, iq): the teacher view's Tg normalised region features stream through shared memory in chunks of TC rows
// (one chunk whenever all Tg * P fit, which covers Swin-T/S/B; ViT at Tg = 196 and Swin-L's 49 x 1536 need several); each warp takes
// student tokens of every crop v != iq, computes the cosine similarities (fp32, warp-reduced dot) and keeps the FIRST
// maximal index (torch.max tie rule, main_esvit.py:736).  Across chunks the running maximum and its index are kept in
// shared memory per token; the dot order and the strict > are those of a single pass, so the indices do not depend on TC.
//   sn rows: crop v<2 at (v*B + b)*Tg + i ; crop v>=2 at 2*B*Tg + ((v-2)*B + b)*Tl + i
//   tn rows: (iq*B + b)*Tg + j
//   idx out: int64 [2, ncrops, B, Tg] (unused slots untouched); trow out: int32 [Rs, 2] (-1 where v == iq)
// RM_MAXV float4 of the student row per lane: 8 up to P = 1024 (Swin-T/S/B, ViT, CvT, ViL), 12 up to P = 1536 (Swin-L)
template <int RM_MAXV>
__global__ void __launch_bounds__(256) region_match_kernel(const float* __restrict__ sn, const float* __restrict__ tn,
                                                           int B, int ncrops, int Tg, int Tl, int P, int TC,
                                                           long long* __restrict__ idx_out, int* __restrict__ trow) {
  extern __shared__ float tsm[];  // [TC][P], then (TC < Tg) the running maximum [per_img] and its index [per_img]
  const int b = blockIdx.x, iq = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float* tb = tn + ((long long)iq * B + b) * Tg * P;
  const int per_img = 2 * Tg + (ncrops - 2) * Tl;  // student tokens of image b over all crops
  float* run_best = tsm + (long long)TC * P;
  int* run_idx = reinterpret_cast<int*>(run_best + per_img);
  for (int j0 = 0; j0 < Tg; j0 += TC) {
    const int jn = min(TC, Tg - j0);
    const bool last = j0 + jn >= Tg;
    if (j0 > 0) __syncthreads();  // every warp is done with the previous chunk
    for (int i = threadIdx.x * 4; i < jn * P; i += blockDim.x * 4)
      *reinterpret_cast<float4*>(tsm + i) = *reinterpret_cast<const float4*>(tb + (long long)j0 * P + i);
    __syncthreads();
    for (int tok = warp; tok < per_img; tok += nw) {
      int v, i;
      long long srow;
      if (tok < 2 * Tg) {
        v = tok / Tg; i = tok - v * Tg;
        srow = ((long long)v * B + b) * Tg + i;
      } else {
        const int u = tok - 2 * Tg;
        v = 2 + u / Tl; i = u - (v - 2) * Tl;
        srow = 2LL * B * Tg + ((long long)(v - 2) * B + b) * Tl + i;
      }
      if (v == iq) {
        if (lane == 0 && last) trow[2 * srow + iq] = -1;
        continue;
      }
      float4 sv[RM_MAXV];
#pragma unroll
      for (int k = 0; k < RM_MAXV; k++) {
        const int c = (k * 32 + lane) * 4;
        sv[k] = c < P ? *reinterpret_cast<const float4*>(sn + srow * P + c) : make_float4(0, 0, 0, 0);
      }
      float best = -INFINITY;
      int besti = 0;
      if (j0 > 0) {
        best = run_best[tok];
        besti = run_idx[tok];
      }
      for (int j = 0; j < jn; j++) {
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < RM_MAXV; k++) {
          const int c = (k * 32 + lane) * 4;
          if (c < P) {
            float4 tv = *reinterpret_cast<const float4*>(tsm + j * P + c);
            d += (sv[k].x * tv.x + sv[k].y * tv.y) + (sv[k].z * tv.z + sv[k].w * tv.w);
          }
        }
        d = warp_sum(d);
        if (d > best) { best = d; besti = j0 + j; }
      }
      if (lane == 0) {
        if (last) {
          idx_out[(((long long)iq * ncrops + v) * B + b) * Tg + i] = besti;
          trow[2 * srow + iq] = (iq * B + b) * Tg + besti;
        } else {
          run_best[tok] = best;
          run_idx[tok] = besti;
        }
      }
    }
  }
}


// ---- teacher probabilities stored once (fp16, scaled by 2^12) -----------------------------------------------------------
// Every teacher row is paired with ~3.5 student rows (cls: 4 - 8 crops of the image, regions: the arg-max matches), and
// both CE kernels were bound by the SFU / FMA pipes, not by HBM: 3 exponentials per student logit, two of them teacher
// terms recomputed for every pairing.  row_softmax_q_kernel computes q = softmax((t - center) / temp) once per teacher row
// (LSE pass, then exp pass over the same row while it is still in L2: one DRAM read) and stores q * 2^12 in fp16: 11
// significant bits down to q = 1.5e-8 (below that, flushed: < 1e-3 of the probability mass even for a uniform row of
// 65536).  The CE kernels then stream q like the student logits.
__device__ __forceinline__ float fast_ex2(float x) {   // ex2.approx (one SFU instruction), as __expf uses
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;\n" : "=f"(y) : "f"(x));
  return y;
}
constexpr int QT = 1024;            // threads of the row-softmax CTA (2 CTAs per SM)
constexpr float Q_SCALE_LOG2 = 12.f, Q_UNSCALE = 1.f / 4096.f;
struct __align__(16) half8 { __half2 v[4]; };
__device__ __forceinline__ void unpack_h8(const half8& h, float* f) {
#pragma unroll
  for (int k = 0; k < 4; k++) { const float2 t = __half22float2(h.v[k]); f[2 * k] = t.x; f[2 * k + 1] = t.y; }
}

// Two passes over the row: LSE, then q.  The second pass re-reads the 2 K bytes this CTA has just streamed: an L2 hit while
// the rows in flight on the whole GPU fit the 50 MB L2 - at K = 65536, 132 SMs x 2 CTAs x 128 KB = 33 MB (four 512-thread
// CTAs per SM would hold 66 MB in flight).  Two 1024-thread CTAs keep the SM's full thread count issuing loads.  A first version kept the row in shared memory: one
// CTA per SM, its load, reduce and store phases never overlapped, 3x the HBM time.
__global__ void __launch_bounds__(QT, 2) row_softmax_q_kernel(const bf16* __restrict__ x, const float* __restrict__ center,
                                                              float inv_temp, float* __restrict__ lse, half8* __restrict__ q, int K) {
  __shared__ float red_m[QT / 32], red_s[QT / 32];
  __shared__ float lse2_sh;
  const long long r = blockIdx.x;
  const bf16x8* xr = reinterpret_cast<const bf16x8*>(x + r * K);
  const float a = inv_temp * 1.4426950408889634f;          // exp(v * inv_temp) = exp2(v * a)
  float m = -INFINITY, s = 0.f;                            // online (max, sum) in the exp2 domain
#pragma unroll 4
  for (int i = threadIdx.x; i < K / 8; i += QT) {   // (unrolled: four independent row loads in flight per thread)
    float f[8];
    unpack8(xr[i], f);
    const float4 c0 = *reinterpret_cast<const float4*>(center + i * 8), c1 = *reinterpret_cast<const float4*>(center + i * 8 + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    float lm = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; j++) { f[j] = (f[j] - c[j]) * a; lm = fmaxf(lm, f[j]); }
    if (lm > m) { s *= fast_ex2(m - lm); m = lm; }
#pragma unroll
    for (int j = 0; j < 8; j++) s += fast_ex2(f[j] - m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    const float nm = fmaxf(m, om);
    s = (m == -INFINITY ? 0.f : s * fast_ex2(m - nm)) + (om == -INFINITY ? 0.f : os * fast_ex2(om - nm));
    m = nm;
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red_m[w] = m; red_s[w] = s; }
  __syncthreads();
  if (w == 0) {
    m = l < QT / 32 ? red_m[l] : -INFINITY;
    s = l < QT / 32 ? red_s[l] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      const float nm = fmaxf(m, om);
      s = (m == -INFINITY ? 0.f : s * fast_ex2(m - nm)) + (om == -INFINITY ? 0.f : os * fast_ex2(om - nm));
      m = nm;
    }
    if (l == 0) {
      const float lse2 = m + log2f(s);
      lse2_sh = lse2;
      lse[r] = lse2 * 0.6931471805599453f;                 // natural-log LSE (what esvit_row_lse returns)
    }
  }
  __syncthreads();
  const float off = Q_SCALE_LOG2 - lse2_sh;
  half8* qr = q + r * (K / 8);
#pragma unroll 4
  for (int i = threadIdx.x; i < K / 8; i += QT) {   // (unrolled: four independent row loads in flight per thread)
    float f[8];
    unpack8(xr[i], f);
    const float4 c0 = *reinterpret_cast<const float4*>(center + i * 8), c1 = *reinterpret_cast<const float4*>(center + i * 8 + 4);
    const float c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    half8 h;
#pragma unroll
    for (int k = 0; k < 4; k++)
      h.v[k] = __floats2half2_rn(fast_ex2(fmaf(f[2 * k] - c[2 * k], a, off)), fast_ex2(fmaf(f[2 * k + 1] - c[2 * k + 1], a, off)));
    qr[i] = h;
  }
}

// the CE kernels on stored teacher probabilities (q12 = q * 2^12, fp16 [Rt, K]): same contract as dino_ce_fwd / bwd
__global__ void __launch_bounds__(LT) dino_ce_q_fwd_kernel(
    const bf16* __restrict__ s, const half8* __restrict__ q12, float* __restrict__ lse_s, const int* __restrict__ trow,
    float inv_tau_s, float* __restrict__ row_loss, int K, const int* __restrict__ order) {
  const long long r = order ? order[blockIdx.x] : blockIdx.x;
  const int t0 = trow[2 * r], t1 = trow[2 * r + 1];
  const bf16x8* sr = reinterpret_cast<const bf16x8*>(s + r * K);
  const half8* q0 = t0 >= 0 ? q12 + (long long)t0 * (K / 8) : nullptr;
  const half8* q1 = t1 >= 0 ? q12 + (long long)t1 * (K / 8) : nullptr;
  const float a = inv_tau_s * 1.4426950408889634f;
  float acc = 0.f, m = -INFINITY, sm = 0.f;                // (m, sm): student online softmax in the exp2 domain
  for (int i = threadIdx.x; i < K / 8; i += LT) {
    float fs[8], qq[8];
    unpack8(sr[i], fs);
#pragma unroll
    for (int j = 0; j < 8; j++) qq[j] = 0.f;
    if (q0) {
      float ft[8];
      unpack_h8(q0[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) qq[j] += ft[j];
    }
    if (q1) {
      float ft[8];
      unpack_h8(q1[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) qq[j] += ft[j];
    }
    float lm = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      acc = fmaf(qq[j], fs[j], acc);
      fs[j] *= a;
      lm = fmaxf(lm, fs[j]);
    }
    if (lm > m) { sm *= fast_ex2(m - lm); m = lm; }
#pragma unroll
    for (int j = 0; j < 8; j++) sm += fast_ex2(fs[j] - m);
  }
  // (max, sum) pairs are combined in the natural-log domain by block_reduce_ms
  m *= 0.6931471805599453f;
  block_reduce_ms(m, sm);
  __shared__ float lse_sh;
  if (threadIdx.x == 0) lse_sh = m + logf(sm);
  acc = block_sum(acc);  // (contains the __syncthreads that publishes lse_sh)
  if (threadIdx.x == 0) {
    const float n = (float)((t0 >= 0) + (t1 >= 0));
    lse_s[r] = lse_sh;
    row_loss[r] = n * lse_sh - acc * (inv_tau_s * Q_UNSCALE);
  }
}

__global__ void __launch_bounds__(LT) dino_ce_q_bwd_kernel(
    const bf16* __restrict__ s, const half8* __restrict__ q12, const float* __restrict__ lse_s, const int* __restrict__ trow,
    const float* __restrict__ w, const float* __restrict__ gscale, float inv_tau_s, bf16* __restrict__ ds, int K,
    const int* __restrict__ order) {
  const long long r = order ? order[blockIdx.x] : blockIdx.x;
  const int t0 = trow[2 * r], t1 = trow[2 * r + 1];
  const bf16x8* sr = reinterpret_cast<const bf16x8*>(s + r * K);
  bf16x8* dr = reinterpret_cast<bf16x8*>(ds + r * K);
  const half8* q0 = t0 >= 0 ? q12 + (long long)t0 * (K / 8) : nullptr;
  const half8* q1 = t1 >= 0 ? q12 + (long long)t1 * (K / 8) : nullptr;
  const float n = (float)((t0 >= 0) + (t1 >= 0));
  const float coef = gscale[0] * w[r] * inv_tau_s;
  const float a = inv_tau_s * 1.4426950408889634f, ls2 = lse_s[r] * 1.4426950408889634f;
  const float cn = coef * n, cq = -coef * Q_UNSCALE;
  for (int i = threadIdx.x; i < K / 8; i += LT) {
    float fs[8], qq[8], g[8];
    unpack8(sr[i], fs);
#pragma unroll
    for (int j = 0; j < 8; j++) qq[j] = 0.f;
    if (q0) {
      float ft[8];
      unpack_h8(q0[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) qq[j] += ft[j];
    }
    if (q1) {
      float ft[8];
      unpack_h8(q1[i], ft);
#pragma unroll
      for (int j = 0; j < 8; j++) qq[j] += ft[j];
    }
#pragma unroll
    for (int j = 0; j < 8; j++) g[j] = fmaf(cn, fast_ex2(fmaf(fs[j], a, -ls2)), cq * qq[j]);
    dr[i] = pack8(g);
  }
}

// ---- mixup targets (main_esvit.py:638-641): one mixed teacher row per student row -----------------------------------
// Student row r = (v, b) of the mixup loss pairs with q~_r = sum_{iq != v} sum_j T_v[j, b] q^{iq}_j, of mass
// C_r = sum_{iq != v} sum_j T_v[j, b].  For non-negative T, q^_r = q~_r / C_r is a probability row, stored in the q12 format
// above, and the loss is the CE of q^ at n_r = 1 and weight w_r = C_r / (n_terms * B) (DESIGN.md §4.8).
//   mixup_weights_kernel: one warp per student row: C_r, w_r and the row of Wn[r, i] = W[(iq, j), r] / C_r (i = iq*B + j,
//     zero-padded to Kp), scaled by 2^14 and split into fp16 hi + lo parts, so the tensor-core product carries ~22 bits of
//     every weight.  (Unscaled, weights below 2^-14 are fp16 subnormals: a weight of 1e-5 met by a teacher probability
//     near 1 lost 3e-3 of the product.)
//   mixup_q_kernel: q^[R, K] = Wn[R, Kp] . q12[Kp, K] * 2^-14 with mma.sync m16n8k16 (fp16 in, fp32 accumulate), hi and lo.
constexpr float MX_WSCALE = 16384.f;  // Wn <= 1 -> <= 2^14: hi normal down to Wn = 2^-28, lo down to Wn = 2^-17
__global__ void __launch_bounds__(256) mixup_weights_kernel(const float* __restrict__ T, int ncrops, int B, int Kp,
                                                            float w_scale, __half* __restrict__ a_hi,
                                                            __half* __restrict__ a_lo, float* __restrict__ w) {
  const int lane = threadIdx.x & 31;
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= (long long)ncrops * B) return;
  const int v = (int)(r / B), b = (int)(r % B);
  const float* Tv = T + (long long)v * B * B;  // T_v[j, b] at Tv[j * B + b]
  float c = 0.f;
  for (int j = lane; j < B; j += 32) c += Tv[(long long)j * B + b];
  c = warp_sum(c);
  const float C = v < 2 ? c : 2.f * c;  // global views pair with the other global view only
  if (lane == 0) w[r] = C * w_scale;
  for (int i = lane; i < Kp; i += 32) {
    const int iq = i / B, j = i - iq * B;
    const float x = (i < 2 * B && iq != v && C > 0.f) ? __fdiv_rn(Tv[(long long)j * B + b], C) * MX_WSCALE : 0.f;
    const __half h = __float2half_rn(x);
    a_hi[r * Kp + i] = h;
    a_lo[r * Kp + i] = __float2half_rn(x - __half2float(h));
  }
}

constexpr int MX_BM = 128, MX_BN = 128, MX_KC = 32, MX_T = 256;
constexpr int MX_AS = MX_KC + 8, MX_QS = MX_BN + 8;  // padded smem rows (halves): conflict-free ldmatrix / epilogue
struct MixSmem {
  union {
    struct {
      __half a_hi[MX_BM][MX_AS], a_lo[MX_BM][MX_AS];
      __half q[MX_KC][MX_QS];
    } ld;
    __half out[MX_BM][MX_QS];
  };
};

__device__ __forceinline__ void ldsm_x4(uint32_t* r, const void* p, bool trans) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(p);
  if (trans)
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
  else
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}

__device__ __forceinline__ void mma_f16(float* d, const uint32_t* a, const uint32_t* b) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
               "{%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// CTA: 128 student rows x 128 columns; 8 warps as 2 (rows) x 4 (columns), 64 x 32 each.  The teacher block (2B x K fp16,
// 16.8 MB at B = 64) is re-read from L2 by each of the R / 128 row tiles; the R x K fp16 output is the HBM traffic.
__global__ void __launch_bounds__(MX_T) mixup_q_kernel(const __half* __restrict__ a_hi, const __half* __restrict__ a_lo,
                                                       const __half* __restrict__ q, __half* __restrict__ out, int R,
                                                       int Rt, int K, int Kp) {
  __shared__ __align__(16) MixSmem sm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
  const int n0 = blockIdx.x * MX_BN;
  const long long m0 = (long long)blockIdx.y * MX_BM;
  float acc[4][4][4];
#pragma unroll
  for (int mt = 0; mt < 4; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[mt][nt][e] = 0.f;

  for (int k0 = 0; k0 < Kp; k0 += MX_KC) {
#pragma unroll
    for (int u = 0; u < 2; u++) {  // weights: 128 rows x 32 halves, hi and lo
      const int idx = tid + u * MX_T, row = idx >> 2, c8 = (idx & 3) * 8;
      const long long gr = m0 + row;
      uint4 vh = make_uint4(0, 0, 0, 0), vl = vh;
      if (gr < R) {
        vh = *reinterpret_cast<const uint4*>(a_hi + gr * Kp + k0 + c8);
        vl = *reinterpret_cast<const uint4*>(a_lo + gr * Kp + k0 + c8);
      }
      *reinterpret_cast<uint4*>(&sm.ld.a_hi[row][c8]) = vh;
      *reinterpret_cast<uint4*>(&sm.ld.a_lo[row][c8]) = vl;
    }
#pragma unroll
    for (int u = 0; u < 2; u++) {  // teacher probabilities: 32 rows x 128 columns (zero past the last row / column)
      const int idx = tid + u * MX_T, row = idx >> 4, c8 = (idx & 15) * 8;
      const int gi = k0 + row, gk = n0 + c8;
      uint4 vq = make_uint4(0, 0, 0, 0);
      if (gi < Rt && gk < K) vq = *reinterpret_cast<const uint4*>(q + (long long)gi * K + gk);
      *reinterpret_cast<uint4*>(&sm.ld.q[row][c8]) = vq;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < MX_KC; kk += 16) {
      uint32_t bf[4][2];
#pragma unroll
      for (int p = 0; p < 2; p++) {
        uint32_t t[4];
        ldsm_x4(t, &sm.ld.q[kk + (lane & 15)][wn * 32 + p * 16 + (lane >> 4) * 8], true);
        bf[2 * p][0] = t[0]; bf[2 * p][1] = t[1]; bf[2 * p + 1][0] = t[2]; bf[2 * p + 1][1] = t[3];
      }
#pragma unroll
      for (int mt = 0; mt < 4; mt++) {
        uint32_t ah[4], al[4];
        const int row = wm * 64 + mt * 16 + (lane & 15), col = kk + (lane >> 4) * 8;
        ldsm_x4(ah, &sm.ld.a_hi[row][col], false);
        ldsm_x4(al, &sm.ld.a_lo[row][col], false);
#pragma unroll
        for (int nt = 0; nt < 4; nt++) {
          mma_f16(acc[mt][nt], al, bf[nt]);
          mma_f16(acc[mt][nt], ah, bf[nt]);
        }
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int mt = 0; mt < 4; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
      const int r = wm * 64 + mt * 16 + (lane >> 2), c = wn * 32 + nt * 8 + (lane & 3) * 2;
      const float u = 1.f / MX_WSCALE;
      *reinterpret_cast<__half2*>(&sm.out[r][c]) = __floats2half2_rn(acc[mt][nt][0] * u, acc[mt][nt][1] * u);
      *reinterpret_cast<__half2*>(&sm.out[r + 8][c]) = __floats2half2_rn(acc[mt][nt][2] * u, acc[mt][nt][3] * u);
    }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < MX_BM * MX_BN / 8 / MX_T; u++) {  // whole 16-byte row segments
    const int idx = tid + u * MX_T, row = idx >> 4, c8 = (idx & 15) * 8;
    const long long gr = m0 + row;
    const int gk = n0 + c8;
    if (gr < R && gk < K) *reinterpret_cast<uint4*>(out + gr * K + gk) = *reinterpret_cast<const uint4*>(&sm.out[row][c8]);
  }
}

}  // namespace

ESVIT_API int esvit_row_lse(const void* x, const float* center, float inv_temp, float* lse, long long R, int K,
                            void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  row_lse_kernel<<<(unsigned)R, LT, 0, (cudaStream_t)stream>>>((const bf16*)x, center, inv_temp, lse, K);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dino_ce_fwd(const void* s, const void* t, const float* center, float* lse_s,
                                const float* lse_t, const int* trow, const int* order, float inv_temp_t, float inv_tau_s,
                                float* row_loss, long long R, int K, void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  dino_ce_fwd_kernel<<<(unsigned)R, LT, 0, (cudaStream_t)stream>>>((const bf16*)s, (const bf16*)t, center, lse_s, lse_t,
                                                                   trow, inv_temp_t, inv_tau_s, row_loss, K, order);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dino_ce_bwd(const void* s, const void* t, const float* center, const float* lse_s,
                                const float* lse_t, const int* trow, const int* order, const float* w, const float* gscale,
                                float inv_temp_t, float inv_tau_s, void* ds, long long R, int K, void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  dino_ce_bwd_kernel<<<(unsigned)R, LT, 0, (cudaStream_t)stream>>>((const bf16*)s, (const bf16*)t, center, lse_s, lse_t,
                                                                   trow, w, gscale, inv_temp_t, inv_tau_s, (bf16*)ds, K, order);
  ESVIT_LAUNCH_CHECK();
}

// ---- the same loss on stored teacher probabilities (see row_softmax_q_kernel) ----
ESVIT_API int esvit_row_softmax_q_max_k(void) { return 1 << 24; }  // (no structural limit: the row is streamed twice)

ESVIT_API int esvit_row_softmax_q(const void* x, const float* center, float inv_temp, float* lse, void* q, long long R,
                                  int K, void* stream) {
  if (K % 8 != 0 || R <= 0 || !center || K > esvit_row_softmax_q_max_k()) return ESVIT_ERR_BAD_ARG;
  row_softmax_q_kernel<<<(unsigned)R, QT, 0, (cudaStream_t)stream>>>((const bf16*)x, center, inv_temp, lse, (half8*)q, K);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dino_ce_q_fwd(const void* s, const void* q, float* lse_s, const int* trow, const int* order,
                                  float inv_tau_s, float* row_loss, long long R, int K, void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  dino_ce_q_fwd_kernel<<<(unsigned)R, LT, 0, (cudaStream_t)stream>>>((const bf16*)s, (const half8*)q, lse_s, trow, inv_tau_s,
                                                                     row_loss, K, order);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_dino_ce_q_bwd(const void* s, const void* q, const float* lse_s, const int* trow, const int* order,
                                  const float* w, const float* gscale, float inv_tau_s, void* ds, long long R, int K,
                                  void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  dino_ce_q_bwd_kernel<<<(unsigned)R, LT, 0, (cudaStream_t)stream>>>((const bf16*)s, (const half8*)q, lse_s, trow, w, gscale,
                                                                     inv_tau_s, (bf16*)ds, K, order);
  ESVIT_LAUNCH_CHECK();
}

// ---- mixup targets (see mixup_q_kernel) ----
ESVIT_API int esvit_mixup_q_kpad(int B) { return (2 * B + MX_KC - 1) / MX_KC * MX_KC; }

ESVIT_API int esvit_mixup_q(const float* targets, const void* q, int ncrops, int B, int K, float w_scale, void* ws,
                            float* w, void* q_out, void* stream) {
  if (K % 8 != 0 || K <= 0 || B <= 0 || ncrops < 2 || (long long)ncrops * B > (1LL << 30)) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int R = ncrops * B, Kp = esvit_mixup_q_kpad(B);
  __half* a_hi = (__half*)ws;
  __half* a_lo = a_hi + (long long)R * Kp;
  mixup_weights_kernel<<<(unsigned)((R + 7) / 8), 256, 0, st>>>(targets, ncrops, B, Kp, w_scale, a_hi, a_lo, w);
  mixup_q_kernel<<<dim3((K + MX_BN - 1) / MX_BN, (R + MX_BM - 1) / MX_BM), MX_T, 0, st>>>(
      a_hi, a_lo, (const __half*)q, (__half*)q_out, R, 2 * B, K, Kp);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_weighted_sum(const float* v, const float* w, int R, float* out, void* stream) {
  if (R <= 0) return ESVIT_ERR_BAD_ARG;
  weighted_sum_kernel<<<1, LT, 0, (cudaStream_t)stream>>>(v, w, R, out);
  ESVIT_LAUNCH_CHECK();
}

// workspace: float [esvit_colsum_workspace_rows() * K]
ESVIT_API int esvit_colsum_workspace_rows(void) { return 32; }

ESVIT_API int esvit_colsum(const void* t, long long R, int K, float* workspace, float* out, void* stream) {
  if (K % 8 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int GY = 32;
  colsum_partial_kernel<<<dim3((K + 255) / 256, GY), dim3(32, CS_ROWS), 0, st>>>((const bf16*)t, R, K, workspace);
  colsum_final_kernel<<<(K + 255) / 256, 256, 0, st>>>(workspace, GY, K, out);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_center_ema(const float* center, const float* colsum, float rows_total, double momentum,
                               float* center_out, int K, void* stream) {
  if (K <= 0) return ESVIT_ERR_BAD_ARG;
  // both factors rounded once from the double, as `center * m` and `bc * (1 - m)` round their Python scalars (1 - m
  // taken from an fp32 m instead is 3 ulps off at m = 0.9, and the center no longer matches the reference bit for bit)
  const float m = (float)momentum, om = (float)(1.0 - momentum);
  center_ema_kernel<<<(K + 255) / 256, 256, 0, (cudaStream_t)stream>>>(center, colsum, rows_total, m, om, center_out, K);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_normalize_rows(const float* x, float* y, long long R, int P, float eps, void* stream) {
  if (P % 4 != 0 || R <= 0) return ESVIT_ERR_BAD_ARG;
  long long need = (R + 7) / 8, cap = (long long)esvit_num_sms() * 16;
  normalize_rows_kernel<<<(int)(need < cap ? need : cap), 256, 0, (cudaStream_t)stream>>>(x, y, R, P, eps);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_region_match(const float* sn, const float* tn, int B, int ncrops, int Tg, int Tl, int P,
                                 long long* idx_out, int* trow, void* stream) {
  if (P % 4 != 0 || P > 1536 || B <= 0 || ncrops < 2) return ESVIT_ERR_BAD_ARG;
  const size_t budget = 220 * 1024, row = (size_t)P * sizeof(float);
  const size_t state = (size_t)(2 * Tg + (ncrops - 2) * Tl) * (sizeof(float) + sizeof(int));
  int TC = Tg;  // all teacher rows in one chunk when they fit, else as many as fit beside the running arg-max state
  size_t smem = (size_t)Tg * row;
  if (smem > budget) {
    if (state + row > budget) return ESVIT_ERR_BAD_ARG;
    TC = (int)((budget - state) / row);
    smem = (size_t)TC * row + state;
  }
  auto kernel = P <= 1024 ? region_match_kernel<8> : region_match_kernel<12>;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return (int)e;
  kernel<<<dim3(B, 2), 256, smem, (cudaStream_t)stream>>>(sn, tn, B, ncrops, Tg, Tl, P, TC, idx_out, trow);
  ESVIT_LAUNCH_CHECK();
}
