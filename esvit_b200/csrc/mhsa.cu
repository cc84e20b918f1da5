// Whole-sequence multi-head self-attention at head dim 64 (the ViT / DeiT backbones), forward and backward, and its
// window mode (CvT) at head dim 64 (spec s1) or 32 (spec s3).
//
// Reference: models/vision_transformer.py  Attention.forward :83-95
//   qkv = Linear(x).reshape(B, N, 3, nH, 64)  ->  softmax(q k^T * scale) v  ->  .transpose(1, 2).reshape(B, N, C)
//
// qkv bf16 [B*L, 3C] token-major as the qkv GEMM writes it (bias included), channel order [q|k|v][head][64].
// out bf16 [B*L, C] in the reference's (head, dim) channel order; lse fp32 [B, nH, L] (natural log) for the backward.
//
// One CTA = 4 warps = 64 query rows (16 per warp) of one (sequence, head); mma.sync m16n8k16 bf16 with fp32
// accumulation, fp32 online softmax in the log2 domain, P rounded to bf16 for PV, K / V tiles of 64 keys double-buffered
// through cp.async.  Rows / keys past L are zero-filled tiles: keys past L get a score of -inf (P = 0 exactly), queries
// past L are computed and never stored.
//
// Backward (no floating-point atomics, so dq / dk / dv are bit-reproducible):
//   prep   D[b,h,i] = sum_d dO * O
//   dq     CTA = 64 queries: P = ex2(s' - lse'), dP = dO V^T, dS = P (dP - D), dQ = scale * dS K   (loop over key tiles)
//   dkdv   CTA = 64 keys:    P^T, dV = P^T dO, dP^T = V dO^T, dS^T = P^T (dP^T - D), dK = scale * dS^T Q  (loop over queries)
// Each output row is owned by exactly one warp.
//
// Window mode (WIN = true; CvT, models/cvt_v4_transformer.py Attention.forward :165-220): "sequence" s is window s of
// the zero-padded Hp x Wp token map (images, then windows row-major, then tokens row-major), L = w*w tokens (any w; the
// 64-row query / key tiles loop as in the dense mode, window token r0 + r in row r of the tile that starts at r0).  q / k
// / v rows are gathered from the token-major qkv [B*Hp*Wp, 3C] of the padded map; out / dout are the CROPPED map
// [B*H*W, C]: padded query rows are not stored (their dO reads as 0, so their dq is 0), padded keys take part as in the
// reference.  lse / dvec are [windows, nH, L] as in the dense mode.  The head dim HD is a template parameter: 64, or 32
// in window mode only, where a tile is 64 rows x 32 (80-B smem rows), QK^T takes 2 k-steps and PV / dQ / dK / dV 4
// n-tiles of 8; one CTA still serves one (window, head) and 64 query (or key) rows.
#include <climits>

#include "wa_common.cuh"

namespace mh {

using wa::cp_async16;
using wa::cp_async_commit;
using wa::cp_async_wait;
using wa::ex2;
using wa::ldsm_x4;
using wa::ldsm_x4_t;
using wa::lg2;
using wa::LN2;
using wa::LOG2E;
using wa::mma16816;

// Head dim HD = 64 (ViT, CvT s1) or 32 (CvT s3, window mode only).  A tile is 64 rows x HD bf16 in shared memory with
// a row stride of HD + 8 elements (144 B rows at 64, 80 B at 32): the eight row addresses of an ldmatrix phase land in
// distinct banks.
template <int HD>
constexpr int LDS = HD + 8;
template <int HD>
constexpr int TILE = 64 * LDS<HD>;  // one 64-row tile
constexpr int NTHR = 128;

// async copy of a [64 rows x 64 bf16] tile whose row 0 starts at src (row stride ld elements); rows >= nvalid are zero
// (dense mode, head dim 64)
__device__ __forceinline__ void load_tile(bf16* dst, const bf16* __restrict__ src, long long ld, int nvalid) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int e = threadIdx.x + k * NTHR;  // 512 chunks of 16 B
    const int r = e >> 3, c = (e & 7) * 8;
    const bool ok = r < nvalid;
    cp_async16(dst + r * LDS<64> + c, src + (ok ? (long long)r * ld : 0) + c, ok ? 16 : 0);
  }
}

// A fragments (16 rows x HD) of rows r0.. of a tile
template <int HD>
__device__ __forceinline__ void load_a(uint32_t (&a)[HD / 16][4], const bf16* t, int r0, int lane) {
  const bf16* p = t + (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS<HD> + (lane >> 4) * 8;
#pragma unroll
  for (int k = 0; k < HD / 16; k++) ldsm_x4(a[k], p + k * 16);
}

// acc[nt] (16 x 8 per nt, 64 columns) = A (16 x HD) . T^T where T's rows are the 64 columns (k = the HD dims)
template <int HD>
__device__ __forceinline__ void mma_abt(float (&acc)[8][4], const uint32_t (&a)[HD / 16][4], const bf16* t, int lane) {
#pragma unroll
  for (int nt = 0; nt < 8; nt++) {
    acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    const bf16* p = t + (nt * 8 + (lane & 7)) * LDS<HD> + (lane >> 3) * 8;
    // one ldmatrix.x4 = two k-steps of 16; HD 64's second pair stays written out (a loop over the pairs changed the
    // register allocation of the HD 64 kernels)
    uint32_t b[4];
    ldsm_x4(b, p);
    mma16816(acc[nt], a[0], b[0], b[1]);
    mma16816(acc[nt], a[1], b[2], b[3]);
    if constexpr (HD == 64) {
      ldsm_x4(b, p + 32);
      mma16816(acc[nt], a[2], b[0], b[1]);
      mma16816(acc[nt], a[3], b[2], b[3]);
    }
  }
}

// o[dt] (16 x HD) += P (16 x 64, fp32 fragments rounded to bf16) . T where T is [64 rows (k) x HD dims]
template <int HD>
__device__ __forceinline__ void mma_pt(float (&o)[HD / 8][4], const float (&p)[8][4], const bf16* t, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
    uint32_t pa[4];
    pa[0] = pack_bf162(p[2 * kk][0], p[2 * kk][1]);
    pa[1] = pack_bf162(p[2 * kk][2], p[2 * kk][3]);
    pa[2] = pack_bf162(p[2 * kk + 1][0], p[2 * kk + 1][1]);
    pa[3] = pack_bf162(p[2 * kk + 1][2], p[2 * kk + 1][3]);
    const bf16* vp = t + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LDS<HD> + (lane >> 4) * 8;
#pragma unroll
    for (int d16 = 0; d16 < HD / 16; d16++) {
      uint32_t vb[4];
      ldsm_x4_t(vb, vp + d16 * 16);
      mma16816(o[2 * d16], pa, vb[0], vb[1]);
      mma16816(o[2 * d16 + 1], pa, vb[2], vb[3]);
    }
  }
}

// 16 x 64 fp32 fragments -> bf16 rows (rA, rB) of dst (row stride ld), rows >= L skipped (dense mode, head dim 64)
__device__ __forceinline__ void store_rows(bf16* __restrict__ dst, long long ld, const float (&o)[8][4], float s0,
                                           float s1, int rA, int rB, int L, int lane) {
#pragma unroll
  for (int dt = 0; dt < 8; dt++) {
    const int d = dt * 8 + (lane & 3) * 2;
    if (rA < L) *reinterpret_cast<uint32_t*>(dst + (long long)rA * ld + d) = pack_bf162(o[dt][0] * s0, o[dt][1] * s0);
    if (rB < L) *reinterpret_cast<uint32_t*>(dst + (long long)rB * ld + d) = pack_bf162(o[dt][2] * s1, o[dt][3] * s1);
  }
}

// window geometry of the WIN kernels (unused by the dense ones)
struct Win {
  int H, W, Hp, Wp, w, nwx, nwin;  // nwx windows per row, nwin per image
};

// padded-map row of token l of window s
__device__ __forceinline__ long long win_row(const Win& g, int s, int l) {
  const int img = s / g.nwin, wi = s - img * g.nwin, wy = wi / g.nwx, wx = wi - wy * g.nwx;
  const int ty = l / g.w, tx = l - ty * g.w;
  return ((long long)img * g.Hp + wy * g.w + ty) * g.Wp + wx * g.w + tx;
}
// cropped-map row of token l of window s, -1 for a padded position
__device__ __forceinline__ long long win_out_row(const Win& g, int s, int l) {
  const int img = s / g.nwin, wi = s - img * g.nwin, wy = wi / g.nwx, wx = wi - wy * g.nwx;
  const int ty = l / g.w, tx = l - ty * g.w, y = wy * g.w + ty, x = wx * g.w + tx;
  return (y < g.H && x < g.W) ? ((long long)img * g.H + y) * g.W + x : -1;
}

// async copy of the [64 rows x HD bf16] tile of tokens r0.. of window s: src = the map's column base, tile row r at the
// (out ? cropped : padded) row of token r0 + r; tokens >= L and padded rows of the cropped map are zero
template <bool OUT, int HD>
__device__ __forceinline__ void load_tile_win(bf16* dst, const bf16* __restrict__ src, long long ld, const Win& g, int s,
                                              int L, int r0) {
  constexpr int SH = HD == 64 ? 3 : 2, CH = 1 << SH;  // 16-B chunks per row
  static_assert(CH * 8 == HD, "head dim 32 or 64");
#pragma unroll
  for (int k = 0; k < 64 * CH / NTHR; k++) {
    const int e = threadIdx.x + k * NTHR;
    const int r = e >> SH, c = (e & (CH - 1)) * 8;
    long long row = -1;
    if (r0 + r < L) row = OUT ? win_out_row(g, s, r0 + r) : win_row(g, s, r0 + r);
    const bool ok = row >= 0;
    cp_async16(dst + r * LDS<HD> + c, src + (ok ? row * ld : 0) + c, ok ? 16 : 0);
  }
}

// 16 x HD fp32 fragments of window s -> bf16: rows rA / rB < L go to (out ? cropped : padded) rows; padded rows of the
// cropped map skipped
template <bool OUT, int HD>
__device__ __forceinline__ void store_rows_win(bf16* __restrict__ dst, long long ld, const float (&o)[HD / 8][4], float s0,
                                               float s1, int rA, int rB, int L, const Win& g, int s, int lane) {
  long long oA = -1, oB = -1;
  if (rA < L) oA = OUT ? win_out_row(g, s, rA) : win_row(g, s, rA);
  if (rB < L) oB = OUT ? win_out_row(g, s, rB) : win_row(g, s, rB);
#pragma unroll
  for (int dt = 0; dt < HD / 8; dt++) {
    const int d = dt * 8 + (lane & 3) * 2;
    if (oA >= 0) *reinterpret_cast<uint32_t*>(dst + oA * ld + d) = pack_bf162(o[dt][0] * s0, o[dt][1] * s0);
    if (oB >= 0) *reinterpret_cast<uint32_t*>(dst + oB * ld + d) = pack_bf162(o[dt][2] * s1, o[dt][3] * s1);
  }
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// ---------------------------------------------------------------------------------------------------------------
template <bool WIN, int HD>
__global__ void __launch_bounds__(NTHR) mhsa_fwd_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ out,
                                                        float* __restrict__ lse, int L, int C, int nH, float c2,
                                                        const Win win) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);  // [Q | K0 | V0 | K1 | V1]
  const int q0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long C3 = 3LL * C;
  const bf16* base = qkv + (long long)b * L * C3 + h * HD;
  if constexpr (WIN) {
    load_tile_win<false, HD>(Qs, qkv + h * HD, C3, win, b, L, q0);
    load_tile_win<false, HD>(Qs + TILE<HD>, qkv + h * HD + C, C3, win, b, L, 0);
    load_tile_win<false, HD>(Qs + 2 * TILE<HD>, qkv + h * HD + 2 * C, C3, win, b, L, 0);
  } else {
    load_tile(Qs, base + q0 * C3, C3, L - q0);
    load_tile(Qs + TILE<HD>, base + C, C3, L);
    load_tile(Qs + 2 * TILE<HD>, base + 2 * C, C3, L);
  }
  cp_async_commit();
  const int nkt = (L + 63) / 64;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[HD / 8][4];
#pragma unroll
  for (int dt = 0; dt < HD / 8; dt++) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
  uint32_t qa[HD / 16][4];
  for (int kt = 0; kt < nkt; kt++) {
    const int st = kt & 1;
    if (kt + 1 < nkt) {
      bf16* nx = Qs + (1 + 2 * (st ^ 1)) * TILE<HD>;
      if constexpr (WIN) {
        load_tile_win<false, HD>(nx, qkv + h * HD + C, C3, win, b, L, (kt + 1) * 64);
        load_tile_win<false, HD>(nx + TILE<HD>, qkv + h * HD + 2 * C, C3, win, b, L, (kt + 1) * 64);
      } else {
        load_tile(nx, base + C + (kt + 1) * 64 * C3, C3, L - (kt + 1) * 64);
        load_tile(nx + TILE<HD>, base + 2 * C + (kt + 1) * 64 * C3, C3, L - (kt + 1) * 64);
      }
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Ks = Qs + (1 + 2 * st) * TILE<HD>;
    if (kt == 0) load_a<HD>(qa, Qs, warp * 16, lane);
    float s[8][4];
    mma_abt<HD>(s, qa, Ks, lane);
    const bool edge = kt * 64 + 64 > L;
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
#pragma unroll
      for (int i = 0; i < 4; i++) s[nt][i] *= c2;
      if (edge) {
        const int key = kt * 64 + nt * 8 + (lane & 3) * 2;
        if (key >= L) s[nt][0] = s[nt][2] = -INFINITY;
        if (key + 1 >= L) s[nt][1] = s[nt][3] = -INFINITY;
      }
    }
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = quad_max(mx0);
    mx1 = quad_max(mx1);  // finite: every key tile holds at least one key < L
    const float a0 = ex2(m0 - mx0), a1 = ex2(m1 - mx1);
    m0 = mx0;
    m1 = mx1;
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      s[nt][0] = ex2(s[nt][0] - m0);
      s[nt][1] = ex2(s[nt][1] - m0);
      s[nt][2] = ex2(s[nt][2] - m1);
      s[nt][3] = ex2(s[nt][3] - m1);
      r0 += s[nt][0] + s[nt][1];
      r1 += s[nt][2] + s[nt][3];
    }
    l0 = l0 * a0 + r0;
    l1 = l1 * a1 + r1;
#pragma unroll
    for (int dt = 0; dt < HD / 8; dt++) {
      o[dt][0] *= a0; o[dt][1] *= a0;
      o[dt][2] *= a1; o[dt][3] *= a1;
    }
    mma_pt<HD>(o, s, Ks + TILE<HD>, lane);
    __syncthreads();  // the next iteration's copy overwrites this stage
  }
  cp_async_wait<0>();
  l0 = quad_sum(l0);
  l1 = quad_sum(l1);
  const int rA = q0 + warp * 16 + (lane >> 2), rB = rA + 8;
  if constexpr (WIN)
    store_rows_win<true, HD>(out + h * HD, C, o, __fdividef(1.f, l0), __fdividef(1.f, l1), rA, rB, L, win, b, lane);
  else
    store_rows(out + (long long)b * L * C + h * HD, C, o, __fdividef(1.f, l0), __fdividef(1.f, l1), rA, rB, L, lane);
  if ((lane & 3) == 0) {
    float* lp = lse + ((long long)b * nH + h) * L;
    if (rA < L) lp[rA] = (m0 + lg2(l0)) * LN2;
    if (rB < L) lp[rB] = (m1 + lg2(l1)) * LN2;
  }
}

// D[b, h, i] = sum_d dO[b, i, h, d] * O[b, i, h, d]; one warp per token row, lanes over (head, dim pair): one head per
// pass at head dim 64, two at 32 (lanes 0-15 head h, 16-31 head h + 1, so a pass still reads 128 contiguous bytes)
// (WIN: B windows; a padded query row has D = 0)
template <bool WIN, int HD>
__global__ void __launch_bounds__(256) mhsa_bwd_prep_kernel(const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                                            float* __restrict__ dvec, int B, int L, int C, int nH,
                                                            const Win win) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= (long long)B * L) return;
  const int b = (int)(row / L), i = (int)(row - (long long)b * L);
  long long orow = row;
  if constexpr (WIN) orow = win_out_row(win, b, i);
  if constexpr (HD == 32) {
    for (int h0 = 0; h0 < nH; h0 += 2) {
      const int h = h0 + (lane >> 4);
      float d = 0.f;
      if (orow >= 0 && h < nH) {
        const long long off = orow * C + h0 * HD + lane * 2;
        const float2 o = __bfloat1622float2(*reinterpret_cast<const bf162*>(out + off));
        const float2 g = __bfloat1622float2(*reinterpret_cast<const bf162*>(dout + off));
        d = o.x * g.x + o.y * g.y;
      }
#pragma unroll
      for (int m = 8; m >= 1; m >>= 1) d += __shfl_xor_sync(0xffffffffu, d, m);
      if ((lane & 15) == 0 && h < nH) dvec[((long long)b * nH + h) * L + i] = d;
    }
  } else {
    for (int h = 0; h < nH; h++) {
      if constexpr (WIN)
        if (orow < 0) {
          if (lane == 0) dvec[((long long)b * nH + h) * L + i] = 0.f;
          continue;
        }
      const long long off = orow * C + h * HD + lane * 2;
      const float2 o = __bfloat1622float2(*reinterpret_cast<const bf162*>(out + off));
      const float2 g = __bfloat1622float2(*reinterpret_cast<const bf162*>(dout + off));
      const float d = warp_sum(o.x * g.x + o.y * g.y);
      if (lane == 0) dvec[((long long)b * nH + h) * L + i] = d;
    }
  }
}

// dQ of 64 query rows; lse / dvec as the forward / prep kernels wrote them
// (HD 32: at most 128 registers, four CTAs per SM; unbounded, ptxas took 183 registers and two CTAs)
template <bool WIN, int HD>
__global__ void __launch_bounds__(NTHR, HD == 32 ? 4 : 0) mhsa_bwd_dq_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout,
                                                           const float* __restrict__ lse, const float* __restrict__ dvec,
                                                           bf16* __restrict__ dqkv, int L, int C, int nH, float c2,
                                                           float scale, const Win win) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);  // [Q | dO | K0 | V0 | K1 | V1]
  const int q0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long C3 = 3LL * C;
  const bf16* base = qkv + (long long)b * L * C3 + h * HD;
  if constexpr (WIN) {
    load_tile_win<false, HD>(Qs, qkv + h * HD, C3, win, b, L, q0);
    load_tile_win<true, HD>(Qs + TILE<HD>, dout + h * HD, C, win, b, L, q0);
    load_tile_win<false, HD>(Qs + 2 * TILE<HD>, qkv + h * HD + C, C3, win, b, L, 0);
    load_tile_win<false, HD>(Qs + 3 * TILE<HD>, qkv + h * HD + 2 * C, C3, win, b, L, 0);
  } else {
    load_tile(Qs, base + q0 * C3, C3, L - q0);
    load_tile(Qs + TILE<HD>, dout + ((long long)b * L + q0) * C + h * HD, C, L - q0);
    load_tile(Qs + 2 * TILE<HD>, base + C, C3, L);
    load_tile(Qs + 3 * TILE<HD>, base + 2 * C, C3, L);
  }
  cp_async_commit();
  const int rA = q0 + warp * 16 + (lane >> 2), rB = rA + 8;
  const float* lp = lse + ((long long)b * nH + h) * L;
  const float* dp = dvec + ((long long)b * nH + h) * L;
  const float lA = rA < L ? lp[rA] * LOG2E : 0.f, lB = rB < L ? lp[rB] * LOG2E : 0.f;
  const float DA = rA < L ? dp[rA] : 0.f, DB = rB < L ? dp[rB] : 0.f;
  const int nkt = (L + 63) / 64;
  float dq[HD / 8][4];
#pragma unroll
  for (int dt = 0; dt < HD / 8; dt++) dq[dt][0] = dq[dt][1] = dq[dt][2] = dq[dt][3] = 0.f;
  uint32_t qa[HD / 16][4], oa[HD / 16][4];
  for (int kt = 0; kt < nkt; kt++) {
    const int st = kt & 1;
    if (kt + 1 < nkt) {
      bf16* nx = Qs + (2 + 2 * (st ^ 1)) * TILE<HD>;
      if constexpr (WIN) {
        load_tile_win<false, HD>(nx, qkv + h * HD + C, C3, win, b, L, (kt + 1) * 64);
        load_tile_win<false, HD>(nx + TILE<HD>, qkv + h * HD + 2 * C, C3, win, b, L, (kt + 1) * 64);
      } else {
        load_tile(nx, base + C + (kt + 1) * 64 * C3, C3, L - (kt + 1) * 64);
        load_tile(nx + TILE<HD>, base + 2 * C + (kt + 1) * 64 * C3, C3, L - (kt + 1) * 64);
      }
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Ks = Qs + (2 + 2 * st) * TILE<HD>;
    if (kt == 0) {
      load_a<HD>(qa, Qs, warp * 16, lane);
      load_a<HD>(oa, Qs + TILE<HD>, warp * 16, lane);
    }
    float p[8][4], g[8][4];
    mma_abt<HD>(p, qa, Ks, lane);
    mma_abt<HD>(g, oa, Ks + TILE<HD>, lane);
    const bool edge = kt * 64 + 64 > L;
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      p[nt][0] = ex2(p[nt][0] * c2 - lA);
      p[nt][1] = ex2(p[nt][1] * c2 - lA);
      p[nt][2] = ex2(p[nt][2] * c2 - lB);
      p[nt][3] = ex2(p[nt][3] * c2 - lB);
      if (edge) {
        const int key = kt * 64 + nt * 8 + (lane & 3) * 2;
        if (key >= L) p[nt][0] = p[nt][2] = 0.f;
        if (key + 1 >= L) p[nt][1] = p[nt][3] = 0.f;
      }
      p[nt][0] *= g[nt][0] - DA;
      p[nt][1] *= g[nt][1] - DA;
      p[nt][2] *= g[nt][2] - DB;
      p[nt][3] *= g[nt][3] - DB;
    }
    mma_pt<HD>(dq, p, Ks, lane);
    __syncthreads();
  }
  cp_async_wait<0>();
  if constexpr (WIN)
    store_rows_win<false, HD>(dqkv + h * HD, C3, dq, scale, scale, rA, rB, L, win, b, lane);
  else
    store_rows(dqkv + (long long)b * L * C3 + h * HD, C3, dq, scale, scale, rA, rB, L, lane);
}

// dK, dV of 64 key rows
// (WIN: at most 168 registers, so three CTAs fit an SM as they did when a window was a single tile; HD 32: at most 96
// registers, five CTAs per SM, as the HD-32 forward)
template <bool WIN, int HD>
__global__ void __launch_bounds__(NTHR, HD == 32 ? 5 : WIN ? 3 : 0)
    mhsa_bwd_dkdv_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ dout, const float* __restrict__ lse,
                         const float* __restrict__ dvec, bf16* __restrict__ dqkv, int L, int C, int nH, float c2,
                         float scale, const Win win) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Ks = reinterpret_cast<bf16*>(smraw);            // [K | V | Q0 | dO0 | Q1 | dO1]
  float* stat = reinterpret_cast<float*>(Ks + 6 * TILE<HD>);  // [2 stages][lse' 64 | D 64]
  const int k0 = blockIdx.x * 64, h = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long C3 = 3LL * C;
  const bf16* base = qkv + (long long)b * L * C3 + h * HD;
  const bf16* gbase = dout + (long long)b * L * C + h * HD;
  const float* lp = lse + ((long long)b * nH + h) * L;
  const float* dp = dvec + ((long long)b * nH + h) * L;
  if constexpr (WIN) {
    load_tile_win<false, HD>(Ks, qkv + h * HD + C, C3, win, b, L, k0);
    load_tile_win<false, HD>(Ks + TILE<HD>, qkv + h * HD + 2 * C, C3, win, b, L, k0);
    load_tile_win<false, HD>(Ks + 2 * TILE<HD>, qkv + h * HD, C3, win, b, L, 0);
    load_tile_win<true, HD>(Ks + 3 * TILE<HD>, dout + h * HD, C, win, b, L, 0);
  } else {
    load_tile(Ks, base + C + k0 * C3, C3, L - k0);
    load_tile(Ks + TILE<HD>, base + 2 * C + k0 * C3, C3, L - k0);
    load_tile(Ks + 2 * TILE<HD>, base, C3, L);
    load_tile(Ks + 3 * TILE<HD>, gbase, C, L);
  }
  cp_async_commit();
  if (threadIdx.x < 64) {  // queries past L: lse' = +inf -> P = 0
    const int q = threadIdx.x;
    stat[q] = q < L ? lp[q] * LOG2E : INFINITY;
    stat[64 + q] = q < L ? dp[q] : 0.f;
  }
  const int nqt = (L + 63) / 64;
  float dk[HD / 8][4], dv[HD / 8][4];
#pragma unroll
  for (int dt = 0; dt < HD / 8; dt++)
#pragma unroll
    for (int i = 0; i < 4; i++) dk[dt][i] = dv[dt][i] = 0.f;
  uint32_t ka[HD / 16][4], va[HD / 16][4];
  for (int qt = 0; qt < nqt; qt++) {
    const int st = qt & 1;
    if (qt + 1 < nqt) {
      bf16* nx = Ks + (2 + 2 * (st ^ 1)) * TILE<HD>;
      const int n0 = (qt + 1) * 64;
      if constexpr (WIN) {
        load_tile_win<false, HD>(nx, qkv + h * HD, C3, win, b, L, n0);
        load_tile_win<true, HD>(nx + TILE<HD>, dout + h * HD, C, win, b, L, n0);
      } else {
        load_tile(nx, base + n0 * C3, C3, L - n0);
        load_tile(nx + TILE<HD>, gbase + (long long)n0 * C, C, L - n0);
      }
      if (threadIdx.x < 64) {
        const int q = n0 + threadIdx.x;
        float* sn = stat + (st ^ 1) * 128;
        sn[threadIdx.x] = q < L ? lp[q] * LOG2E : INFINITY;
        sn[64 + threadIdx.x] = q < L ? dp[q] : 0.f;
      }
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Qs = Ks + (2 + 2 * st) * TILE<HD>;
    const float* sl = stat + st * 128;
    if (qt == 0) {
      load_a<HD>(ka, Ks, warp * 16, lane);
      load_a<HD>(va, Ks + TILE<HD>, warp * 16, lane);
    }
    float p[8][4], g[8][4];
    mma_abt<HD>(p, ka, Qs, lane);         // S^T: keys x queries
    mma_abt<HD>(g, va, Qs + TILE<HD>, lane);  // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      const int q = nt * 8 + (lane & 3) * 2;
      const float2 lq = *reinterpret_cast<const float2*>(sl + q);
      p[nt][0] = ex2(p[nt][0] * c2 - lq.x);
      p[nt][1] = ex2(p[nt][1] * c2 - lq.y);
      p[nt][2] = ex2(p[nt][2] * c2 - lq.x);
      p[nt][3] = ex2(p[nt][3] * c2 - lq.y);
    }
    mma_pt<HD>(dv, p, Qs + TILE<HD>, lane);   // dV += P^T dO
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      const int q = nt * 8 + (lane & 3) * 2;
      const float2 dq = *reinterpret_cast<const float2*>(sl + 64 + q);
      p[nt][0] *= g[nt][0] - dq.x;
      p[nt][1] *= g[nt][1] - dq.y;
      p[nt][2] *= g[nt][2] - dq.x;
      p[nt][3] *= g[nt][3] - dq.y;
    }
    mma_pt<HD>(dk, p, Qs, lane);          // dK += dS^T Q
    __syncthreads();
  }
  cp_async_wait<0>();
  const int rA = k0 + warp * 16 + (lane >> 2), rB = rA + 8;
  if constexpr (WIN) {
    store_rows_win<false, HD>(dqkv + h * HD + C, C3, dk, scale, scale, rA, rB, L, win, b, lane);
    store_rows_win<false, HD>(dqkv + h * HD + 2 * C, C3, dv, 1.f, 1.f, rA, rB, L, win, b, lane);
  } else {
    bf16* dst = dqkv + (long long)b * L * C3 + h * HD;
    store_rows(dst + C, C3, dk, scale, scale, rA, rB, L, lane);
    store_rows(dst + 2 * C, C3, dv, 1.f, 1.f, rA, rB, L, lane);
  }
}

template <int HD>
constexpr size_t FWD_SMEM = 5 * TILE<HD> * sizeof(bf16);
template <int HD>
constexpr size_t DQ_SMEM = 6 * TILE<HD> * sizeof(bf16);
template <int HD>
constexpr size_t DKDV_SMEM = 6 * TILE<HD> * sizeof(bf16) + 2 * 128 * sizeof(float);

static bool ok_args(const void* a, const void* b, int B, int L, int C, int nH, int hd) {
  return a && b && B >= 1 && B <= 65535 && L >= 1 && nH >= 1 && C == nH * hd && ((uintptr_t)a & 15) == 0 &&
         ((uintptr_t)b & 15) == 0;
}

// head dim of the window mode: 32 or 64, 0 for anything else
static int win_head_dim(int C, int nH) {
  if (nH < 1) return 0;
  return C == 64 * nH ? 64 : C == 32 * nH ? 32 : 0;
}

template <typename K>
static cudaError_t opt_in(K kernel, size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                          : cudaSuccess;
}

// window geometry of a B x H x W map in windows of w x w (rejects what the WIN kernels cannot address: the window
// count is a grid dimension, and the token rows of the padded map are counted in int by the prep grid)
static bool win_geo(int B, int H, int W, int w, Win* g, int* nwin_total) {
  if (B < 1 || H < 1 || W < 1 || w < 1 || w > H || w > W) return false;
  g->H = H; g->W = W; g->w = w;
  g->Hp = (H + w - 1) / w * w; g->Wp = (W + w - 1) / w * w;
  g->nwx = g->Wp / w; g->nwin = (g->Hp / w) * g->nwx;
  const long long n = (long long)B * g->nwin;
  if (n > 65535 || n * w * w > INT_MAX) return false;
  *nwin_total = (int)n;
  return true;
}

template <bool WIN, int HD>
static int fwd_launch(const void* qkv, void* out, float* lse, int B, int L, int C, int nH, float scale, const Win& win,
                      void* stream) {
  const dim3 grid((L + 63) / 64, nH, B);
  mhsa_fwd_kernel<WIN, HD><<<grid, NTHR, FWD_SMEM<HD>, (cudaStream_t)stream>>>((const bf16*)qkv, (bf16*)out, lse, L, C, nH,
                                                                       scale * LOG2E, win);
  ESVIT_LAUNCH_CHECK();
}

template <bool WIN, int HD>
static int bwd_launch(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv, int B,
                      int L, int C, int nH, float scale, const Win& win, void* stream) {
  cudaError_t e = opt_in(mhsa_bwd_dq_kernel<WIN, HD>, DQ_SMEM<HD>);
  if (e == cudaSuccess) e = opt_in(mhsa_bwd_dkdv_kernel<WIN, HD>, DKDV_SMEM<HD>);
  if (e != cudaSuccess) return (int)e;
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = (long long)B * L;
  mhsa_bwd_prep_kernel<WIN, HD><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>((const bf16*)out, (const bf16*)dout, dvec, B, L,
                                                                        C, nH, win);
  const dim3 grid((L + 63) / 64, nH, B);
  const float c2 = scale * LOG2E;
  mhsa_bwd_dq_kernel<WIN, HD><<<grid, NTHR, DQ_SMEM<HD>, st>>>((const bf16*)qkv, (const bf16*)dout, lse, dvec, (bf16*)dqkv, L, C,
                                                       nH, c2, scale, win);
  mhsa_bwd_dkdv_kernel<WIN, HD><<<grid, NTHR, DKDV_SMEM<HD>, st>>>((const bf16*)qkv, (const bf16*)dout, lse, dvec, (bf16*)dqkv, L,
                                                           C, nH, c2, scale, win);
  ESVIT_LAUNCH_CHECK();
}

}  // namespace mh

ESVIT_API int esvit_mhsa_fwd(const void* qkv, void* out, float* lse, int B, int L, int C, int nH, float scale,
                             void* stream) {
  if (!mh::ok_args(qkv, out, B, L, C, nH, 64) || !lse) return ESVIT_ERR_BAD_ARG;
  return mh::fwd_launch<false, 64>(qkv, out, lse, B, L, C, nH, scale, mh::Win{}, stream);
}

ESVIT_API int esvit_mhsa_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec,
                             void* dqkv, int B, int L, int C, int nH, float scale, void* stream) {
  if (!mh::ok_args(qkv, dqkv, B, L, C, nH, 64) || !mh::ok_args(out, dout, B, L, C, nH, 64) || !lse || !dvec)
    return ESVIT_ERR_BAD_ARG;
  return mh::bwd_launch<false, 64>(qkv, out, dout, lse, dvec, dqkv, B, L, C, nH, scale, mh::Win{}, stream);
}

ESVIT_API int esvit_mhsa_win_fwd(const void* qkv, void* out, float* lse, int B, int H, int W, int w, int C, int nH,
                                 float scale, void* stream) {
  mh::Win g;
  int nw;
  const int hd = mh::win_head_dim(C, nH);
  if (!hd || !mh::win_geo(B, H, W, w, &g, &nw) || !mh::ok_args(qkv, out, nw, w * w, C, nH, hd) || !lse)
    return ESVIT_ERR_BAD_ARG;
  return hd == 64 ? mh::fwd_launch<true, 64>(qkv, out, lse, nw, w * w, C, nH, scale, g, stream)
                  : mh::fwd_launch<true, 32>(qkv, out, lse, nw, w * w, C, nH, scale, g, stream);
}

ESVIT_API int esvit_mhsa_win_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec,
                                 void* dqkv, int B, int H, int W, int w, int C, int nH, float scale, void* stream) {
  mh::Win g;
  int nw;
  const int hd = mh::win_head_dim(C, nH);
  if (!hd || !mh::win_geo(B, H, W, w, &g, &nw) || !mh::ok_args(qkv, dqkv, nw, w * w, C, nH, hd) ||
      !mh::ok_args(out, dout, nw, w * w, C, nH, hd) || !lse || !dvec)
    return ESVIT_ERR_BAD_ARG;
  return hd == 64 ? mh::bwd_launch<true, 64>(qkv, out, dout, lse, dvec, dqkv, nw, w * w, C, nH, scale, g, stream)
                  : mh::bwd_launch<true, 32>(qkv, out, dout, lse, dvec, dqkv, nw, w * w, C, nH, scale, g, stream);
}
