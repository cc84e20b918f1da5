// Vision Longformer sliding-chunk attention with one global token (ViL, W = 7, head dim 32), forward and backward.
//
// Reference: layers/longformer2d.py  Long2DSCSelfAttention.forward :139-330 with Nglo = 1, exact = 0 (zero padding),
// rpe = True, sharew = True, only_glo = False, add_pooled = False; layers/slidingchunk_2d.py (the nine rolled einsums
// :24-127 and the zero mask _get_invalid_locations_mask_zero :267-287, called with the chunk counts as nx, ny :272).
//
// Token layout per image: N = 1 + nx*ny rows, row 0 the global token, then the nx x ny map row-major (:159-169).
// q bf16 [B*N, C] (the query GEMM output, unscaled; the kernels apply `scale`), kv bf16 [B*N, 2C] channel order
// [k|v][head][32] (:160), out / dout bf16 [B*N, C], dq bf16 [B*N, C], dkv bf16 [B*N, 2C].
// The map is zero-padded to mx*7 x my*7 and cut into mx x my chunks of 7 x 7 (chunk id cm*my + cn).  Query l of chunk
// (cm, cn) sees the global key, then neighbour chunk j = 3*(dx+1) + (dy+1) at (cm+dx, cn+dy):
//   mode 0: all nine j (order of slidingchunk_qk :34-63);
//   mode i in 1..8: its own chunk (j = 4) and j = (i > 4 ? i : i-1) (mode_dict :12-21, :68-76, mask columns :341-350);
//   mode -1: its own chunk only (:64-67, :155-156).
// A stored mode outside -1..8 is clamped into that range (read_mode), so no value can address outside the bias.
// A key is masked (-inf) when its chunk lies off the chunk grid or its position lies in the zero padding (the closed
// form of the zero mask).  One softmax over [global | local] (:280).  The mode is read from device memory, so a
// captured CUDA graph follows the value written before each replay.
// bias fp32 [nH, 49, 1 + 9*49]: column 0 = local->global (g2l[1], :238), column 1 + j*49 + r = the relative-position
// bias of key r of neighbour j (relative_position_index :57-102 gathered by the caller); in mode i > 0 only columns of
// j = 4 and the mode's chunk are read, and dbias holds zeros elsewhere (so the caller's gather is mode-independent).
// bias_g fp32 [nH, N]: the global row's bias (g2g, then g2l[0] broadcast, :316-322).
//
// Local forward: one CTA (4 warps) per (image, head, chunk): 64 query rows (49 used, 16 per warp), one 64-key tile per
// neighbour chunk (49 keys; the own chunk's tile carries the global key in row 49 and goes first, so every row's running
// max is finite from the first tile on), mma.sync m16n8k16 bf16 with fp32 accumulation and an fp32 online softmax in
// the log2 domain.  K / V rows are gathered straight from kv with cp.async (no rolled, padded or unfolded copies).
// Global forward: one CTA per (image, head): each thread a strided share of the N keys with its own online softmax,
// combined in a fixed thread order.
//
// Backward (no floating-point atomics: every output is written by one thread, partials are summed in a fixed order):
//   local dq   CTA per (chunk, head, image segment), images in order: P = ex2(s' - lse'), dP = dO V^T, dS = P (dP - D),
//              dQ = scale dS K; writes D = rowsum(dO * O), dS summed over its images into a [49, 442] bias partial, and
//              the chunk's share of the global key's dK / dV (column 49 of the own tile).
//   global     CTA per (image, head): the global row's dq, P and dS of every key (kept for dkdv and the bias), and the
//              global key's dK / dV (its own term plus the chunk shares in chunk order).
//   local dkdv CTA per (image, head, key chunk): loops over the query chunks that see this chunk (c - offset_j for the
//              mode's j), dV = P^T dO, dK = scale dS^T Q, plus the global query's term.
//   reduce     dbias = the bias partials summed over (segment, chunk) in order; dbias_g = dS_g summed over images.
#include "wa_common.cuh"

namespace vil {

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

constexpr int W = 7, W2 = 49, HD = 32, LD = 40, TILE = 64 * LD, NTHR = 128;
constexpr int NB = 1 + 9 * W2;  // bias columns

struct Geo {
  int B, nx, ny, mx, my, N, C, nH, nchunk;
};

// neighbour chunk j of tile t (the own chunk first)
__device__ __forceinline__ int tile_nb(int mode, int t) {
  if (t == 0) return 4;
  if (mode == 0) return t - 1 + (t >= 5);
  return mode > 4 ? mode : mode - 1;
}
__device__ __forceinline__ int ntiles(int mode) { return mode == 0 ? 9 : (mode < 0 ? 1 : 2); }
__device__ __forceinline__ int read_mode(const int* p) { return min(max(*p, -1), 8); }

// kv / q row of key r of neighbour j of chunk (cm, cn) of image b; the own tile's row 49 is the global token; -1 masked
__device__ __forceinline__ long long key_row(const Geo& g, int b, int cm, int cn, int j, int r) {
  if (r == W2 && j == 4) return (long long)b * g.N;
  if (r >= W2) return -1;
  const int X = (cm + j / 3 - 1) * W + r / W, Y = (cn + j % 3 - 1) * W + r % W;
  if (X < 0 || X >= g.nx || Y < 0 || Y >= g.ny) return -1;
  return (long long)b * g.N + 1 + X * g.ny + Y;
}
// row of query l of chunk (cm, cn), -1 for a padded position
__device__ __forceinline__ long long q_row(const Geo& g, int b, int cm, int cn, int l) {
  if (l >= W2) return -1;
  const int X = cm * W + l / W, Y = cn * W + l % W;
  if (X >= g.nx || Y >= g.ny) return -1;
  return (long long)b * g.N + 1 + X * g.ny + Y;
}

// [64 x 32] bf16 tile of rows row(r) (zero where row(r) < 0) of a matrix with row stride ld, columns from src
template <typename RowFn>
__device__ __forceinline__ void load_tile(bf16* dst, const bf16* __restrict__ src, long long ld, RowFn row) {
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const int e = threadIdx.x + k * NTHR;  // 256 chunks of 16 B
    const int r = e >> 2, c = (e & 3) * 8;
    const long long rr = row(r);
    cp_async16(dst + r * LD + c, src + (rr >= 0 ? rr * ld : 0) + c, rr >= 0 ? 16 : 0);
  }
}

__device__ __forceinline__ void load_a(uint32_t (&a)[2][4], const bf16* t, int r0, int lane) {
  const bf16* p = t + (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
  ldsm_x4(a[0], p);
  ldsm_x4(a[1], p + 16);
}

// acc[nt] (16 x 64) = A (16 x 32) . T^T, T = 64 rows x 32
__device__ __forceinline__ void mma_abt(float (&acc)[8][4], const uint32_t (&a)[2][4], const bf16* t, int lane) {
#pragma unroll
  for (int nt = 0; nt < 8; nt++) {
    acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
    uint32_t b[4];
    ldsm_x4(b, t + (nt * 8 + (lane & 7)) * LD + (lane >> 3) * 8);
    mma16816(acc[nt], a[0], b[0], b[1]);
    mma16816(acc[nt], a[1], b[2], b[3]);
  }
}

// o (16 x 32) += P (16 x 64, rounded to bf16) . T, T = 64 rows (k) x 32
__device__ __forceinline__ void mma_pt(float (&o)[4][4], const float (&p)[8][4], const bf16* t, int lane) {
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
    uint32_t pa[4];
    pa[0] = pack_bf162(p[2 * kk][0], p[2 * kk][1]);
    pa[1] = pack_bf162(p[2 * kk][2], p[2 * kk][3]);
    pa[2] = pack_bf162(p[2 * kk + 1][0], p[2 * kk + 1][1]);
    pa[3] = pack_bf162(p[2 * kk + 1][2], p[2 * kk + 1][3]);
    const bf16* vp = t + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
#pragma unroll
    for (int d16 = 0; d16 < 2; d16++) {
      uint32_t vb[4];
      ldsm_x4_t(vb, vp + d16 * 16);
      mma16816(o[2 * d16], pa, vb[0], vb[1]);
      mma16816(o[2 * d16 + 1], pa, vb[2], vb[3]);
    }
  }
}

__device__ __forceinline__ void store_row(bf16* __restrict__ dst, const float (&o)[4][4], int hi, float s, int lane) {
#pragma unroll
  for (int dt = 0; dt < 4; dt++)
    *reinterpret_cast<uint32_t*>(dst + dt * 8 + (lane & 3) * 2) = pack_bf162(o[dt][2 * hi] * s, o[dt][2 * hi + 1] * s);
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// scores of one 16 x 64 fragment block against the tile of neighbour j, log2 domain, masked keys -inf:
// s = c2 * acc + bias * log2(e); rows >= 49 get no bias
__device__ __forceinline__ void scores(float (&s)[8][4], const Geo& g, const float* __restrict__ bias_h, int b, int cm,
                                       int cn, int j, int lA, int lB, float c2, int lane) {
#pragma unroll
  for (int nt = 0; nt < 8; nt++) {
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int r = nt * 8 + (lane & 3) * 2 + e;
      const bool ok = key_row(g, b, cm, cn, j, r) >= 0;
      const int col = r < W2 ? 1 + j * W2 + r : 0;
      const float bA = lA < W2 ? __ldg(bias_h + lA * NB + col) * LOG2E : 0.f;
      const float bB = lB < W2 ? __ldg(bias_h + lB * NB + col) * LOG2E : 0.f;
      s[nt][e] = ok ? s[nt][e] * c2 + bA : -INFINITY;
      s[nt][2 + e] = ok ? s[nt][2 + e] * c2 + bB : -INFINITY;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NTHR) sc_fwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                      const float* __restrict__ bias, const int* __restrict__ mode_p,
                                                      bf16* __restrict__ out, float* __restrict__ lse, const Geo g,
                                                      float c2) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);  // [Q | K0 | V0 | K1 | V1]
  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int cm = chunk / g.my, cn = chunk - cm * g.my;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mode = read_mode(mode_p);
  const int nt_ = ntiles(mode);
  const long long C2 = 2LL * g.C;
  load_tile(Qs, q + h * HD, g.C, [&](int r) { return q_row(g, b, cm, cn, r); });
  load_tile(Qs + TILE, kv + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, 4, r); });
  load_tile(Qs + 2 * TILE, kv + g.C + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, 4, r); });
  cp_async_commit();
  const int lA = warp * 16 + (lane >> 2), lB = lA + 8;
  const float* bias_h = bias + (long long)h * W2 * NB;
  float m0 = -INFINITY, m1 = -INFINITY, s0 = 0.f, s1 = 0.f;
  float o[4][4];
#pragma unroll
  for (int dt = 0; dt < 4; dt++) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
  uint32_t qa[2][4];
  for (int t = 0; t < nt_; t++) {
    const int st = t & 1;
    if (t + 1 < nt_) {
      const int jn = tile_nb(mode, t + 1);
      bf16* nx = Qs + (1 + 2 * (st ^ 1)) * TILE;
      load_tile(nx, kv + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, jn, r); });
      load_tile(nx + TILE, kv + g.C + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, jn, r); });
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Ks = Qs + (1 + 2 * st) * TILE;
    if (t == 0) load_a(qa, Qs, warp * 16, lane);
    float s[8][4];
    mma_abt(s, qa, Ks, lane);
    scores(s, g, bias_h, b, cm, cn, tile_nb(mode, t), lA, lB, c2, lane);
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      mx0 = fmaxf(mx0, fmaxf(s[nt][0], s[nt][1]));
      mx1 = fmaxf(mx1, fmaxf(s[nt][2], s[nt][3]));
    }
    mx0 = quad_max(mx0);  // finite: tile 0 holds the global key
    mx1 = quad_max(mx1);
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
    s0 = s0 * a0 + r0;
    s1 = s1 * a1 + r1;
#pragma unroll
    for (int dt = 0; dt < 4; dt++) {
      o[dt][0] *= a0; o[dt][1] *= a0;
      o[dt][2] *= a1; o[dt][3] *= a1;
    }
    mma_pt(o, s, Ks + TILE, lane);
    __syncthreads();
  }
  cp_async_wait<0>();
  s0 = quad_sum(s0);
  s1 = quad_sum(s1);
  const long long oA = q_row(g, b, cm, cn, lA), oB = q_row(g, b, cm, cn, lB);
  if (oA >= 0) store_row(out + oA * g.C + h * HD, o, 0, __fdividef(1.f, s0), lane);
  if (oB >= 0) store_row(out + oB * g.C + h * HD, o, 1, __fdividef(1.f, s1), lane);
  if ((lane & 3) == 0) {
    float* lp = lse + (((long long)b * g.nH + h) * g.nchunk + chunk) * W2;
    if (lA < W2) lp[lA] = (m0 + lg2(s0)) * LN2;
    if (lB < W2) lp[lB] = (m1 + lg2(s1)) * LN2;
  }
}

// 32 bf16 of a row -> fp32
__device__ __forceinline__ void load_row32(float (&v)[HD], const bf16* __restrict__ p) {
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(p) + k);
    const bf162* h2 = reinterpret_cast<const bf162*>(&u);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float2 f = __bfloat1622float2(h2[i]);
      v[k * 8 + 2 * i] = f.x;
      v[k * 8 + 2 * i + 1] = f.y;
    }
  }
}

// global query (row 0) of (image, head) over all N keys
__global__ void __launch_bounds__(NTHR, 4) glo_fwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                       const float* __restrict__ bias_g, bf16* __restrict__ out,
                                                       float* __restrict__ lse_g, const Geo g, float c2) {
  __shared__ float qs[HD];
  __shared__ float red[NTHR][HD + 3];
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const long long base = (long long)b * g.N;
  if (tid < HD) qs[tid] = __bfloat162float(q[base * g.C + h * HD + tid]);
  __syncthreads();
  float m = -INFINITY, l = 0.f, o[HD];
#pragma unroll
  for (int d = 0; d < HD; d++) o[d] = 0.f;
  const float* bh = bias_g + (long long)h * g.N;
  for (int r = tid; r < g.N; r += NTHR) {
    float k[HD];
    load_row32(k, kv + (base + r) * 2 * g.C + h * HD);
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD; d++) s = fmaf(qs[d], k[d], s);
    s = s * c2 + __ldg(bh + r) * LOG2E;
    const float mn = fmaxf(m, s), a = ex2(m - mn), p = ex2(s - mn);
    m = mn;
    l = l * a + p;
    load_row32(k, kv + (base + r) * 2 * g.C + g.C + h * HD);  // v
#pragma unroll
    for (int d = 0; d < HD; d++) o[d] = fmaf(p, k[d], o[d] * a);
  }
  red[tid][0] = m;
  red[tid][1] = l;
#pragma unroll
  for (int d = 0; d < HD; d++) red[tid][2 + d] = o[d];
  __syncthreads();
  if (tid < HD) {
    float M = -INFINITY;
    for (int i = 0; i < NTHR; i++) M = fmaxf(M, red[i][0]);
    float L = 0.f, O = 0.f;
    for (int i = 0; i < NTHR; i++) {
      const float a = ex2(red[i][0] - M);  // 0 for a thread without keys
      L += red[i][1] * a;
      O += red[i][2 + tid] * a;
    }
    out[base * g.C + h * HD + tid] = __float2bfloat16(O / L);
    if (tid == 0) lse_g[(long long)b * g.nH + h] = (M + lg2(L)) * LN2;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// local dQ over images [b0, b1) of one (chunk, head); dvec = D of every local query row; part_bias fp32 [49, NB] of
// this (segment, head, chunk); part_g fp32 [B, nH, nchunk, 2 * 32] = the chunk's dS^T Q | P^T dO at the global key
__global__ void __launch_bounds__(NTHR) sc_dq_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                     const float* __restrict__ bias, const int* __restrict__ mode_p,
                                                     const bf16* __restrict__ out, const bf16* __restrict__ dout,
                                                     const float* __restrict__ lse, float* __restrict__ dvec,
                                                     bf16* __restrict__ dq, float* __restrict__ part_bias,
                                                     float* __restrict__ part_g, const Geo g, int seg_len, float c2,
                                                     float scale) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);     // [Q | dO | O | K0 | V0 | K1 | V1]
  float* acc = reinterpret_cast<float*>(Qs + 7 * TILE);  // [9][64][64] dS summed over images
  float* stat = acc + 9 * 64 * 64;                       // lse' 64 | D 64 | dS_glo 64 | P_glo 64
  const int chunk = blockIdx.x, h = blockIdx.y, seg = blockIdx.z;
  const int cm = chunk / g.my, cn = chunk - cm * g.my;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mode = read_mode(mode_p);
  const int nt_ = ntiles(mode);
  const long long C2 = 2LL * g.C;
  const int lA = warp * 16 + (lane >> 2), lB = lA + 8;
  const float* bias_h = bias + (long long)h * W2 * NB;
  for (int i = threadIdx.x; i < 9 * 64 * 64; i += NTHR) acc[i] = 0.f;
  const int b0 = seg * seg_len, b1 = min(g.B, b0 + seg_len);
  for (int b = b0; b < b1; b++) {
    load_tile(Qs, q + h * HD, g.C, [&](int r) { return q_row(g, b, cm, cn, r); });
    load_tile(Qs + TILE, dout + h * HD, g.C, [&](int r) { return q_row(g, b, cm, cn, r); });
    load_tile(Qs + 2 * TILE, out + h * HD, g.C, [&](int r) { return q_row(g, b, cm, cn, r); });
    load_tile(Qs + 3 * TILE, kv + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, 4, r); });
    load_tile(Qs + 4 * TILE, kv + g.C + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, 4, r); });
    cp_async_commit();
    const long long srow = (((long long)b * g.nH + h) * g.nchunk + chunk) * W2;
    float dq_[4][4];
#pragma unroll
    for (int dt = 0; dt < 4; dt++) dq_[dt][0] = dq_[dt][1] = dq_[dt][2] = dq_[dt][3] = 0.f;
    uint32_t qa[2][4], oa[2][4];
    float LA = 0.f, LB = 0.f, DA = 0.f, DB = 0.f;
    for (int t = 0; t < nt_; t++) {
      const int st = t & 1;
      if (t + 1 < nt_) {
        const int jn = tile_nb(mode, t + 1);
        bf16* nx = Qs + (3 + 2 * (st ^ 1)) * TILE;
        load_tile(nx, kv + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, jn, r); });
        load_tile(nx + TILE, kv + g.C + h * HD, C2, [&](int r) { return key_row(g, b, cm, cn, jn, r); });
      }
      cp_async_commit();
      cp_async_wait<1>();
      __syncthreads();
      if (t == 0) {
        if (threadIdx.x < 64) {  // D = rowsum(dO * O) (0 on padded rows: dO reads as 0); lse'
          const int l = threadIdx.x;
          float d = 0.f;
          for (int k = 0; k < HD; k++)
            d = fmaf(__bfloat162float(Qs[TILE + l * LD + k]), __bfloat162float(Qs[2 * TILE + l * LD + k]), d);
          stat[64 + l] = d;
          stat[l] = l < W2 ? lse[srow + l] * LOG2E : 0.f;
          if (l < W2) dvec[srow + l] = d;
        }
        __syncthreads();
        load_a(qa, Qs, warp * 16, lane);
        load_a(oa, Qs + TILE, warp * 16, lane);
        LA = stat[lA]; LB = stat[lB];
        DA = stat[64 + lA]; DB = stat[64 + lB];
      }
      const bf16* Ks = Qs + (3 + 2 * st) * TILE;
      const int j = tile_nb(mode, t);
      float p[8][4], dp[8][4];
      mma_abt(p, qa, Ks, lane);
      mma_abt(dp, oa, Ks + TILE, lane);
      scores(p, g, bias_h, b, cm, cn, j, lA, lB, c2, lane);
      float* at = acc + t * 64 * 64;
#pragma unroll
      for (int nt = 0; nt < 8; nt++) {
        const int col = nt * 8 + (lane & 3) * 2;
        p[nt][0] = ex2(p[nt][0] - LA);
        p[nt][1] = ex2(p[nt][1] - LA);
        p[nt][2] = ex2(p[nt][2] - LB);
        p[nt][3] = ex2(p[nt][3] - LB);
        if (t == 0 && col == 48) {  // column 49 of the own tile: the global key
          stat[128 + lA] = p[nt][1] * (dp[nt][1] - DA);
          stat[128 + lB] = p[nt][3] * (dp[nt][3] - DB);
          stat[192 + lA] = p[nt][1];
          stat[192 + lB] = p[nt][3];
        }
        p[nt][0] *= dp[nt][0] - DA;
        p[nt][1] *= dp[nt][1] - DA;
        p[nt][2] *= dp[nt][2] - DB;
        p[nt][3] *= dp[nt][3] - DB;
        at[lA * 64 + col] += p[nt][0];
        at[lA * 64 + col + 1] += p[nt][1];
        at[lB * 64 + col] += p[nt][2];
        at[lB * 64 + col + 1] += p[nt][3];
      }
      mma_pt(dq_, p, Ks, lane);
      __syncthreads();
    }
    cp_async_wait<0>();
    const long long oA = q_row(g, b, cm, cn, lA), oB = q_row(g, b, cm, cn, lB);
    if (oA >= 0) store_row(dq + oA * g.C + h * HD, dq_, 0, scale, lane);
    if (oB >= 0) store_row(dq + oB * g.C + h * HD, dq_, 1, scale, lane);
    if (threadIdx.x < 2 * HD) {  // the global key's share: sum_l dS_l q_l | sum_l P_l dO_l over the 49 rows in order
      const int d = threadIdx.x & (HD - 1), w = threadIdx.x >> 5;
      const float* coef = stat + (w ? 192 : 128);
      const bf16* src = Qs + (w ? TILE : 0) + d;
      float s = 0.f;
      for (int l = 0; l < W2; l++) s = fmaf(coef[l], __bfloat162float(src[l * LD]), s);
      part_g[(((long long)b * g.nH + h) * g.nchunk + chunk) * 2 * HD + threadIdx.x] = s;
    }
    __syncthreads();  // the next image's loads overwrite Q / dO / O and stat
  }
  float* pb = part_bias + (((long long)seg * g.nH + h) * g.nchunk + chunk) * W2 * NB;
  for (int i = threadIdx.x; i < W2 * NB; i += NTHR) {
    const int l = i / NB, col = i - l * NB;
    float v = 0.f;
    if (col == 0) {
      v = acc[l * 64 + W2];
    } else {
      const int jj = (col - 1) / W2, r = (col - 1) - jj * W2;
      int t = -1;
      if (jj == 4) t = 0;
      else if (mode == 0) t = jj < 4 ? jj + 1 : jj;
      else if (mode > 0 && jj == tile_nb(mode, 1)) t = 1;
      if (t >= 0) v = acc[(t * 64 + l) * 64 + r];
    }
    pb[i] = v;
  }
}

// global row backward per (image, head): dq of row 0, P_g / dS_g of every key (pds [B, nH, N, 2]), and dK / dV of the
// global key (its own term plus the chunk shares of part_g in chunk order)
__global__ void __launch_bounds__(NTHR) glo_bwd_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                       const float* __restrict__ bias_g, const bf16* __restrict__ out,
                                                       const bf16* __restrict__ dout, const float* __restrict__ lse_g,
                                                       const float* __restrict__ part_g, float* __restrict__ pds,
                                                       bf16* __restrict__ dq, bf16* __restrict__ dkv, const Geo g,
                                                       float c2, float scale) {
  __shared__ float qs[HD], gs[HD], dsh;
  __shared__ float red[NTHR][HD + 1];
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const long long base = (long long)b * g.N;
  if (tid < HD) {
    qs[tid] = __bfloat162float(q[base * g.C + h * HD + tid]);
    gs[tid] = __bfloat162float(dout[base * g.C + h * HD + tid]);
  }
  if (tid == 0) {
    float d = 0.f;
    for (int k = 0; k < HD; k++)
      d = fmaf(__bfloat162float(dout[base * g.C + h * HD + k]), __bfloat162float(out[base * g.C + h * HD + k]), d);
    dsh = d;
  }
  __syncthreads();
  const float D = dsh, L = lse_g[(long long)b * g.nH + h] * LOG2E;
  const float* bh = bias_g + (long long)h * g.N;
  float* pd = pds + ((long long)b * g.nH + h) * g.N * 2;
  float acc[HD];
#pragma unroll
  for (int d = 0; d < HD; d++) acc[d] = 0.f;
  for (int r = tid; r < g.N; r += NTHR) {
    float k[HD], v[HD];
    load_row32(k, kv + (base + r) * 2 * g.C + h * HD);
    load_row32(v, kv + (base + r) * 2 * g.C + g.C + h * HD);
    float s = 0.f, dp = 0.f;
#pragma unroll
    for (int d = 0; d < HD; d++) {
      s = fmaf(qs[d], k[d], s);
      dp = fmaf(gs[d], v[d], dp);
    }
    const float p = ex2(s * c2 + __ldg(bh + r) * LOG2E - L), ds = p * (dp - D);
    pd[2 * r] = p;
    pd[2 * r + 1] = ds;
#pragma unroll
    for (int d = 0; d < HD; d++) acc[d] = fmaf(ds, k[d], acc[d]);
  }
#pragma unroll
  for (int d = 0; d < HD; d++) red[tid][d] = acc[d];
  __syncthreads();
  if (tid < HD) {
    float s = 0.f;
    for (int i = 0; i < NTHR; i++) s += red[i][tid];
    dq[base * g.C + h * HD + tid] = __float2bfloat16(s * scale);
  } else if (tid < 3 * HD) {  // the global key: dK (tid 32..63), dV (tid 64..95)
    const int d = tid & (HD - 1), w = tid < 2 * HD ? 0 : 1;
    const float p0 = pd[0], ds0 = pd[1];  // written by thread 0 before the barrier
    float s = w ? p0 * gs[d] : ds0 * qs[d];
    const float* pg = part_g + ((long long)b * g.nH + h) * g.nchunk * 2 * HD + w * HD + d;
    for (int c = 0; c < g.nchunk; c++) s += pg[(long long)c * 2 * HD];
    dkv[base * 2 * g.C + w * g.C + h * HD + d] = __float2bfloat16(w ? s : s * scale);
  }
}

// local dK / dV of the 49 keys of one (image, head, chunk)
__global__ void __launch_bounds__(NTHR) sc_dkdv_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                       const float* __restrict__ bias, const int* __restrict__ mode_p,
                                                       const bf16* __restrict__ dout, const float* __restrict__ lse,
                                                       const float* __restrict__ dvec, const float* __restrict__ pds,
                                                       bf16* __restrict__ dkv, const Geo g, float c2, float scale) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Ks = reinterpret_cast<bf16*>(smraw);              // [K | V | Q0 | dO0 | Q1 | dO1]
  float* stat = reinterpret_cast<float*>(Ks + 6 * TILE);  // [2 stages][lse' 64 | D 64]; q_g 32 | dO_g 32
  const int chunk = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int cm = chunk / g.my, cn = chunk - cm * g.my;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int mode = read_mode(mode_p);
  const long long C2 = 2LL * g.C;
  // the query chunks that see this chunk: (cm, cn) - offset_j for the mode's neighbours j on the grid, j packed in 4 bits
  unsigned long long js = 0;
  int n = 0;
  for (int t = 0; t < ntiles(mode); t++) {
    const int j = tile_nb(mode, t), m2 = cm - (j / 3 - 1), n2 = cn - (j % 3 - 1);
    if (m2 >= 0 && m2 < g.mx && n2 >= 0 && n2 < g.my) js |= (unsigned long long)j << (4 * n++);
  }
  load_tile(Ks, kv + h * HD, C2, [&](int r) { return r < W2 ? key_row(g, b, cm, cn, 4, r) : -1LL; });
  load_tile(Ks + TILE, kv + g.C + h * HD, C2, [&](int r) { return r < W2 ? key_row(g, b, cm, cn, 4, r) : -1LL; });
  auto load_q = [&](int i, int st) {
    const int j = (int)(js >> (4 * i)) & 15, m2 = cm - (j / 3 - 1), n2 = cn - (j % 3 - 1), c = m2 * g.my + n2;
    bf16* dst = Ks + (2 + 2 * st) * TILE;
    load_tile(dst, q + h * HD, g.C, [&](int r) { return q_row(g, b, m2, n2, r); });
    load_tile(dst + TILE, dout + h * HD, g.C, [&](int r) { return q_row(g, b, m2, n2, r); });
    if (threadIdx.x < 64) {  // query rows past 49: lse' = +inf -> P = 0
      const int l = threadIdx.x;
      const long long srow = (((long long)b * g.nH + h) * g.nchunk + c) * W2;
      stat[st * 128 + l] = l < W2 ? lse[srow + l] * LOG2E : INFINITY;
      stat[st * 128 + 64 + l] = l < W2 ? dvec[srow + l] : 0.f;
    }
  };
  if (n > 0) load_q(0, 0);
  cp_async_commit();
  float* glo = stat + 256;
  if (threadIdx.x < 2 * HD) {
    const long long row = (long long)b * g.N;
    glo[threadIdx.x] = __bfloat162float(threadIdx.x < HD ? q[row * g.C + h * HD + threadIdx.x]
                                                         : dout[row * g.C + h * HD + threadIdx.x - HD]);
  }
  const float* bias_h = bias + (long long)h * W2 * NB;
  float dk[4][4], dv[4][4];
#pragma unroll
  for (int dt = 0; dt < 4; dt++)
#pragma unroll
    for (int i = 0; i < 4; i++) dk[dt][i] = dv[dt][i] = 0.f;
  uint32_t ka[2][4], va[2][4];
  const int rA = warp * 16 + (lane >> 2), rB = rA + 8;
  for (int i = 0; i < n; i++) {
    const int st = i & 1;
    if (i + 1 < n) load_q(i + 1, st ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Qs = Ks + (2 + 2 * st) * TILE;
    const float* sl = stat + st * 128;
    if (i == 0) {
      load_a(ka, Ks, warp * 16, lane);
      load_a(va, Ks + TILE, warp * 16, lane);
    }
    const int j = (int)(js >> (4 * i)) & 15;
    float p[8][4], dp[8][4];
    mma_abt(p, ka, Qs, lane);          // S^T: keys x queries
    mma_abt(dp, va, Qs + TILE, lane);  // dP^T = V dO^T
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int l = nt * 8 + (lane & 3) * 2 + e;
        const float* bl = bias_h + (long long)l * NB + 1 + j * W2;
        const float bA = (l < W2 && rA < W2) ? __ldg(bl + rA) * LOG2E : 0.f;
        const float bB = (l < W2 && rB < W2) ? __ldg(bl + rB) * LOG2E : 0.f;
        p[nt][e] = ex2(p[nt][e] * c2 + bA - sl[l]);
        p[nt][2 + e] = ex2(p[nt][2 + e] * c2 + bB - sl[l]);
      }
    }
    mma_pt(dv, p, Qs + TILE, lane);  // dV += P^T dO
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
      const int l = nt * 8 + (lane & 3) * 2;
      p[nt][0] *= dp[nt][0] - sl[64 + l];
      p[nt][1] *= dp[nt][1] - sl[64 + l + 1];
      p[nt][2] *= dp[nt][2] - sl[64 + l];
      p[nt][3] *= dp[nt][3] - sl[64 + l + 1];
    }
    mma_pt(dk, p, Qs, lane);  // dK += dS^T Q
    __syncthreads();
  }
  cp_async_wait<0>();
  __syncthreads();  // glo
  const long long oA = rA < W2 ? key_row(g, b, cm, cn, 4, rA) : -1, oB = rB < W2 ? key_row(g, b, cm, cn, 4, rB) : -1;
  const float* pd = pds + ((long long)b * g.nH + h) * g.N * 2;
#pragma unroll
  for (int hi = 0; hi < 2; hi++) {
    const long long row = hi ? oB : oA;
    if (row < 0) continue;
    const long long r = row - (long long)b * g.N;
    const float pg = pd[2 * r], dsg = pd[2 * r + 1];
#pragma unroll
    for (int dt = 0; dt < 4; dt++) {
      const int d = dt * 8 + (lane & 3) * 2;
      dk[dt][2 * hi] = (dk[dt][2 * hi] + dsg * glo[d]) * scale;
      dk[dt][2 * hi + 1] = (dk[dt][2 * hi + 1] + dsg * glo[d + 1]) * scale;
      dv[dt][2 * hi] += pg * glo[HD + d];
      dv[dt][2 * hi + 1] += pg * glo[HD + d + 1];
    }
    store_row(dkv + row * C2 + h * HD, dk, hi, 1.f, lane);
    store_row(dkv + row * C2 + g.C + h * HD, dv, hi, 1.f, lane);
  }
}

// dbias [nH, 49*NB] = sum over (segment, chunk) of the partials; dbias_g [nH, N] = sum over images of dS_g
__global__ void reduce_kernel(const float* __restrict__ part_bias, const float* __restrict__ pds,
                              float* __restrict__ dbias, float* __restrict__ dbias_g, const Geo g, int nseg) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nb = (long long)g.nH * W2 * NB, ng = (long long)g.nH * g.N;
  if (i < nb) {
    const int h = (int)(i / (W2 * NB));
    const long long e = i - (long long)h * W2 * NB;
    float s = 0.f;
    for (int sg = 0; sg < nseg; sg++)
      for (int c = 0; c < g.nchunk; c++) s += part_bias[(((long long)sg * g.nH + h) * g.nchunk + c) * W2 * NB + e];
    dbias[i] = s;
  } else if (i < nb + ng) {
    const long long k = i - nb;
    const int h = (int)(k / g.N);
    const long long r = k - (long long)h * g.N;
    float s = 0.f;
    for (int b = 0; b < g.B; b++) s += pds[(((long long)b * g.nH + h) * g.N + r) * 2 + 1];
    dbias_g[k] = s;
  }
}

constexpr size_t FWD_SMEM = 5 * TILE * sizeof(bf16);
constexpr size_t DQ_SMEM = 7 * TILE * sizeof(bf16) + (9 * 64 * 64 + 256) * sizeof(float);
constexpr size_t DKDV_SMEM = 6 * TILE * sizeof(bf16) + (256 + 2 * HD) * sizeof(float);

static bool geo(int B, int nx, int ny, int nH, Geo* g) {
  if (B < 1 || B > 65535 || nx < 1 || ny < 1 || nH < 1 || nH > 65535) return false;
  g->B = B; g->nx = nx; g->ny = ny; g->nH = nH; g->C = nH * HD;
  g->mx = (nx + W - 1) / W; g->my = (ny + W - 1) / W;
  g->N = 1 + nx * ny; g->nchunk = g->mx * g->my;
  return (long long)B * g->N * 2 * g->C < (1LL << 40);
}

// images per dq segment: enough (chunk, head, segment) CTAs for two waves of 132 SMs
static int seg_len(const Geo& g) {
  const int per = g.nchunk * g.nH;
  int nseg = (264 + per - 1) / per;
  if (nseg > g.B) nseg = g.B;
  return (g.B + nseg - 1) / nseg;
}

static long long ws_floats(const Geo& g) {
  const int sl = seg_len(g), nseg = (g.B + sl - 1) / sl;
  return (long long)nseg * g.nH * g.nchunk * W2 * NB             // bias partials
         + (long long)g.B * g.nH * g.nchunk * 2 * HD              // global-key shares
         + (long long)g.B * g.nH * g.N * 2;                       // P_g, dS_g
}

static bool aligned(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace vil

ESVIT_API int esvit_vil_sc_ws_floats(int B, int nx, int ny, int nH) {
  vil::Geo g;
  if (!vil::geo(B, nx, ny, nH, &g)) return -1;
  const long long n = vil::ws_floats(g);
  return n > 0x7fffffffLL ? -1 : (int)n;
}

ESVIT_API int esvit_vil_sc_fwd(const void* q, const void* kv, const float* bias, const float* bias_g, const int* mode,
                               void* out, float* lse, float* lse_g, int B, int nx, int ny, int nH, float scale,
                               void* stream) {
  vil::Geo g;
  if (!vil::geo(B, nx, ny, nH, &g) || !q || !kv || !bias || !bias_g || !mode || !out || !lse || !lse_g ||
      !vil::aligned(q) || !vil::aligned(kv) || !vil::aligned(out))
    return ESVIT_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const float c2 = scale * vil::LOG2E;
  vil::sc_fwd_kernel<<<dim3(g.nchunk, nH, B), vil::NTHR, vil::FWD_SMEM, st>>>(
      (const bf16*)q, (const bf16*)kv, bias, mode, (bf16*)out, lse, g, c2);
  vil::glo_fwd_kernel<<<dim3(nH, B), vil::NTHR, 0, st>>>((const bf16*)q, (const bf16*)kv, bias_g, (bf16*)out, lse_g, g,
                                                         c2);
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_vil_sc_bwd(const void* q, const void* kv, const float* bias, const float* bias_g, const int* mode,
                               const void* out, const void* dout, const float* lse, const float* lse_g, float* dvec,
                               float* ws, void* dq, void* dkv, float* dbias, float* dbias_g, int B, int nx, int ny,
                               int nH, float scale, void* stream) {
  vil::Geo g;
  if (!vil::geo(B, nx, ny, nH, &g) || !q || !kv || !bias || !bias_g || !mode || !out || !dout || !lse || !lse_g ||
      !dvec || !ws || !dq || !dkv || !dbias || !dbias_g || !vil::aligned(q) || !vil::aligned(kv) ||
      !vil::aligned(out) || !vil::aligned(dout) || !vil::aligned(dq) || !vil::aligned(dkv))
    return ESVIT_ERR_BAD_ARG;
  cudaError_t e = cudaFuncSetAttribute(vil::sc_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)vil::DQ_SMEM);
  if (e != cudaSuccess) return (int)e;
  cudaStream_t st = (cudaStream_t)stream;
  const float c2 = scale * vil::LOG2E;
  const int sl = vil::seg_len(g), nseg = (B + sl - 1) / sl;
  float* part_bias = ws;
  float* part_g = part_bias + (long long)nseg * nH * g.nchunk * vil::W2 * vil::NB;
  float* pds = part_g + (long long)B * nH * g.nchunk * 2 * vil::HD;
  vil::sc_dq_kernel<<<dim3(g.nchunk, nH, nseg), vil::NTHR, vil::DQ_SMEM, st>>>(
      (const bf16*)q, (const bf16*)kv, bias, mode, (const bf16*)out, (const bf16*)dout, lse, dvec, (bf16*)dq,
      part_bias, part_g, g, sl, c2, scale);
  vil::glo_bwd_kernel<<<dim3(nH, B), vil::NTHR, 0, st>>>((const bf16*)q, (const bf16*)kv, bias_g, (const bf16*)out,
                                                         (const bf16*)dout, lse_g, part_g, pds, (bf16*)dq, (bf16*)dkv,
                                                         g, c2, scale);
  vil::sc_dkdv_kernel<<<dim3(g.nchunk, nH, B), vil::NTHR, vil::DKDV_SMEM, st>>>(
      (const bf16*)q, (const bf16*)kv, bias, mode, (const bf16*)dout, lse, dvec, pds, (bf16*)dkv, g, c2, scale);
  const long long n = (long long)nH * vil::W2 * vil::NB + (long long)nH * g.N;
  vil::reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(part_bias, pds, dbias, dbias_g, g, nseg);
  ESVIT_LAUNCH_CHECK();
}
