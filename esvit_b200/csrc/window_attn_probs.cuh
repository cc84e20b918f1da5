// Attention probabilities of a (shifted-)window attention call, fp32 [B*nWy*nWx, nH, ws*ws, ws*ws] in the reference's
// layout (models/swin_transformer.py:141-147 softmax, window_partition of the rolled, padded frame :295-308): what
// SwinTransformer.forward_selfattention returns.  Rows AND columns of padded slots are included - the reference pads
// after norm1, so a padded slot's q/k is the qkv bias and its row is a real softmax.
//
// The training kernels never write P.  These kernels recompute S = scale*q k^T + bias (+ -100 shift mask) with the same
// gather (issue7 / issue14, q and k only), the same closed-form bias and region ids and the same bf16 mma.sync, and take
// the row max and sum themselves: the forward writes no log-sum-exp for query tiles that hold no real token (it skips
// them, their outputs are cropped), while the reference returns those rows.
//
// The output is the traffic (ws 7: 9 604 B per (window, head), ws 14: 153 664 B), so P is staged in shared memory and
// stored by whole rows: every warp store covers 128 (ws 7, scalar) or 512 (ws 14, float4) contiguous bytes.  Stores are
// streaming (st.global.cs): nothing here is re-read.
#pragma once
#include "wa_common.cuh"
#include "window_attn7.cuh"
#include "window_attn14.cuh"

namespace wa {

// ws = 7: one CTA = 4 warps = one (window, head) at a time, persistent over windows with the forward's 2-stage cp.async
// gather; a warp holds its 16 x 64 score tile in registers, writes P into a [49 x 49] block and the CTA stores the block.
template <bool SHIFT>
__global__ void __launch_bounds__(128, 4) window_attn_probs7_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bexp,
    float* __restrict__ probs, Geo g, float scale, int nwin_total) {
  constexpr int WS = 7, NT = 49, NP = NT * NT;
  using C = Cfg<WS>;
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* tiles = reinterpret_cast<bf16*>(smraw);                 // [2 stages][Q | K]
  float* Ps = reinterpret_cast<float*>(tiles + 2 * 2 * TILE7);  // [49][49] P of the window being stored
  int* tokb = reinterpret_cast<int*>(Ps + NP + 3);              // [2][64]
  int* ridb = tokb + 2 * 64;                                    // [2][64]

  const int h = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = warp * 16, rA = r0 + (lane >> 2), rB = rA + 8;
  int win = blockIdx.y, stage = 0;
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));
  if (win < nwin_total) issue7<false, 128, 2>(g, win, h, qkv, bchunk, nullptr, nullptr, nullptr, tiles, nullptr, tokb, ridb);
  cp_async_commit();

  float breg[C::NT8][4];
  {
    const float* bh = bexp + (long long)h * 4096 + (lane & 3) * 2;
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      const float2 a = __ldg(reinterpret_cast<const float2*>(bh + rA * 64 + nt * 8));
      const float2 b = __ldg(reinterpret_cast<const float2*>(bh + rB * 64 + nt * 8));
      breg[nt][0] = a.x; breg[nt][1] = a.y; breg[nt][2] = b.x; breg[nt][3] = b.y;
    }
  }
  const float c = scale * LOG2E;
  const int frag_off = (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;

  for (; win < nwin_total; win += gridDim.y, stage ^= 1) {
    const int nxt = win + gridDim.y;
    if (nxt < nwin_total)
      issue7<false, 128, 2>(g, nxt, h, qkv, bchunk, nullptr, nullptr, nullptr, tiles + (stage ^ 1) * 2 * TILE7, nullptr,
                            tokb + (stage ^ 1) * 64, ridb + (stage ^ 1) * 64);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();  // this stage has landed, and the previous window's P block has been stored
    const bf16* Qs = tiles + stage * 2 * TILE7;
    const bf16* Ks = Qs + TILE7;
    const int* rid = ridb + stage * 64;

    uint32_t qa[2][4];
    ldsm_x4(qa[0], Qs + frag_off);
    ldsm_x4(qa[1], Qs + frag_off + 16);
    float acc[C::NT8][4];
    float m0 = -INFINITY, m1 = -INFINITY;
    int ridA = 0, ridB = 0;
    if (SHIFT) { ridA = rid[rA]; ridB = rid[rB]; }
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
      uint32_t kb[4];
      ldsm_x4(kb, Ks + (nt * 8 + (lane & 7)) * LD + (lane >> 3) * 8);
      mma16816(acc[nt], qa[0], kb[0], kb[1]);
      mma16816(acc[nt], qa[1], kb[2], kb[3]);
#pragma unroll
      for (int i = 0; i < 4; i++) acc[nt][i] = fmaf(acc[nt][i], c, breg[nt][i]);
      if (SHIFT) {
        const int2 rc = *reinterpret_cast<const int2*>(rid + nt * 8 + (lane & 3) * 2);
        if (ridA != rc.x) acc[nt][0] += -100.f * LOG2E;
        if (ridA != rc.y) acc[nt][1] += -100.f * LOG2E;
        if (ridB != rc.x) acc[nt][2] += -100.f * LOG2E;
        if (ridB != rc.y) acc[nt][3] += -100.f * LOG2E;
      }
      m0 = fmaxf(m0, fmaxf(acc[nt][0], acc[nt][1]));
      m1 = fmaxf(m1, fmaxf(acc[nt][2], acc[nt][3]));
    }
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      acc[nt][0] = ex2(acc[nt][0] - m0);
      acc[nt][1] = ex2(acc[nt][1] - m0);
      acc[nt][2] = ex2(acc[nt][2] - m1);
      acc[nt][3] = ex2(acc[nt][3] - m1);
      s0 += acc[nt][0] + acc[nt][1];
      s1 += acc[nt][2] + acc[nt][3];
    }
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float i0 = 1.f / s0, i1 = 1.f / s1;
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      const int col = nt * 8 + (lane & 3) * 2;
      if (col < NT) {
        if (rA < NT) Ps[rA * NT + col] = acc[nt][0] * i0;
        if (rB < NT) Ps[rB * NT + col] = acc[nt][2] * i1;
      }
      if (col + 1 < NT) {
        if (rA < NT) Ps[rA * NT + col + 1] = acc[nt][1] * i0;
        if (rB < NT) Ps[rB * NT + col + 1] = acc[nt][3] * i1;
      }
    }
    __syncthreads();  // P block complete; every warp is done with this stage's tiles
    float* dst = probs + ((long long)win * g.nH + h) * NP;
    for (int i = threadIdx.x; i < NP; i += 128) __stcs(dst + i, Ps[i]);
  }
  cp_async_wait<0>();
}

static size_t probs7_smem() { return (size_t)2 * 2 * TILE7 * 2 + (size_t)(49 * 49 + 3) * 4 + (size_t)4 * 64 * 4; }

// ------------------------------------------------------------------------------------------------
// ws = 14: one CTA = 7 warps, a warp owns image rows {w, w+7} of the window (the forward's slot layout: 16 shared-memory
// rows per image row, so an mma tile is one (query image row, key image row) pair).  A [14 x 196] row block is too large
// to keep as scores, so a warp makes three passes over the 14 key image rows: the row maxima, then P of its 8 upper
// query rows (rA), then of its 6 lower rows (rB).  Each of the last two writes unnormalised ex2(s - m) into the warp's
// [8][196] staging rows and sums them; the warp then stores the rows (contiguous in probs, 16-byte aligned) as float4,
// scaled by 1 / sum.
constexpr int PW14 = 8 * NT14;  // floats of one warp's staging rows

template <bool SHIFT>
__device__ __forceinline__ void scores14(float (&s)[2][4], const uint32_t (&qa)[2][4], const bf16* Ks, const float* btl,
                                         const int* rid, int yi, int yj, int lane, float c, float kpad, int ridA,
                                         int ridB) {
#pragma unroll
  for (int hf = 0; hf < 2; hf++) {
    s[hf][0] = s[hf][1] = s[hf][2] = s[hf][3] = 0.f;
    uint32_t kb[4];
    ldsm_x4(kb, Ks + (yj * 16 + hf * 8 + (lane & 7)) * LD + (lane >> 3) * 8);
    mma16816(s[hf], qa[0], kb[0], kb[1]);
    mma16816(s[hf], qa[1], kb[2], kb[3]);
  }
  const Bias6 b = load_bias_q(btl + (yi - yj + 13) * 32);
  s[0][0] = fmaf(s[0][0], c, b.v[0]);
  s[0][1] = fmaf(s[0][1], c, b.v[1]);
  s[0][2] = fmaf(s[0][2], c, b.v[2]);
  s[0][3] = fmaf(s[0][3], c, b.v[3]);
  s[1][0] = fmaf(s[1][0], c, b.v[4]) + kpad;
  s[1][1] = fmaf(s[1][1], c, b.v[5]) + kpad;
  s[1][2] = fmaf(s[1][2], c, b.v[0]) + kpad;
  s[1][3] = fmaf(s[1][3], c, b.v[1]) + kpad;
  if (SHIFT) {
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
      const int2 rc = *reinterpret_cast<const int2*>(rid + yj * 16 + hf * 8 + (lane & 3) * 2);
      if (ridA != rc.x) s[hf][0] += NEG_MASK2;
      if (ridA != rc.y) s[hf][1] += NEG_MASK2;
      if (ridB != rc.x) s[hf][2] += NEG_MASK2;
      if (ridB != rc.y) s[hf][3] += NEG_MASK2;
    }
  }
}

template <bool SHIFT>
__global__ void __launch_bounds__(T14, 2) window_attn_probs14_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bias_table,
    float* __restrict__ probs, Geo g, float scale, int nwin_total) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);  // [Q | K] x [224][LD]
  bf16* Ks = Qs + TILE14;
  float* pst = reinterpret_cast<float*>(Ks + TILE14);  // [7 warps][8][196] staging rows
  float* linv = pst + 7 * PW14;                        // [7 warps][8] 1 / row sum
  float* bt2 = linv + 7 * 8;                           // [27][32]
  int* tok = reinterpret_cast<int*>(bt2 + 27 * 32);    // [224]
  int* rid = tok + R14;                                // [224]

  const int h = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, cq = lane & 3;

  zero_pad_rows14<2>(Qs);
  for (int i = threadIdx.x; i < 14 * 2; i += T14) {
    const int row = (i >> 1) * 16 + 14 + (i & 1);
    tok[row] = -1;
    rid[row] = 0;
  }
  stage_bias14(bias_table, bt2, g.nH, h);
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));

  const float c = scale * LOG2E;
  const float kpad = (cq == 3) ? -INFINITY : 0.f;  // key columns 14, 15 of every image row
  const float* btl = bt2 + 15 + r - 2 * cq;
  float* pw = pst + warp * PW14;
  float* lw = linv + warp * 8;

  for (int win = blockIdx.y; win < nwin_total; win += gridDim.y) {
    __syncthreads();  // previous window's tiles consumed (and the one-time init above visible)
    issue14<2>(g, win, h, qkv, bchunk, Qs, tok, rid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

#pragma unroll 1
    for (int rd = 0; rd < 2; rd++) {
      const int yi = warp + 7 * rd;
      uint32_t qa[2][4];
      {
        const bf16* p = Qs + (yi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        ldsm_x4(qa[0], p);
        ldsm_x4(qa[1], p + 16);
      }
      int ridA = 0, ridB = 0;
      if (SHIFT) { ridA = rid[yi * 16 + r]; ridB = rid[yi * 16 + r + 8]; }
      float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll 2
      for (int yj = 0; yj < 14; yj++) {
        float s[2][4];
        scores14<SHIFT>(s, qa, Ks, btl, rid, yi, yj, lane, c, kpad, ridA, ridB);
        m0 = fmaxf(m0, fmaxf(fmaxf(s[0][0], s[0][1]), fmaxf(s[1][0], s[1][1])));
        m1 = fmaxf(m1, fmaxf(fmaxf(s[0][2], s[0][3]), fmaxf(s[1][2], s[1][3])));
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));

#pragma unroll 1
      for (int half = 0; half < 2; half++) {  // 0: query rows r (8 rows), 1: rows r + 8 (6 rows; 14, 15 are padding)
        const float m = half ? m1 : m0;
        const bool live = half == 0 || r < 6;
        float l = 0.f;
#pragma unroll 2
        for (int yj = 0; yj < 14; yj++) {
          float s[2][4];
          scores14<SHIFT>(s, qa, Ks, btl, rid, yi, yj, lane, c, kpad, ridA, ridB);
          const float p0 = ex2((half ? s[0][2] : s[0][0]) - m), p1 = ex2((half ? s[0][3] : s[0][1]) - m);
          const float p2 = ex2((half ? s[1][2] : s[1][0]) - m), p3 = ex2((half ? s[1][3] : s[1][1]) - m);  // 0: key padding
          l += (p0 + p1) + (p2 + p3);
          if (live) {
            float* row = pw + r * NT14 + yj * 14 + 2 * cq;
            *reinterpret_cast<float2*>(row) = make_float2(p0, p1);
            if (cq < 3) *reinterpret_cast<float2*>(row + 8) = make_float2(p2, p3);
          }
        }
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        if (cq == 0) lw[r] = 1.f / l;
        __syncwarp();
        const int nrows = half ? 6 : 8;
        const float4* src = reinterpret_cast<const float4*>(pw);
        float4* dst = reinterpret_cast<float4*>(probs + (((long long)win * g.nH + h) * NT14 + yi * 14 + half * 8) * NT14);
        for (int i = lane; i < nrows * (NT14 / 4); i += 32) {
          float4 v = src[i];
          const float sc = lw[i / (NT14 / 4)];
          v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
          __stcs(dst + i, v);
        }
        __syncwarp();  // staging rows free for the next half
      }
    }
  }
}

static size_t probs14_smem() {
  return (size_t)2 * TILE14 * 2 + (size_t)(7 * PW14 + 7 * 8 + 27 * 32) * 4 + (size_t)2 * R14 * 4;
}

}  // namespace wa
