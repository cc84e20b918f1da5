// ws = 14 fast path of the (shifted-)window attention core (Swin-S/B W14: 196 tokens per window).
//
// Slot layout: image row y of the window occupies 16 consecutive shared-memory rows (14 slots + 2 zero rows), so an
// mma tile (16 queries x 16 keys) is exactly ONE (query image row yi, key image row yj) pair.  That costs 224 instead
// of 208 padded slots (+16 % MMAs) and buys what the generic kernel spent most of its instructions on:
//   * the rel-pos bias of a tile pair is one row (dy = yi - yj) of the table and depends only on xi - xj, which is a
//     per-thread CONSTANT in the accumulator layout: six shared-memory loads at fixed offsets, no index arithmetic;
//   * the bias-table gradient of a tile pair goes to that one row as six per-thread partial sums at fixed (slot, lane)
//     addresses - reduced with fire-and-forget global REDs into a lane-expanded [nH][27][6][32] buffer that a tiny
//     kernel folds into the table (the generic kernel issued one shared-memory CAS loop per score element);
//   * no [N, N] score tile in registers: forward = online softmax over 64-key chunks, backward = two register-only
//     phases (queries as rows for dQ, keys as rows for dK/dV; P is recomputed from the saved log-sum-exp).
// One CTA = 7 warps; a warp owns image rows {w, w+7}.  Query rows whose 14 slots are all padding (local crops: 6x6
// tokens in a 14x14 window) are skipped - their outputs are cropped by the reference (:318-319) and their dO is 0.
//
// Reference: models/swin_transformer.py WindowAttention.forward :120-152, SwinTransformerBlock.forward :283-325.
#pragma once
#include "wa_common.cuh"

namespace wa {

constexpr int R14 = 224;           // 14 image rows x 16 slots
constexpr int TILE14 = R14 * LD;   // bf16 elements of one q / k / v / dO tile
constexpr int NT14 = 196;
constexpr int T14 = 224;           // threads per CTA
constexpr int GACC14 = 27 * 6 * 32;  // floats per head of the lane-expanded bias-gradient accumulator
constexpr float NEG_MASK2 = -100.f * LOG2E;

// stage the rel-pos bias of head h as bt2[dy + 13][dx + 15] (log2 domain; |dx| > 13 never reaches a live score)
__device__ __forceinline__ void stage_bias14(const float* __restrict__ bias_table, float* bt2, int nH, int h) {
  for (int i = threadIdx.x; i < 27 * 32; i += T14) {
    const int dyi = i >> 5, dx = (i & 31) - 15;
    bt2[i] = (dx >= -13 && dx <= 13) ? bias_table[(dyi * 27 + dx + 13) * nH + h] * LOG2E : 0.f;
  }
}

// zero rows (x = 14, 15 of every image row) of NTILES tiles; they are never written afterwards
template <int NTILES>
__device__ __forceinline__ void zero_pad_rows14(bf16* tiles) {
  for (int i = threadIdx.x; i < NTILES * 14 * 2 * 4; i += T14) {
    const int c16 = i & 3, ps = (i >> 2) & 1, y = (i >> 3) % 14, tt = (i >> 3) / 14;
    *reinterpret_cast<uint4*>(tiles + tt * TILE14 + (y * 16 + 14 + ps) * LD + c16 * 8) = make_uint4(0, 0, 0, 0);
  }
}

// async gather of the q/k/v rows of one window into [Q | K | V] tiles ([Q | K] for NPART = 2); padded slots get the
// bf16 qkv bias from registers (see window_attn7.cuh: a global read would hammer one cache line from thousands of CTAs)
template <int NPART = 3>
__device__ __forceinline__ void issue14(const Geo& g, int win, int h, const bf16* __restrict__ qkv,
                                        const uint4 (&bchunk)[3], bf16* tiles, int* tok, int* rid) {
  const int wx = win % g.nWx, wy = (win / g.nWx) % g.nWy, b = win / (g.nWx * g.nWy);
  const int c16 = threadIdx.x & 3;
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
    const int t = (threadIdx.x >> 2) + (T14 / 4) * kk;
    if (t < NT14) {
      int tk, r;
      slot_info<14>(g, b, wy, wx, t, tk, r);
      const int row = t + 2 * (t / 14);
      bf16* dst = tiles + row * LD + c16 * 8;
      if (tk < 0) {
#pragma unroll
        for (int part = 0; part < NPART; part++) *reinterpret_cast<uint4*>(dst + part * TILE14) = bchunk[part];
      } else {
        const bf16* src = qkv + (long long)tk * 3 * g.C + h * HD + c16 * 8;
#pragma unroll
        for (int part = 0; part < NPART; part++) cp_async16(dst + part * TILE14, src + part * g.C, 16);
      }
      if (c16 == 0) {
        tok[row] = tk;
        rid[row] = r;
      }
    }
  }
}

// rel-pos bias of one tile pair for this thread (br = bt2 + row(dy) + 15 + r - 2c)
//   QUERY-major (rows = queries): b[0..5] = dx of (rA,2c) (rA,2c+1) (rB,2c) (rB,2c+1) (rA,2c+8) (rA,2c+9)
struct Bias6 { float v[6]; };
__device__ __forceinline__ Bias6 load_bias_q(const float* br) {
  Bias6 b;
  b.v[0] = br[0]; b.v[1] = br[-1]; b.v[2] = br[8]; b.v[3] = br[7]; b.v[4] = br[-8]; b.v[5] = br[-9];
  return b;
}
//   KEY-major (rows = keys, br = bt2 + row(dy) + 15 + 2c - r): (kA,2c) (kA,2c+1) (kB,2c) (kB,2c+1) (kA,2c+8) (kA,2c+9)
__device__ __forceinline__ Bias6 load_bias_k(const float* br) {
  Bias6 b;
  b.v[0] = br[0]; b.v[1] = br[1]; b.v[2] = br[-8]; b.v[3] = br[-7]; b.v[4] = br[8]; b.v[5] = br[9];
  return b;
}

// ------------------------------------------------------------------------------------------------
template <bool SHIFT>
__global__ void __launch_bounds__(T14, 2) window_attn_fwd14_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bias_table,
    bf16* __restrict__ out, float* __restrict__ lse, Geo g, float scale, int nwin_total) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* tiles = reinterpret_cast<bf16*>(smraw);                // [2 stages][Q | K | V]
  float* bt2 = reinterpret_cast<float*>(tiles + 2 * 3 * TILE14);  // [27][32]
  int* tokb = reinterpret_cast<int*>(bt2 + 27 * 32);            // [2][224]
  int* ridb = tokb + 2 * R14;                                  // [2][224]

  const int h = blockIdx.x;  // heads fastest (see window_attn7.cuh)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, cq = lane & 3;
  int win = blockIdx.y, stage = 0;

  zero_pad_rows14<6>(tiles);
  for (int i = threadIdx.x; i < 2 * 14 * 2; i += T14) {
    const int row = (i >> 2) * 16 + 14 + (i & 1) + ((i >> 1) & 1) * R14;  // both stages
    if ((i >> 2) < 14) { tokb[row] = -1; ridb[row] = 0; }
  }
  stage_bias14(bias_table, bt2, g.nH, h);
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));
  if (win < nwin_total) issue14(g, win, h, qkv, bchunk, tiles, tokb, ridb);
  cp_async_commit();

  const float c = scale * LOG2E;
  const float kpad = (cq == 3) ? -INFINITY : 0.f;  // key columns 14, 15 of every image row (accumulator n-tile 1)
  const float* btl = bt2 + 15 + r - 2 * cq;

  for (; win < nwin_total; win += gridDim.y, stage ^= 1) {
    const int nxt = win + gridDim.y;
    if (nxt < nwin_total)
      issue14(g, nxt, h, qkv, bchunk, tiles + (stage ^ 1) * 3 * TILE14, tokb + (stage ^ 1) * R14, ridb + (stage ^ 1) * R14);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Qs = tiles + stage * 3 * TILE14;
    const bf16* Ks = Qs + TILE14;
    const bf16* Vs = Ks + TILE14;
    const int* tok = tokb + stage * R14;
    const int* rid = ridb + stage * R14;

#pragma unroll 1
    for (int rd = 0; rd < 2; rd++) {
      const int yi = warp + 7 * rd;
      const int rowA = yi * 16 + r, rowB = rowA + 8;
      const int tA = tok[rowA], tB = tok[rowB];
      float* lrow = lse + ((long long)win * g.nH + h) * NT14 + yi * 14;
      if (!__any_sync(0xffffffffu, tA >= 0 || tB >= 0)) {  // all-padding query row: outputs are cropped away
        if (cq == 0) {
          lrow[r] = 0.f;
          if (r < 6) lrow[r + 8] = 0.f;
        }
        continue;
      }
      uint32_t qa[2][4];
      {
        const bf16* p = Qs + (yi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        ldsm_x4(qa[0], p);
        ldsm_x4(qa[1], p + 16);
      }
      int ridA = 0, ridB = 0;
      if (SHIFT) { ridA = rid[rowA]; ridB = rid[rowB]; }
      float o[4][4];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

#pragma unroll
      for (int ch = 0; ch < 4; ch++) {
        float s[4][2][4];
        float cm0 = -INFINITY, cm1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int yj = 4 * ch + j;
          if (yj < 14) {
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
              s[j][hf][0] = s[j][hf][1] = s[j][hf][2] = s[j][hf][3] = 0.f;
              uint32_t kb[4];
              ldsm_x4(kb, Ks + (yj * 16 + hf * 8 + (lane & 7)) * LD + (lane >> 3) * 8);
              mma16816(s[j][hf], qa[0], kb[0], kb[1]);
              mma16816(s[j][hf], qa[1], kb[2], kb[3]);
            }
            const Bias6 b = load_bias_q(btl + (yi - yj + 13) * 32);
            s[j][0][0] = fmaf(s[j][0][0], c, b.v[0]);
            s[j][0][1] = fmaf(s[j][0][1], c, b.v[1]);
            s[j][0][2] = fmaf(s[j][0][2], c, b.v[2]);
            s[j][0][3] = fmaf(s[j][0][3], c, b.v[3]);
            s[j][1][0] = fmaf(s[j][1][0], c, b.v[4]) + kpad;
            s[j][1][1] = fmaf(s[j][1][1], c, b.v[5]) + kpad;
            s[j][1][2] = fmaf(s[j][1][2], c, b.v[0]) + kpad;
            s[j][1][3] = fmaf(s[j][1][3], c, b.v[1]) + kpad;
            if (SHIFT) {
#pragma unroll
              for (int hf = 0; hf < 2; hf++) {
                const int2 rc = *reinterpret_cast<const int2*>(rid + yj * 16 + hf * 8 + cq * 2);
                if (ridA != rc.x) s[j][hf][0] += NEG_MASK2;
                if (ridA != rc.y) s[j][hf][1] += NEG_MASK2;
                if (ridB != rc.x) s[j][hf][2] += NEG_MASK2;
                if (ridB != rc.y) s[j][hf][3] += NEG_MASK2;
              }
            }
            cm0 = fmaxf(cm0, fmaxf(fmaxf(s[j][0][0], s[j][0][1]), fmaxf(s[j][1][0], s[j][1][1])));
            cm1 = fmaxf(cm1, fmaxf(fmaxf(s[j][0][2], s[j][0][3]), fmaxf(s[j][1][2], s[j][1][3])));
          }
        }
        cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 1));
        cm0 = fmaxf(cm0, __shfl_xor_sync(0xffffffffu, cm0, 2));
        cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 1));
        cm1 = fmaxf(cm1, __shfl_xor_sync(0xffffffffu, cm1, 2));
        const float mn0 = fmaxf(m0, cm0), mn1 = fmaxf(m1, cm1);  // finite: every chunk has 14 live keys per row
        const float a0 = ex2(m0 - mn0), a1 = ex2(m1 - mn1);
        m0 = mn0;
        m1 = mn1;
        l0 *= a0;
        l1 *= a1;
#pragma unroll
        for (int dt = 0; dt < 4; dt++) {
          o[dt][0] *= a0; o[dt][1] *= a0; o[dt][2] *= a1; o[dt][3] *= a1;
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int yj = 4 * ch + j;
          if (yj < 14) {
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
              s[j][hf][0] = ex2(s[j][hf][0] - m0);
              s[j][hf][1] = ex2(s[j][hf][1] - m0);
              s[j][hf][2] = ex2(s[j][hf][2] - m1);
              s[j][hf][3] = ex2(s[j][hf][3] - m1);
              l0 += s[j][hf][0] + s[j][hf][1];
              l1 += s[j][hf][2] + s[j][hf][3];
            }
            uint32_t pa[4];
            pa[0] = pack_bf162(s[j][0][0], s[j][0][1]);
            pa[1] = pack_bf162(s[j][0][2], s[j][0][3]);
            pa[2] = pack_bf162(s[j][1][0], s[j][1][1]);
            pa[3] = pack_bf162(s[j][1][2], s[j][1][3]);
            const bf16* vp = Vs + (yj * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
            uint32_t vb[4];
            ldsm_x4_t(vb, vp);
            mma16816(o[0], pa, vb[0], vb[1]);
            mma16816(o[1], pa, vb[2], vb[3]);
            ldsm_x4_t(vb, vp + 16);
            mma16816(o[2], pa, vb[0], vb[1]);
            mma16816(o[3], pa, vb[2], vb[3]);
          }
        }
      }
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float i0 = __fdividef(1.f, l0), i1 = __fdividef(1.f, l1);
      if (cq == 0) {  // natural-log LSE for the backward
        lrow[r] = (m0 + lg2(l0)) * LN2;
        if (r < 6) lrow[r + 8] = (m1 + lg2(l1)) * LN2;
      }
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        const int d = h * HD + dt * 8 + cq * 2;
        if (tA >= 0) *reinterpret_cast<uint32_t*>(out + (long long)tA * g.C + d) = pack_bf162(o[dt][0] * i0, o[dt][1] * i0);
        if (tB >= 0) *reinterpret_cast<uint32_t*>(out + (long long)tB * g.C + d) = pack_bf162(o[dt][2] * i1, o[dt][3] * i1);
      }
    }
    __syncthreads();  // everyone is done with this stage before the next-but-one gather overwrites it
  }
  cp_async_wait<0>();
}

static size_t fwd14_smem() { return (size_t)2 * 3 * TILE14 * 2 + (size_t)27 * 32 * 4 + (size_t)4 * R14 * 4; }

// ------------------------------------------------------------------------------------------------
// backward.  gacc: this call's lane-expanded bias-gradient accumulator [nH][27][6][32] (zeroed by the caller).
template <bool SHIFT>
__global__ void __launch_bounds__(T14, 2) window_attn_bwd14_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bias_table,
    const bf16* __restrict__ out, const bf16* __restrict__ dout, const float* __restrict__ lse,
    bf16* __restrict__ dqkv, float* __restrict__ gacc, float* __restrict__ dqkv_bias, Geo g, float scale,
    int nwin_total) {
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* Qs = reinterpret_cast<bf16*>(smraw);  // [Q | K | V | dO] x [224][LD]
  bf16* Ks = Qs + TILE14;
  bf16* Vs = Ks + TILE14;
  bf16* dOs = Vs + TILE14;
  float* bt2 = reinterpret_cast<float*>(dOs + TILE14);  // [27][32]
  float* Dsm = bt2 + 27 * 32;                           // [224] rowsum(dO * O)
  float* Lsm = Dsm + R14;                               // [224] lse * log2e
  float* dqb = Lsm + R14;                               // [3][32] qkv-bias grads of this head
  int* tok = reinterpret_cast<int*>(dqb + 3 * HD);      // [224]
  int* rid = tok + R14;                                 // [224]

  const int h = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane >> 2, cq = lane & 3;

  zero_pad_rows14<4>(Qs);
  for (int i = threadIdx.x; i < 14 * 2; i += T14) {
    const int row = (i >> 1) * 16 + 14 + (i & 1);
    tok[row] = -1;
    rid[row] = 0;
    Dsm[row] = 0.f;
    Lsm[row] = 0.f;
  }
  for (int i = threadIdx.x; i < 3 * HD; i += T14) dqb[i] = 0.f;
  stage_bias14(bias_table, bt2, g.nH, h);
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));

  const float c = scale * LOG2E;
  const float kpad = (cq == 3) ? -INFINITY : 0.f;   // phase A: key columns 14, 15 (n-tile 1)
  const float kpadB = (r >= 6) ? -INFINITY : 0.f;   // phase B: key rows 14, 15 (rows r + 8)
  const float* btq = bt2 + 15 + r - 2 * cq;         // query-major per-thread diagonal
  const float* btk = bt2 + 15 + 2 * cq - r;         // key-major
  float* gh = gacc + (long long)h * GACC14 + lane;

  for (int win = blockIdx.y; win < nwin_total; win += gridDim.y) {
    __syncthreads();  // previous window fully consumed (and the one-time init above visible)
    {
      const int wx = win % g.nWx, wy = (win / g.nWx) % g.nWy, b = win / (g.nWx * g.nWy);
      const int c16 = threadIdx.x & 3;
      uint4 dv[4], ov[4];
      int rows[4];
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        const int t = (threadIdx.x >> 2) + (T14 / 4) * kk;
        dv[kk] = make_uint4(0, 0, 0, 0);
        ov[kk] = make_uint4(0, 0, 0, 0);
        rows[kk] = -1;
        if (t < NT14) {
          int tk, rr;
          slot_info<14>(g, b, wy, wx, t, tk, rr);
          const int row = t + 2 * (t / 14);
          rows[kk] = row;
          bf16* dst = Qs + row * LD + c16 * 8;
          if (tk < 0) {
#pragma unroll
            for (int part = 0; part < 3; part++) *reinterpret_cast<uint4*>(dst + part * TILE14) = bchunk[part];
          } else {
            const bf16* src = qkv + (long long)tk * 3 * g.C + h * HD + c16 * 8;
#pragma unroll
            for (int part = 0; part < 3; part++) cp_async16(dst + part * TILE14, src + part * g.C, 16);
            const long long off = (long long)tk * g.C + h * HD + c16 * 8;
            dv[kk] = __ldg(reinterpret_cast<const uint4*>(dout + off));
            ov[kk] = __ldg(reinterpret_cast<const uint4*>(out + off));
          }
          if (c16 == 0) {
            tok[row] = tk;
            rid[row] = rr;
            Lsm[row] = lse[((long long)win * g.nH + h) * NT14 + t] * LOG2E;
          }
        }
      }
      cp_async_commit();
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        float fd[8], fo[8], part = 0.f;
        unpack8(*reinterpret_cast<const bf16x8*>(&dv[kk]), fd);
        unpack8(*reinterpret_cast<const bf16x8*>(&ov[kk]), fo);
#pragma unroll
        for (int j = 0; j < 8; j++) part += fd[j] * fo[j];
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        if (rows[kk] >= 0) {
          *reinterpret_cast<uint4*>(dOs + rows[kk] * LD + c16 * 8) = dv[kk];
          if (c16 == 0) Dsm[rows[kk]] = part;
        }
      }
      cp_async_wait<0>();
    }
    __syncthreads();

    // image rows that hold a real token (bit y).  An all-padding QUERY row has dO = 0, so dS = 0 there: it adds nothing
    // to dQ / dK / dV / the bias gradients and both phases skip it (padded KEY rows stay: their dK / dV are part of
    // the qkv-bias gradient).
    unsigned qvalid = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) {
      const unsigned bal = __ballot_sync(0xffffffffu, tok[k * 32 + lane] >= 0);
      qvalid |= ((bal & 0xffffu) ? 1u : 0u) << (2 * k);
      qvalid |= ((bal >> 16) ? 1u : 0u) << (2 * k + 1);
    }

    // ---------------- phase A: rows = queries of image row yi ----------------
#pragma unroll 1
    for (int rd = 0; rd < 2; rd++) {
      const int yi = warp + 7 * rd;
      if (!((qvalid >> yi) & 1u)) continue;
      const int rowA = yi * 16 + r, rowB = rowA + 8;
      uint32_t qa[2][4], da[2][4];
      {
        const int off = (yi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        ldsm_x4(qa[0], Qs + off);
        ldsm_x4(qa[1], Qs + off + 16);
        ldsm_x4(da[0], dOs + off);
        ldsm_x4(da[1], dOs + off + 16);
      }
      const float lA = Lsm[rowA], lB = Lsm[rowB], DA = Dsm[rowA], DB = Dsm[rowB];
      int ridA = 0, ridB = 0;
      if (SHIFT) { ridA = rid[rowA]; ridB = rid[rowB]; }
      float dq[4][4];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) dq[dt][0] = dq[dt][1] = dq[dt][2] = dq[dt][3] = 0.f;
#pragma unroll 2
      for (int yj = 0; yj < 14; yj++) {
        float sv[2][4], ds[2][4];
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          sv[hf][0] = sv[hf][1] = sv[hf][2] = sv[hf][3] = 0.f;
          ds[hf][0] = ds[hf][1] = ds[hf][2] = ds[hf][3] = 0.f;
          const int boff = (yj * 16 + hf * 8 + (lane & 7)) * LD + (lane >> 3) * 8;
          uint32_t kb[4];
          ldsm_x4(kb, Ks + boff);
          mma16816(sv[hf], qa[0], kb[0], kb[1]);
          mma16816(sv[hf], qa[1], kb[2], kb[3]);
          ldsm_x4(kb, Vs + boff);
          mma16816(ds[hf], da[0], kb[0], kb[1]);
          mma16816(ds[hf], da[1], kb[2], kb[3]);
        }
        const Bias6 b = load_bias_q(btq + (yi - yj + 13) * 32);
        sv[0][0] = fmaf(sv[0][0], c, b.v[0]) - lA;
        sv[0][1] = fmaf(sv[0][1], c, b.v[1]) - lA;
        sv[0][2] = fmaf(sv[0][2], c, b.v[2]) - lB;
        sv[0][3] = fmaf(sv[0][3], c, b.v[3]) - lB;
        sv[1][0] = fmaf(sv[1][0], c, b.v[4]) - lA + kpad;
        sv[1][1] = fmaf(sv[1][1], c, b.v[5]) - lA + kpad;
        sv[1][2] = fmaf(sv[1][2], c, b.v[0]) - lB + kpad;
        sv[1][3] = fmaf(sv[1][3], c, b.v[1]) - lB + kpad;
        if (SHIFT) {
#pragma unroll
          for (int hf = 0; hf < 2; hf++) {
            const int2 rc = *reinterpret_cast<const int2*>(rid + yj * 16 + hf * 8 + cq * 2);
            if (ridA != rc.x) sv[hf][0] += NEG_MASK2;
            if (ridA != rc.y) sv[hf][1] += NEG_MASK2;
            if (ridB != rc.x) sv[hf][2] += NEG_MASK2;
            if (ridB != rc.y) sv[hf][3] += NEG_MASK2;
          }
        }
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          ds[hf][0] = ex2(sv[hf][0]) * (ds[hf][0] - DA);
          ds[hf][1] = ex2(sv[hf][1]) * (ds[hf][1] - DA);
          ds[hf][2] = ex2(sv[hf][2]) * (ds[hf][2] - DB);
          ds[hf][3] = ex2(sv[hf][3]) * (ds[hf][3] - DB);
        }
        // rel-pos-bias gradient of this tile pair: row dy of the table, six per-thread diagonals (see the header).
        // dS was formed with the true probabilities, so it is the gradient w.r.t. the natural-domain table entry.
        {
          float* gp = gh + (yi - yj + 13) * 192;
          atomicAdd(gp, ds[0][0] + ds[1][2]);        // dx = r - 2c
          atomicAdd(gp + 32, ds[0][1] + ds[1][3]);   // dx = r - 2c - 1
          atomicAdd(gp + 64, ds[0][2]);              // dx = r - 2c + 8
          atomicAdd(gp + 96, ds[0][3]);              // dx = r - 2c + 7
          atomicAdd(gp + 128, ds[1][0]);             // dx = r - 2c - 8
          atomicAdd(gp + 160, ds[1][1]);             // dx = r - 2c - 9
        }
        uint32_t sa[4];
        sa[0] = pack_bf162(ds[0][0], ds[0][1]);
        sa[1] = pack_bf162(ds[0][2], ds[0][3]);
        sa[2] = pack_bf162(ds[1][0], ds[1][1]);
        sa[3] = pack_bf162(ds[1][2], ds[1][3]);
        const bf16* kp = Ks + (yj * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        uint32_t kb[4];
        ldsm_x4_t(kb, kp);
        mma16816(dq[0], sa, kb[0], kb[1]);
        mma16816(dq[1], sa, kb[2], kb[3]);
        ldsm_x4_t(kb, kp + 16);
        mma16816(dq[2], sa, kb[0], kb[1]);
        mma16816(dq[3], sa, kb[2], kb[3]);
      }
      const int tA = tok[rowA], tB = tok[rowB];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        const int d = h * HD + dt * 8 + cq * 2;
        if (tA >= 0)
          *reinterpret_cast<uint32_t*>(dqkv + (long long)tA * 3 * g.C + d) = pack_bf162(dq[dt][0] * scale, dq[dt][1] * scale);
        if (tB >= 0)
          *reinterpret_cast<uint32_t*>(dqkv + (long long)tB * 3 * g.C + d) = pack_bf162(dq[dt][2] * scale, dq[dt][3] * scale);
      }
      colsum_to_smem(dq, scale, dqb, lane);
    }

    // ---------------- phase B: rows = keys of image row yj (transposed recompute) ----------------
#pragma unroll 1
    for (int rd = 0; rd < 2; rd++) {
      const int yj = warp + 7 * rd;
      const int rowA = yj * 16 + r, rowB = rowA + 8;
      uint32_t ka[2][4], va[2][4];
      {
        const int off = (yj * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        ldsm_x4(ka[0], Ks + off);
        ldsm_x4(ka[1], Ks + off + 16);
        ldsm_x4(va[0], Vs + off);
        ldsm_x4(va[1], Vs + off + 16);
      }
      int ridA = 0, ridB = 0;
      if (SHIFT) { ridA = rid[rowA]; ridB = rid[rowB]; }
      float dv[4][4], dk[4][4];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        dv[dt][0] = dv[dt][1] = dv[dt][2] = dv[dt][3] = 0.f;
        dk[dt][0] = dk[dt][1] = dk[dt][2] = dk[dt][3] = 0.f;
      }
#pragma unroll 2
      for (int qi = 0; qi < 14; qi++) {
        if (!((qvalid >> qi) & 1u)) continue;
        float pT[2][4], dsT[2][4];
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          pT[hf][0] = pT[hf][1] = pT[hf][2] = pT[hf][3] = 0.f;
          dsT[hf][0] = dsT[hf][1] = dsT[hf][2] = dsT[hf][3] = 0.f;
          const int boff = (qi * 16 + hf * 8 + (lane & 7)) * LD + (lane >> 3) * 8;
          uint32_t qb[4];
          ldsm_x4(qb, Qs + boff);
          mma16816(pT[hf], ka[0], qb[0], qb[1]);
          mma16816(pT[hf], ka[1], qb[2], qb[3]);
          ldsm_x4(qb, dOs + boff);
          mma16816(dsT[hf], va[0], qb[0], qb[1]);
          mma16816(dsT[hf], va[1], qb[2], qb[3]);
        }
        const Bias6 b = load_bias_k(btk + (qi - yj + 13) * 32);
        const int q0 = qi * 16 + cq * 2;  // this thread's query columns: q0, q0+1, q0+8, q0+9
        const float2 l0 = *reinterpret_cast<const float2*>(Lsm + q0), l1 = *reinterpret_cast<const float2*>(Lsm + q0 + 8);
        const float2 D0 = *reinterpret_cast<const float2*>(Dsm + q0), D1 = *reinterpret_cast<const float2*>(Dsm + q0 + 8);
        float sv[2][4];
        sv[0][0] = fmaf(pT[0][0], c, b.v[0]) - l0.x;
        sv[0][1] = fmaf(pT[0][1], c, b.v[1]) - l0.y;
        sv[0][2] = fmaf(pT[0][2], c, b.v[2]) - l0.x + kpadB;
        sv[0][3] = fmaf(pT[0][3], c, b.v[3]) - l0.y + kpadB;
        sv[1][0] = fmaf(pT[1][0], c, b.v[4]) - l1.x;
        sv[1][1] = fmaf(pT[1][1], c, b.v[5]) - l1.y;
        sv[1][2] = fmaf(pT[1][2], c, b.v[0]) - l1.x + kpadB;
        sv[1][3] = fmaf(pT[1][3], c, b.v[1]) - l1.y + kpadB;
        if (SHIFT) {
#pragma unroll
          for (int hf = 0; hf < 2; hf++) {
            const int2 rq = *reinterpret_cast<const int2*>(rid + q0 + hf * 8);
            if (ridA != rq.x) sv[hf][0] += NEG_MASK2;
            if (ridA != rq.y) sv[hf][1] += NEG_MASK2;
            if (ridB != rq.x) sv[hf][2] += NEG_MASK2;
            if (ridB != rq.y) sv[hf][3] += NEG_MASK2;
          }
        }
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          const float2 Dq = hf ? D1 : D0;
          pT[hf][0] = ex2(sv[hf][0]);
          pT[hf][1] = ex2(sv[hf][1]);
          pT[hf][2] = ex2(sv[hf][2]);
          pT[hf][3] = ex2(sv[hf][3]);
          dsT[hf][0] = pT[hf][0] * (dsT[hf][0] - Dq.x);
          dsT[hf][1] = pT[hf][1] * (dsT[hf][1] - Dq.y);
          dsT[hf][2] = pT[hf][2] * (dsT[hf][2] - Dq.x);
          dsT[hf][3] = pT[hf][3] * (dsT[hf][3] - Dq.y);
        }
        uint32_t pa[4], sa[4];
        pa[0] = pack_bf162(pT[0][0], pT[0][1]);
        pa[1] = pack_bf162(pT[0][2], pT[0][3]);
        pa[2] = pack_bf162(pT[1][0], pT[1][1]);
        pa[3] = pack_bf162(pT[1][2], pT[1][3]);
        sa[0] = pack_bf162(dsT[0][0], dsT[0][1]);
        sa[1] = pack_bf162(dsT[0][2], dsT[0][3]);
        sa[2] = pack_bf162(dsT[1][0], dsT[1][1]);
        sa[3] = pack_bf162(dsT[1][2], dsT[1][3]);
        const int toff = (qi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        uint32_t bb[4];
        ldsm_x4_t(bb, dOs + toff);
        mma16816(dv[0], pa, bb[0], bb[1]);
        mma16816(dv[1], pa, bb[2], bb[3]);
        ldsm_x4_t(bb, dOs + toff + 16);
        mma16816(dv[2], pa, bb[0], bb[1]);
        mma16816(dv[3], pa, bb[2], bb[3]);
        ldsm_x4_t(bb, Qs + toff);
        mma16816(dk[0], sa, bb[0], bb[1]);
        mma16816(dk[1], sa, bb[2], bb[3]);
        ldsm_x4_t(bb, Qs + toff + 16);
        mma16816(dk[2], sa, bb[0], bb[1]);
        mma16816(dk[3], sa, bb[2], bb[3]);
      }
      const int tA = tok[rowA], tB = tok[rowB];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        const int d = h * HD + dt * 8 + cq * 2;
        if (tA >= 0) {
          bf16* base = dqkv + (long long)tA * 3 * g.C + d;
          *reinterpret_cast<uint32_t*>(base + g.C) = pack_bf162(dk[dt][0] * scale, dk[dt][1] * scale);
          *reinterpret_cast<uint32_t*>(base + 2 * g.C) = pack_bf162(dv[dt][0], dv[dt][1]);
        }
        if (tB >= 0) {
          bf16* base = dqkv + (long long)tB * 3 * g.C + d;
          *reinterpret_cast<uint32_t*>(base + g.C) = pack_bf162(dk[dt][2] * scale, dk[dt][3] * scale);
          *reinterpret_cast<uint32_t*>(base + 2 * g.C) = pack_bf162(dv[dt][2], dv[dt][3]);
        }
      }
      colsum_to_smem(dk, scale, dqb + HD, lane);
      colsum_to_smem(dv, 1.f, dqb + 2 * HD, lane);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * HD; i += T14)
    atomicAdd(&dqkv_bias[(i / HD) * g.C + h * HD + (i % HD)], dqb[i]);
}

static size_t bwd14_smem() {
  return (size_t)4 * TILE14 * 2 + (size_t)(27 * 32 + 2 * R14 + 3 * HD) * 4 + (size_t)2 * R14 * 4;
}

// fold the lane-expanded accumulator into dbias_table [(27*27), nH] (+=).  One block per (dy row, head).
__global__ void __launch_bounds__(192) fold_dbias14_kernel(const float* __restrict__ gacc, float* __restrict__ dbias_table,
                                                           int nH) {
  __shared__ float bins[32];
  const int dyi = blockIdx.x, h = blockIdx.y;
  if (threadIdx.x < 32) bins[threadIdx.x] = 0.f;
  __syncthreads();
  const int slot = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int base = (lane >> 2) - 2 * (lane & 3);
  const int off = slot == 0 ? 0 : slot == 1 ? -1 : slot == 2 ? 8 : slot == 3 ? 7 : slot == 4 ? -8 : -9;
  const int dx = base + off;
  const float v = gacc[((long long)h * 27 + dyi) * 192 + threadIdx.x];
  if (dx >= -13 && dx <= 13) atomicAdd(&bins[dx + 13], v);
  __syncthreads();
  if (threadIdx.x < 27) dbias_table[(dyi * 27 + threadIdx.x) * nH + h] += bins[threadIdx.x];
}

}  // namespace wa
