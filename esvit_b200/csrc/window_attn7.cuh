// ws = 7 fast path of the (shifted-)window attention core (KP = 64 slots; every Swin W=7 stage, both crop sizes).
//
// One CTA = 4 warps = one (window, head) at a time, PERSISTENT over windows, with a 2-stage cp.async pipeline:
// the q/k/v (and dO / O) rows of window i+1 are gathered into the other shared-memory stage while window i is
// computed, so the DRAM latency of the gather (the first versions' bottleneck: ~6 us per window exposed) is hidden.
// Padded slots copy the bf16 qkv bias instead of a token row; slots >= 49 are zero-filled by the copy engine.
//
// Instruction diet (the first version issued ~40 instructions per score element):
//   * scores live in the log2 domain: s' = acc*(scale*log2e) + bias*log2e (one FMA), P = ex2(s' - m');
//   * the rel-pos bias of this head is expanded ONCE per persistent CTA - forward: straight into the accumulator
//     fragment layout in registers; backward: into a [64][72] fp32 shared-memory table - with -inf in the padded
//     rows/columns, which also replaces every bounds check;
//   * the shift mask is a template flag, so un-shifted blocks carry no mask code.
#pragma once
#include "wa_common.cuh"

namespace wa {

constexpr int BLD = 72;        // row stride (floats) of the expanded bias table: 72 % 32 == 8 -> conflict-free float2 reads
constexpr int TILE7 = 64 * LD;  // bf16 elements of one 64-row tile

// Rel-pos bias of every head expanded ONCE per call to a dense [nH][64][64] fp32 table in the log2 domain with -inf in
// the padded rows/columns (it doubles as the key-padding mask).  The first versions expanded it in every CTA's
// prologue: ~3700 instructions per warp of index arithmetic, more than the whole attention loop of a late stage.
__global__ void __launch_bounds__(256) expand_bias7_kernel(const float* __restrict__ bias_table, float* __restrict__ bexp,
                                                           int nH) {
  const int h = blockIdx.x;
  for (int i = threadIdx.x; i < 64 * 64; i += blockDim.x) {
    const int row = i >> 6, col = i & 63;
    float v = -INFINITY;
    if (col < 49) v = row < 49 ? bias_table[bias_index<7>(row, col) * nH + h] * LOG2E : 0.f;
    bexp[(long long)h * 4096 + i] = v;
  }
}

// Issue the async gathers of one window into a pipeline stage: tiles [Q | K | V] (+ [dO | O] and lse for BWD).
// Padded slots hold the qkv bias of this head: every thread keeps ITS three 16-byte bias chunks (q,k,v at its c16) in
// registers and stores them to shared memory directly - gathering them from global memory made thousands of CTAs hammer
// the same few cache lines (local crops: 5x slower gathers than global crops with the same window count).
template <bool BWD, int NTHREADS = 128>
__device__ __forceinline__ void issue7(const Geo& g, int win, int h, const bf16* __restrict__ qkv,
                                       const uint4 (&bchunk)[3], const bf16* __restrict__ dout,
                                       const bf16* __restrict__ out, const float* __restrict__ lse, bf16* tiles,
                                       float* Lraw, int* tok, int* rid) {
  constexpr int WS = 7, NT = 49;
  const int wx = win % g.nWx, wy = (win / g.nWx) % g.nWy, b = win / (g.nWx * g.nWy);
  // 4 adjacent lanes cover one 64-byte (slot, q|k|v) segment (coalesced like a row copy); a thread serves the SAME
  // two slots for all of q, k, v (+ dO, O), so the slot geometry is computed twice per thread per window, not 6-10x.
  const int c16 = threadIdx.x & 3;
#pragma unroll
  for (int kk = 0; kk < 256 / NTHREADS; kk++) {
    const int t = (threadIdx.x >> 2) + (NTHREADS / 4) * kk;
    int tk = -1, r = 0;
    if (t < NT) slot_info<WS>(g, b, wy, wx, t, tk, r);
    const bf16* src_row = qkv + (long long)(tk >= 0 ? tk : 0) * 3 * g.C + h * HD + c16 * 8;
    const int nbytes = (t < NT && g.dbg != 1) ? 16 : 0;  // slots >= 49: zero fill (dbg 1: no global reads at all)
    if (t < NT && tk < 0) {
#pragma unroll
      for (int part = 0; part < 3; part++)
        *reinterpret_cast<uint4*>(tiles + part * TILE7 + t * LD + c16 * 8) = bchunk[part];
    } else {
#pragma unroll
      for (int part = 0; part < 3; part++)
        cp_async16(tiles + part * TILE7 + t * LD + c16 * 8, src_row + part * g.C, nbytes);
    }
    if (BWD) {
      const long long off = (long long)(tk >= 0 ? tk : 0) * g.C + h * HD + c16 * 8;
      const int nb = (tk >= 0 && g.dbg != 1) ? 16 : 0;  // padded slots: their output is cropped -> dO = O = 0
      cp_async16(tiles + 3 * TILE7 + t * LD + c16 * 8, dout + off, nb);
      cp_async16(tiles + 4 * TILE7 + t * LD + c16 * 8, out + off, nb);
    }
    if (c16 == 0) {
      tok[t] = tk;
      rid[t] = r;
      if (BWD) cp_async4(Lraw + t, lse + ((long long)win * g.nH + h) * NT + (t < NT ? t : 0), t < NT ? 4 : 0);
    }
  }
}

// ------------------------------------------------------------------------------------------------
template <bool SHIFT>
__global__ void __launch_bounds__(128, 4) window_attn_fwd7_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bexp,
    bf16* __restrict__ out, float* __restrict__ lse, Geo g, float scale, int nwin_total) {
  constexpr int WS = 7;
  using C = Cfg<WS>;
  static_assert(C::KP == 64 && C::NW == 4, "fast path assumes a 64-slot window and 4 warps");
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* tiles = reinterpret_cast<bf16*>(smraw);                  // [2 stages][Q | K | V]
  int* tokb = reinterpret_cast<int*>(tiles + 2 * 3 * TILE7);      // [2][64]
  int* ridb = tokb + 2 * 64;                                     // [2][64]

  const int h = blockIdx.x;  // heads fastest: the nH CTAs sharing a window's token rows run together (DRAM page locality)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = warp * 16, rA = r0 + (lane >> 2), rB = rA + 8;
  int win = blockIdx.y, stage = 0;
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));
  if (win < nwin_total) issue7<false>(g, win, h, qkv, bchunk, nullptr, nullptr, nullptr, tiles, nullptr, tokb, ridb);
  cp_async_commit();

  // rel-pos bias of (head h, this warp's 16 query rows) in accumulator-fragment layout, from the expanded table
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
      issue7<false>(g, nxt, h, qkv, bchunk, nullptr, nullptr, nullptr, tiles + (stage ^ 1) * 3 * TILE7, nullptr,
                    tokb + (stage ^ 1) * 64, ridb + (stage ^ 1) * 64);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Qs = tiles + stage * 3 * TILE7;
    const bf16* Ks = Qs + TILE7;
    const bf16* Vs = Ks + TILE7;
    const int* tok = tokb + stage * 64;
    const int* rid = ridb + stage * 64;
    if (g.dbg == 2) { __syncthreads(); continue; }
    const int tA = rA < C::NT ? tok[rA] : -1, tB = rB < C::NT ? tok[rB] : -1;
    // a query tile whose 16 slots are all padding (local crops: the window rows below the map) produces only rows
    // the reference crops away (:318-319) - skip its math; the warp's issue slots go to the co-resident CTAs
    if (!__any_sync(0xffffffffu, tA >= 0 || tB >= 0)) {
      if ((lane & 3) == 0) {  // keep the saved statistics defined (the backward skips the same tiles)
        float* l = lse + ((long long)win * g.nH + h) * C::NT;
        if (rA < C::NT) l[rA] = 0.f;
        if (rB < C::NT) l[rB] = 0.f;
      }
      __syncthreads();
      continue;
    }

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
    // two partial sums per row (even / odd column of the fragment pair)
    float s0x = 0.f, s0y = 0.f, s1x = 0.f, s1y = 0.f;
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      acc[nt][0] = ex2(acc[nt][0] - m0);
      acc[nt][1] = ex2(acc[nt][1] - m0);
      acc[nt][2] = ex2(acc[nt][2] - m1);
      acc[nt][3] = ex2(acc[nt][3] - m1);
      s0x += acc[nt][0]; s0y += acc[nt][1];
      s1x += acc[nt][2]; s1y += acc[nt][3];
    }
    float s0 = s0x + s0y, s1 = s1x + s1y;
    s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
    s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
    s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
    const float i0 = __fdividef(1.f, s0), i1 = __fdividef(1.f, s1);
    if ((lane & 3) == 0) {  // natural-log LSE for the backward
      float* l = lse + ((long long)win * g.nH + h) * C::NT;
      if (rA < C::NT) l[rA] = (m0 + lg2(s0)) * LN2;
      if (rB < C::NT) l[rB] = (m1 + lg2(s1)) * LN2;
    }
#pragma unroll
    for (int nt = 0; nt < C::NT8; nt++) {
      acc[nt][0] *= i0; acc[nt][1] *= i0;
      acc[nt][2] *= i1; acc[nt][3] *= i1;
    }
    float o[4][4];
#pragma unroll
    for (int dt = 0; dt < 4; dt++) o[dt][0] = o[dt][1] = o[dt][2] = o[dt][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < C::MT; kk++) {
      uint32_t pa[4];
      pa[0] = pack_bf162(acc[2 * kk][0], acc[2 * kk][1]);
      pa[1] = pack_bf162(acc[2 * kk][2], acc[2 * kk][3]);
      pa[2] = pack_bf162(acc[2 * kk + 1][0], acc[2 * kk + 1][1]);
      pa[3] = pack_bf162(acc[2 * kk + 1][2], acc[2 * kk + 1][3]);
      const bf16* vp = Vs + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
      uint32_t vb[4];
      ldsm_x4_t(vb, vp);
      mma16816(o[0], pa, vb[0], vb[1]);
      mma16816(o[1], pa, vb[2], vb[3]);
      ldsm_x4_t(vb, vp + 16);
      mma16816(o[2], pa, vb[0], vb[1]);
      mma16816(o[3], pa, vb[2], vb[3]);
    }
#pragma unroll
    for (int dt = 0; dt < 4; dt++) {
      const int d = h * HD + dt * 8 + (lane & 3) * 2;
      if (tA >= 0) *reinterpret_cast<uint32_t*>(out + (long long)tA * g.C + d) = pack_bf162(o[dt][0], o[dt][1]);
      if (tB >= 0) *reinterpret_cast<uint32_t*>(out + (long long)tB * g.C + d) = pack_bf162(o[dt][2], o[dt][3]);
    }
    __syncthreads();  // everyone is done with this stage before the next-but-one gather overwrites it
  }
  cp_async_wait<0>();
}

static size_t fwd7_smem() { return (size_t)2 * 3 * TILE7 * 2 + (size_t)4 * 64 * 4; }

// ------------------------------------------------------------------------------------------------
// backward: no shared-memory transposition and no atomics in the inner loop.
//   phase A  warp = 16-query tile : S, P, dP, dS  -> dQ = dS K ;  dS also summed into register accumulators
//                                   (this warp's queries x all keys, over all windows) = rel-pos-bias gradient
//   phase B  warp = 16-key tile   : S^T = K Q^T, P^T, dP^T = V dO^T, dS^T recomputed in the transposed layout
//                                   -> dV = P^T dO, dK = dS^T Q straight from the accumulator fragments
// qkv-bias gradients are the column sums of dQ / dK / dV over all 49 slots (padded ones included).
template <bool SHIFT>
__global__ void __launch_bounds__(128, 3) window_attn_bwd7_kernel(
    const bf16* __restrict__ qkv, const bf16* __restrict__ qkv_bias, const float* __restrict__ bexp,
    const bf16* __restrict__ out, const bf16* __restrict__ dout, const float* __restrict__ lse,
    bf16* __restrict__ dqkv, float* __restrict__ dbias_table, float* __restrict__ dqkv_bias, Geo g, float scale,
    int nwin_total) {
  constexpr int WS = 7;
  using C = Cfg<WS>;
  // (a variant that ran phase A and phase B on two concurrent 4-warp groups of an 8-warp CTA measured 20 % SLOWER:
  // 2 CTAs/SM at the 128-register cap lose more than the halved per-window latency gains)
  constexpr int NTHREADS = 128;
  static_assert(C::KP == 64 && C::NW == 4, "fast path assumes a 64-slot window and 4 tiles per phase");
  extern __shared__ __align__(16) unsigned char smraw[];
  bf16* tiles = reinterpret_cast<bf16*>(smraw);                       // [2 stages][Q | K | V | dO | O]
  float* bm = reinterpret_cast<float*>(tiles + 2 * 5 * TILE7);         // [64][BLD] expanded bias (log2 domain, -inf pad)
  float* dbt = bm + C::KP * BLD;                                      // [NB] bias-gradient bins
  float* dqb = dbt + C::NB + 1;                                       // [3][32] (+1: NB is odd, keep 8-byte alignment)
  float* Dsm = dqb + 3 * HD;                                          // [64] rowsum(dO * O)
  float* Lrawb = Dsm + C::KP;                                         // [2][64] natural-log lse of the stage
  int* tokb = reinterpret_cast<int*>(Lrawb + 2 * 64);                 // [2][64]
  int* ridb = tokb + 2 * 64;                                          // [2][64]

  const int h = blockIdx.x;  // heads fastest: the nH CTAs sharing a window's token rows run together (DRAM page locality)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int win = blockIdx.y, stage = 0;
  uint4 bchunk[3];
#pragma unroll
  for (int part = 0; part < 3; part++)
    bchunk[part] = __ldg(reinterpret_cast<const uint4*>(qkv_bias + part * g.C + h * HD + (threadIdx.x & 3) * 8));
  if (win < nwin_total) issue7<true, NTHREADS>(g, win, h, qkv, bchunk, dout, out, lse, tiles, Lrawb, tokb, ridb);
  cp_async_commit();

  for (int i = threadIdx.x; i < C::KP * C::KP / 4; i += NTHREADS) {  // copy the expanded table of head h (float4)
    const int row = i >> 4, c4 = (i & 15) * 4;
    float4 v = __ldg(reinterpret_cast<const float4*>(bexp + (long long)h * 4096 + row * 64 + c4));
    if (row >= C::NT) v = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);  // padded query rows: P = 0
    *reinterpret_cast<float4*>(bm + row * BLD + c4) = v;
  }
  for (int i = threadIdx.x; i < C::NB; i += NTHREADS) dbt[i] = 0.f;
  for (int i = threadIdx.x; i < 3 * HD; i += NTHREADS) dqb[i] = 0.f;
  float dsacc[C::NT8][4];
#pragma unroll
  for (int nt = 0; nt < C::NT8; nt++) dsacc[nt][0] = dsacc[nt][1] = dsacc[nt][2] = dsacc[nt][3] = 0.f;

  const float c = scale * LOG2E;
  const int r0 = warp * 16;                       // this warp's query tile (phase A) / key tile (phase B)
  const int rA = r0 + (lane >> 2), rB = rA + 8;
  const int frag_off = (r0 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;  // A-fragment rows of the tile

  for (; win < nwin_total; win += gridDim.y, stage ^= 1) {
    const int nxt = win + gridDim.y;
    if (nxt < nwin_total)
      issue7<true, NTHREADS>(g, nxt, h, qkv, bchunk, dout, out, lse, tiles + (stage ^ 1) * 5 * TILE7, Lrawb + (stage ^ 1) * 64,
                   tokb + (stage ^ 1) * 64, ridb + (stage ^ 1) * 64);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* Qs = tiles + stage * 5 * TILE7;
    const bf16* Ks = Qs + TILE7;
    const bf16* Vs = Ks + TILE7;
    const bf16* dOs = Vs + TILE7;
    const bf16* Os = dOs + TILE7;
    const float* Lraw = Lrawb + stage * 64;
    const int* tok = tokb + stage * 64;
    const int* rid = ridb + stage * 64;
    if (g.dbg == 2) { __syncthreads(); continue; }
    {  // D[t] = rowsum(dO * O): two threads per row
      const int t = threadIdx.x >> 1, half = threadIdx.x & 1;
      float part = 0.f;
#pragma unroll
      for (int k = 0; k < 2; k++) {
        float fd[8], fo[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dOs + t * LD + half * 16 + k * 8), fd);
        unpack8(*reinterpret_cast<const bf16x8*>(Os + t * LD + half * 16 + k * 8), fo);
#pragma unroll
        for (int j = 0; j < 8; j++) part += fd[j] * fo[j];
      }
      part += __shfl_xor_sync(0xffffffffu, part, 1);
      if (half == 0) Dsm[t] = part;
    }
    __syncthreads();

    const int tA = rA < C::NT ? tok[rA] : -1, tB = rB < C::NT ? tok[rB] : -1;
    int ridA = 0, ridB = 0;
    if (SHIFT) { ridA = rid[rA]; ridB = rid[rB]; }
    // 16-slot tiles that hold a real token (bit t = tile t).  An all-padding QUERY tile has dO = 0 (its rows are cropped
    // away): dS = 0 there, so it adds nothing to dQ / dK / dV / the bias gradients and both phases skip it.  (Padded
    // KEY tiles are kept: their dK / dV are part of the qkv-bias gradient.)
    const unsigned b0 = __ballot_sync(0xffffffffu, tok[lane] >= 0), b1 = __ballot_sync(0xffffffffu, tok[lane + 32] >= 0);
    const unsigned qvalid = ((b0 & 0xffffu) ? 1u : 0u) | ((b0 >> 16) ? 2u : 0u) | ((b1 & 0xffffu) ? 4u : 0u) | ((b1 >> 16) ? 8u : 0u);
    // ---------------- phase A: rows = queries ----------------
    if ((qvalid >> warp) & 1u) {
      uint32_t qa[2][4], da[2][4];
      ldsm_x4(qa[0], Qs + frag_off);
      ldsm_x4(qa[1], Qs + frag_off + 16);
      ldsm_x4(da[0], dOs + frag_off);
      ldsm_x4(da[1], dOs + frag_off + 16);
      const float lA = Lraw[rA] * LOG2E, lB = Lraw[rB] * LOG2E, DA = Dsm[rA], DB = Dsm[rB];
      float dq[4][4];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) dq[dt][0] = dq[dt][1] = dq[dt][2] = dq[dt][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        float ds2[2][4];
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          const int nt = 2 * kk + hf;
          float sacc[4] = {0.f, 0.f, 0.f, 0.f};
          ds2[hf][0] = ds2[hf][1] = ds2[hf][2] = ds2[hf][3] = 0.f;
          uint32_t kb[4];
          const int boff = (nt * 8 + (lane & 7)) * LD + (lane >> 3) * 8;
          ldsm_x4(kb, Ks + boff);
          mma16816(sacc, qa[0], kb[0], kb[1]);
          mma16816(sacc, qa[1], kb[2], kb[3]);
          ldsm_x4(kb, Vs + boff);
          mma16816(ds2[hf], da[0], kb[0], kb[1]);
          mma16816(ds2[hf], da[1], kb[2], kb[3]);
          const int c0 = nt * 8 + (lane & 3) * 2;
          const float2 bA = *reinterpret_cast<const float2*>(bm + rA * BLD + c0);
          const float2 bB = *reinterpret_cast<const float2*>(bm + rB * BLD + c0);
          float sv[4] = {fmaf(sacc[0], c, bA.x) - lA, fmaf(sacc[1], c, bA.y) - lA, fmaf(sacc[2], c, bB.x) - lB,
                         fmaf(sacc[3], c, bB.y) - lB};
          if (SHIFT) {
            const int2 rc = *reinterpret_cast<const int2*>(rid + c0);
            if (ridA != rc.x) sv[0] += -100.f * LOG2E;
            if (ridA != rc.y) sv[1] += -100.f * LOG2E;
            if (ridB != rc.x) sv[2] += -100.f * LOG2E;
            if (ridB != rc.y) sv[3] += -100.f * LOG2E;
          }
          ds2[hf][0] = ex2(sv[0]) * (ds2[hf][0] - DA);
          ds2[hf][1] = ex2(sv[1]) * (ds2[hf][1] - DA);
          ds2[hf][2] = ex2(sv[2]) * (ds2[hf][2] - DB);
          ds2[hf][3] = ex2(sv[3]) * (ds2[hf][3] - DB);
#pragma unroll
          for (int e = 0; e < 4; e++) dsacc[nt][e] += ds2[hf][e];
        }
        uint32_t sa[4];
        sa[0] = pack_bf162(ds2[0][0], ds2[0][1]);
        sa[1] = pack_bf162(ds2[0][2], ds2[0][3]);
        sa[2] = pack_bf162(ds2[1][0], ds2[1][1]);
        sa[3] = pack_bf162(ds2[1][2], ds2[1][3]);
        const bf16* kp = Ks + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
        uint32_t kb[4];
        ldsm_x4_t(kb, kp);
        mma16816(dq[0], sa, kb[0], kb[1]);
        mma16816(dq[1], sa, kb[2], kb[3]);
        ldsm_x4_t(kb, kp + 16);
        mma16816(dq[2], sa, kb[0], kb[1]);
        mma16816(dq[3], sa, kb[2], kb[3]);
      }
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        const int d = h * HD + dt * 8 + (lane & 3) * 2;
        if (tA >= 0)
          *reinterpret_cast<uint32_t*>(dqkv + (long long)tA * 3 * g.C + d) = pack_bf162(dq[dt][0] * scale, dq[dt][1] * scale);
        if (tB >= 0)
          *reinterpret_cast<uint32_t*>(dqkv + (long long)tB * 3 * g.C + d) = pack_bf162(dq[dt][2] * scale, dq[dt][3] * scale);
      }
      colsum_to_smem(dq, scale, dqb, lane);
    }
    // ---------------- phase B: rows = keys (transposed recompute) ----------------
    {
      uint32_t ka[2][4], va[2][4];
      ldsm_x4(ka[0], Ks + frag_off);
      ldsm_x4(ka[1], Ks + frag_off + 16);
      ldsm_x4(va[0], Vs + frag_off);
      ldsm_x4(va[1], Vs + frag_off + 16);
      float dv[4][4], dk[4][4];
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        dv[dt][0] = dv[dt][1] = dv[dt][2] = dv[dt][3] = 0.f;
        dk[dt][0] = dk[dt][1] = dk[dt][2] = dk[dt][3] = 0.f;
      }
#pragma unroll
      for (int qq = 0; qq < 4; qq++) {
        if (!((qvalid >> qq) & 1u)) continue;
        float pT[2][4], dsT[2][4];
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
          const int nt = 2 * qq + hf;  // 8-query tile
          pT[hf][0] = pT[hf][1] = pT[hf][2] = pT[hf][3] = 0.f;
          dsT[hf][0] = dsT[hf][1] = dsT[hf][2] = dsT[hf][3] = 0.f;
          uint32_t qb[4];
          const int boff = (nt * 8 + (lane & 7)) * LD + (lane >> 3) * 8;
          ldsm_x4(qb, Qs + boff);
          mma16816(pT[hf], ka[0], qb[0], qb[1]);
          mma16816(pT[hf], ka[1], qb[2], qb[3]);
          ldsm_x4(qb, dOs + boff);
          mma16816(dsT[hf], va[0], qb[0], qb[1]);
          mma16816(dsT[hf], va[1], qb[2], qb[3]);
          const int q0 = nt * 8 + (lane & 3) * 2;  // the two query columns of this thread
          const float2 lq = *reinterpret_cast<const float2*>(Lraw + q0);
          const float2 Dq = *reinterpret_cast<const float2*>(Dsm + q0);
          // bias[query][key]: rows q0, q0+1 of the table, columns = this thread's key rows
          float sv[4] = {fmaf(pT[hf][0], c, bm[q0 * BLD + rA]) - lq.x * LOG2E,
                         fmaf(pT[hf][1], c, bm[(q0 + 1) * BLD + rA]) - lq.y * LOG2E,
                         fmaf(pT[hf][2], c, bm[q0 * BLD + rB]) - lq.x * LOG2E,
                         fmaf(pT[hf][3], c, bm[(q0 + 1) * BLD + rB]) - lq.y * LOG2E};
          if (SHIFT) {
            const int2 rq = *reinterpret_cast<const int2*>(rid + q0);
            if (ridA != rq.x) sv[0] += -100.f * LOG2E;
            if (ridA != rq.y) sv[1] += -100.f * LOG2E;
            if (ridB != rq.x) sv[2] += -100.f * LOG2E;
            if (ridB != rq.y) sv[3] += -100.f * LOG2E;
          }
          pT[hf][0] = ex2(sv[0]); pT[hf][1] = ex2(sv[1]); pT[hf][2] = ex2(sv[2]); pT[hf][3] = ex2(sv[3]);
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
        const int toff = (qq * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8;
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
#pragma unroll
      for (int dt = 0; dt < 4; dt++) {
        const int d = h * HD + dt * 8 + (lane & 3) * 2;
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
    __syncthreads();  // stage (and Dsm) free for the next-but-one gather
  }
  cp_async_wait<0>();
  // flush the register-resident rel-pos-bias gradient of this warp's query rows.  dS was formed with the true
  // probabilities, so it is the gradient w.r.t. the natural-domain score, i.e. w.r.t. the table entry.
#pragma unroll
  for (int nt = 0; nt < C::NT8; nt++)
#pragma unroll
    for (int e = 0; e < 4; e++) {
      const int row = (e < 2) ? rA : rB;
      const int col = nt * 8 + (lane & 3) * 2 + (e & 1);
      if (row < C::NT && col < C::NT) atomicAdd(&dbt[bias_index<WS>(row, col)], dsacc[nt][e]);
    }
  __syncthreads();
  for (int i = threadIdx.x; i < C::NB; i += NTHREADS) atomicAdd(&dbias_table[i * g.nH + h], dbt[i]);
  for (int i = threadIdx.x; i < 3 * HD; i += NTHREADS)
    atomicAdd(&dqkv_bias[(i / HD) * g.C + h * HD + (i % HD)], dqb[i]);
}

static size_t bwd7_smem() {
  using C = Cfg<7>;
  return (size_t)2 * 5 * TILE7 * 2 + (size_t)(C::KP * BLD + C::NB + 1 + 3 * HD + C::KP + 2 * 64) * 4 + (size_t)4 * 64 * 4;
}

}  // namespace wa
