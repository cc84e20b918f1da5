// (Shifted-)window attention core, forward and backward: entry points.  Kernels: window_attn7.cuh (ws = 7, 64-slot
// windows) and window_attn14.cuh (ws = 14, image-row tiles); persistent CTAs, head = blockIdx.x.
// A window holds 49 (ws 7) or 196 (ws 14) tokens and head_dim is 32, so a head of a window is a handful of
// m16n8k16 tiles: the kernels keep S / P / O in warp registers (mma.sync) instead of 64-row warpgroup tiles.
//
// Reference: models/swin_transformer.py
//   WindowAttention.forward :120-152      scores = (q*scale) k^T + rel-pos bias (+ shift mask) -> softmax -> @ v
//   SwinTransformerBlock.forward :283-325 zero pad AFTER norm1, roll(-shift), window_partition, ...,
//                                         window_reverse, roll(+shift), crop
//   create_attn_mask :249-272             -100 between tokens of different shift regions
//
// The pad / cyclic roll / window_partition / window_reverse / roll-back / crop copies of the reference are
// folded into the kernel's addressing: a CTA computes, for each of its ws*ws window slots, which token of
// the un-padded [B, H, W] map sits there after pad+roll (or that it is a padded slot, whose q/k/v is the qkv
// bias because the reference pads the *normalised* activations with zeros before the qkv Linear), gathers
// those rows from the token-major qkv tensor and scatters its output rows back to token order.
// The relative-position bias and the -100 shift mask come from closed forms (SURVEY.md §7): no [nW, N, N] mask tensor
// exists; the bias is expanded once per call (ws 7) or staged per CTA as a [27][32] table (ws 14).
//
// Math: bf16 mma.sync m16n8k16 with fp32 accumulate; softmax in fp32 registers; P rounded to bf16 for PV
// (same as the reference under autocast).  head_dim is 32 in every Swin variant.
// The backward recomputes P from the saved log-sum-exp (no [B_, nH, N, N] tensor is saved).  esvit_window_attn_probs
// (window_attn_probs.cuh) writes P itself, for SwinTransformer.forward_selfattention.
#include <cstdlib>

#include "wa_common.cuh"
#include "window_attn7.cuh"
#include "window_attn14.cuh"
#include "window_attn_probs.cuh"

namespace wa {

static bool make_geo(Geo& g, int B, int H, int W, int C, int nH, int ws, int shift) {
  if (B <= 0 || H <= 0 || W <= 0 || nH <= 0 || C != nH * HD || (ws != 7 && ws != 14) || shift < 0 || shift >= ws) return false;
  g.B = B; g.H = H; g.W = W; g.C = C; g.nH = nH; g.shift = shift;
  g.Hp = (H + ws - 1) / ws * ws;
  g.Wp = (W + ws - 1) / ws * ws;
  g.nWy = g.Hp / ws;
  g.nWx = g.Wp / ws;
  const char* d = getenv("ESVIT_ATTN_DBG");
  g.dbg = d ? atoi(d) : 0;
  return true;
}

// persistent grid: `per_sm` resident CTAs per SM, heads on blockIdx.x.  ESVIT_ATTN_GY (tests) forces a small grid so a
// few windows exercise the multi-window loops.
static int windows_grid(int nwin, int nH, int per_sm) {
  int gy = esvit_num_sms() * per_sm / nH;  // floor: one CTA too many would be a whole extra wave
  if (gy < 1) gy = 1;
  const char* e = getenv("ESVIT_ATTN_GY");
  if (e && atoi(e) > 0) gy = atoi(e);
  return gy > nwin ? nwin : gy;
}

template <typename K>
static cudaError_t opt_in_smem(K kernel, size_t smem) {
  return smem > 48 * 1024 ? cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                          : cudaSuccess;
}

}  // namespace wa

// qkv bf16 [B,H,W,3C] = qkv GEMM output INCLUDING its bias (channel order [q|k|v][head][32]); qkv_bias bf16 [3C] is
// what a padded slot holds; bias_table fp32 [(2ws-1)^2, nH]; bias_ws fp32 [nH*8192] scratch (ws 7: expanded
// bias; ws 14 backward: bias-gradient accumulator); out bf16 [B,H,W,C]; lse fp32 [B*nW, nH, ws*ws]
// ws = 7: expand the rel-pos bias table into bias_ws [nH][64][64] (log2 domain, -inf padding) once, for every attention
// call of the step that uses this table (pass bias_ready = 1 to them).  ws = 14: nothing to do.
ESVIT_API int esvit_window_attn_expand_bias(const float* bias_table, float* bias_ws, int nH, int ws, void* stream) {
  if (nH <= 0 || (ws != 7 && ws != 14) || !bias_table) return ESVIT_ERR_BAD_ARG;
  if (ws == 7) {
    if (!bias_ws) return ESVIT_ERR_BAD_ARG;
    wa::expand_bias7_kernel<<<nH, 256, 0, (cudaStream_t)stream>>>(bias_table, bias_ws, nH);
  }
  ESVIT_LAUNCH_CHECK();
}

ESVIT_API int esvit_window_attn_fwd(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws,
                                    int bias_ready, void* out, float* lse, int B, int H, int W, int C, int nH, int ws,
                                    int shift, float scale, void* stream) {
  wa::Geo g;
  if (!wa::make_geo(g, B, H, W, C, nH, ws, shift)) return ESVIT_ERR_BAD_ARG;
  const int nwin = B * g.nWy * g.nWx;
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* q = (const bf16*)qkv;
  const bf16* qb = (const bf16*)qkv_bias;
  if (ws == 7) {
    if (!bias_ws) return ESVIT_ERR_BAD_ARG;
    if (!bias_ready) wa::expand_bias7_kernel<<<nH, 256, 0, st>>>(bias_table, bias_ws, nH);
    const size_t smem = wa::fwd7_smem();
    const int gx = wa::windows_grid(nwin, nH, 16);  // persistent: ~4 waves of 4 resident CTAs per SM
    if (shift > 0)
      wa::window_attn_fwd7_kernel<true><<<dim3(nH, gx), 128, smem, st>>>(q, qb, bias_ws, (bf16*)out, lse, g, scale, nwin);
    else
      wa::window_attn_fwd7_kernel<false><<<dim3(nH, gx), 128, smem, st>>>(q, qb, bias_ws, (bf16*)out, lse, g, scale, nwin);
  } else {
    const size_t smem = wa::fwd14_smem();
    cudaError_t e = wa::opt_in_smem(wa::window_attn_fwd14_kernel<true>, smem);
    if (e == cudaSuccess) e = wa::opt_in_smem(wa::window_attn_fwd14_kernel<false>, smem);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(nH, wa::windows_grid(nwin, nH, 2));
    if (shift > 0)
      wa::window_attn_fwd14_kernel<true><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, (bf16*)out, lse, g, scale, nwin);
    else
      wa::window_attn_fwd14_kernel<false><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, (bf16*)out, lse, g, scale, nwin);
  }
  ESVIT_LAUNCH_CHECK();
}

// dqkv bf16 [B,H,W,3C] is fully written; dbias_table fp32 [(2ws-1)^2, nH] and dqkv_bias fp32 [3C] (the COMPLETE
// qkv-bias gradient: column sums of dq/dk/dv over all window slots, padded ones included) are ACCUMULATED into
// (caller zero-fills).
ESVIT_API int esvit_window_attn_bwd(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws,
                                    int bias_ready, const void* out, const void* dout, const float* lse, void* dqkv,
                                    float* dbias_table, float* dqkv_bias, int B, int H, int W, int C, int nH, int ws,
                                    int shift, float scale, void* stream) {
  wa::Geo g;
  if (!wa::make_geo(g, B, H, W, C, nH, ws, shift)) return ESVIT_ERR_BAD_ARG;
  const int nwin = B * g.nWy * g.nWx;
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* q = (const bf16*)qkv;
  const bf16* qb = (const bf16*)qkv_bias;
  if (ws == 7) {
    if (!bias_ws) return ESVIT_ERR_BAD_ARG;
    if (!bias_ready) wa::expand_bias7_kernel<<<nH, 256, 0, st>>>(bias_table, bias_ws, nH);
    const size_t smem = wa::bwd7_smem();
    cudaError_t e = wa::opt_in_smem(wa::window_attn_bwd7_kernel<true>, smem);
    if (e == cudaSuccess) e = wa::opt_in_smem(wa::window_attn_bwd7_kernel<false>, smem);
    if (e != cudaSuccess) return (int)e;
    const int gx = wa::windows_grid(nwin, nH, 12);  // 3 CTAs / SM resident, ~4 waves of persistent CTAs
    if (shift > 0)
      wa::window_attn_bwd7_kernel<true><<<dim3(nH, gx), 128, smem, st>>>(q, qb, bias_ws, (const bf16*)out,
                                                                         (const bf16*)dout, lse, (bf16*)dqkv,
                                                                         dbias_table, dqkv_bias, g, scale, nwin);
    else
      wa::window_attn_bwd7_kernel<false><<<dim3(nH, gx), 128, smem, st>>>(q, qb, bias_ws, (const bf16*)out,
                                                                          (const bf16*)dout, lse, (bf16*)dqkv,
                                                                          dbias_table, dqkv_bias, g, scale, nwin);
  } else {
    if (!bias_ws) return ESVIT_ERR_BAD_ARG;
    const size_t smem = wa::bwd14_smem();
    cudaError_t e = wa::opt_in_smem(wa::window_attn_bwd14_kernel<true>, smem);
    if (e == cudaSuccess) e = wa::opt_in_smem(wa::window_attn_bwd14_kernel<false>, smem);
    if (e == cudaSuccess) e = cudaMemsetAsync(bias_ws, 0, (size_t)nH * wa::GACC14 * sizeof(float), st);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(nH, wa::windows_grid(nwin, nH, 2));
    if (shift > 0)
      wa::window_attn_bwd14_kernel<true><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, (const bf16*)out, (const bf16*)dout,
                                                                      lse, (bf16*)dqkv, bias_ws, dqkv_bias, g, scale, nwin);
    else
      wa::window_attn_bwd14_kernel<false><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, (const bf16*)out, (const bf16*)dout,
                                                                       lse, (bf16*)dqkv, bias_ws, dqkv_bias, g, scale, nwin);
    wa::fold_dbias14_kernel<<<dim3(27, nH), 192, 0, st>>>(bias_ws, dbias_table, nH);
  }
  ESVIT_LAUNCH_CHECK();
}

// probs fp32 [B*nWy*nWx, nH, ws*ws, ws*ws] is fully written: the softmax of every (window, head) of the call, padded slots
// included, windows of the frame rolled by -shift (the reference's window_partition order).  Inputs as in
// esvit_window_attn_fwd; nothing else is written (ws 7 with bias_ready = 0 expands the table into bias_ws first).
ESVIT_API int esvit_window_attn_probs(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws,
                                      int bias_ready, float* probs, int B, int H, int W, int C, int nH, int ws,
                                      int shift, float scale, void* stream) {
  wa::Geo g;
  if (!wa::make_geo(g, B, H, W, C, nH, ws, shift) || !qkv || !qkv_bias || !bias_table || !probs) return ESVIT_ERR_BAD_ARG;
  const int nwin = B * g.nWy * g.nWx;
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* q = (const bf16*)qkv;
  const bf16* qb = (const bf16*)qkv_bias;
  if (ws == 7) {
    if (!bias_ws) return ESVIT_ERR_BAD_ARG;
    if (!bias_ready) wa::expand_bias7_kernel<<<nH, 256, 0, st>>>(bias_table, bias_ws, nH);
    const size_t smem = wa::probs7_smem();
    const dim3 grid(nH, wa::windows_grid(nwin, nH, 16));
    if (shift > 0)
      wa::window_attn_probs7_kernel<true><<<grid, 128, smem, st>>>(q, qb, bias_ws, probs, g, scale, nwin);
    else
      wa::window_attn_probs7_kernel<false><<<grid, 128, smem, st>>>(q, qb, bias_ws, probs, g, scale, nwin);
  } else {
    const size_t smem = wa::probs14_smem();
    cudaError_t e = wa::opt_in_smem(wa::window_attn_probs14_kernel<true>, smem);
    if (e == cudaSuccess) e = wa::opt_in_smem(wa::window_attn_probs14_kernel<false>, smem);
    if (e != cudaSuccess) return (int)e;
    const dim3 grid(nH, wa::windows_grid(nwin, nH, 2));
    if (shift > 0)
      wa::window_attn_probs14_kernel<true><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, probs, g, scale, nwin);
    else
      wa::window_attn_probs14_kernel<false><<<grid, wa::T14, smem, st>>>(q, qb, bias_table, probs, g, scale, nwin);
  }
  ESVIT_LAUNCH_CHECK();
}
