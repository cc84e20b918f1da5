/* esvit_b200 C ABI — the drop-in boundary of the H100-native EsViT multi-crop self-distillation step.
 *
 * Every entry point takes raw DEVICE pointers + sizes + a cudaStream_t (as void*), launches sm_90a kernels on
 * that stream and returns an int status: 0 = ok, otherwise a cudaError_t value or ESVIT_ERR_BAD_ARG (1001) for an
 * unsupported shape.  No entry point allocates, frees or synchronises; all buffers (inputs, outputs, workspaces)
 * are owned by the caller (PyTorch's caching allocator on the host side) and must stay alive in stream order.
 * Entry points are re-entrant and keep no mutable global state.
 *
 * The reference (microsoft/esvit) is pure Python/PyTorch and has no FFI of its own; each function below names the
 * reference code it replaces (file:line relative to the reference tree).  INTEGRATION.md shows the ctypes binding
 * and the module-level swap a maintainer would add to main_esvit.py.
 *
 * Conventions: "bf16" = __nv_bfloat16 bits; token-major activations [B, H*W, C] (same order as the reference);
 * fp32 residual stream; bf16 GEMM operands.  "ACCUMULATED" outputs must be zero-filled by the caller.
 */
#ifndef ESVIT_B200_H
#define ESVIT_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define ESVIT_ERR_BAD_ARG 1001

/* ---- residual add + LayerNorm ------------------------------------------------------------------------------
 * replaces: x = shortcut + drop_path(branch); y = norm(x)      models/swin_transformer.py:329-331, :283, :687
 * xout = x + keep[row / tokens_per_sample] * delta (delta/keep/xout may be NULL; delta = proj / fc2 GEMM output
 * including its bias); y = LN(xout) (y may be NULL).  x may be NULL (= 0) when delta is given: xout = fp32(delta), the
 * first LN after PatchMerging's reduction GEMM (:411-415) without a separate bf16 -> fp32 pass.
 * x fp32 [T,C]; delta bf16 [T,C]; y bf16 or fp32 [T,C]; mean/rstd fp32 [T] (saved for backward).  keep fp32 has one
 * entry per tokens_per_sample rows: per sample ([T / tps], tps = tokens of one sample) or per row ([T], tps = 1, the
 * layout the training step passes).  xout is written only when delta is given.  C % 4 == 0, C <= 2048, T >= 1. */
int esvit_add_ln_fwd(const float* x, const void* delta, const float* keep, int tokens_per_sample,
                     const float* gamma, const float* beta, float eps, float* xout, void* y, int y_is_bf16,
                     float* mean, float* rstd, long long T, int C, void* stream);
/* dx = dxo + LNbwd(dy); ddelta = keep * dx (bf16); dgamma/dbeta/ddelta_bias ACCUMULATED (ddelta_bias = column sums of
 * ddelta = gradient of the proj / fc2 bias).  dy / dxo / dx / ddelta / ddelta_bias may be NULL; dy = NULL (a residual
 * add without norm: dx = dxo) leaves dgamma / dbeta untouched and does not read xs / mean / rstd / gamma. */
int esvit_add_ln_bwd(const void* dy, int dy_is_bf16, const float* dxo, const float* xs, const float* mean,
                     const float* rstd, const float* gamma, const float* keep, int tokens_per_sample, float* dx,
                     void* ddelta, float* dgamma, float* dbeta, float* ddelta_bias, long long T, int C, void* stream);

/* ---- PatchMerging gather + LayerNorm(4C) ---------------------------------- models/swin_transformer.py:393-417
 * x fp32 [B,H,W,C] -> y bf16 [B,ceil(H/2)*ceil(W/2),4C]; odd H / W are zero-padded and the pad counts in the 4C
 * statistics (the 4C->2C reduction that follows runs on esvit_gemm_bf16).  C % 4 == 0, 4C <= 3072.
 * bwd: dx written at every real position; dgamma / dbeta [4C] ACCUMULATED. */
int esvit_patch_merge_ln_fwd(const float* x, const float* gamma, const float* beta, float eps, void* y, float* mean,
                             float* rstd, int B, int H, int W, int C, void* stream);
int esvit_patch_merge_ln_bwd(const void* dy, const float* x, const float* mean, const float* rstd,
                             const float* gamma, float* dx, float* dgamma, float* dbeta, int B, int H, int W, int C,
                             void* stream);

/* ---- token mean (AdaptiveAvgPool1d(1)) ------------------------------------- models/swin_transformer.py:688-689 */
int esvit_token_mean_fwd(const float* region, float* pooled, int B, int N, int C, void* stream);
int esvit_token_mean_bwd(const float* dpooled, const float* dregion_in, float* dregion, int B, int N, int C,
                         void* stream);

/* ---- PatchEmbed: 4x4/4 conv (3->E) + LayerNorm -------------------------------- models/swin_transformer.py:537-547
 * img fp32 [B,3,H,W], H and W multiples of 4; w fp32 [E,3,4,4]; out fp32 [B,(H/4)*(W/4),E]; E <= 128 or E = 192.
 * bwd ACCUMULATES dw/dbias/dgamma/dbeta. */
int esvit_patch_embed_fwd(const float* img, const float* w, const float* bias, const float* gamma, const float* beta,
                          float eps, float* out, float* mean, float* rstd, int B, int H, int W, int E, void* stream);
int esvit_patch_embed_bwd(const float* img, const float* w, const float* bias, const float* gamma, const float* mean,
                          const float* rstd, const float* dout, float* dw, float* dbias, float* dgamma, float* dbeta,
                          int B, int H, int W, int E, void* stream);

/* ---- (shifted-)window attention core ----------------------------- models/swin_transformer.py:120-152, :283-325
 * Folds pad / roll / window_partition / rel-pos bias / -100 shift mask / softmax / PV / window_reverse / roll / crop.
 * qkv bf16 [B,H,W,3C] ([q|k|v][head][32]) is the qkv GEMM output including its bias; qkv_bias bf16 [3C] is what a
 * padded slot holds (the bias alone); bias_table fp32 [(2ws-1)^2, nH]; out bf16 [B,H,W,C]; lse fp32
 * [B*nWindows, nH, ws*ws].  ws in {7,14}; head_dim 32; B, H, W, nH >= 1 and 0 <= shift < ws (else status 1001).
 * bias_ws fp32 [nH*8192]: caller-owned scratch (ws 7: the rel-pos bias expanded to [nH][64][64]; ws 14 backward: the
 * lane-expanded bias-gradient accumulator [nH][27][6][32], cleared and folded into dbias_table inside the call).
 * bias_ready (ws 7): 1 = bias_ws already holds the expansion written by esvit_window_attn_expand_bias for this table
 * (one expansion per table per step instead of one per call), 0 = the call expands it itself.
 * bwd: dqkv fully written; dbias_table fp32 and dqkv_bias fp32 [3C] (complete qkv-bias gradient) ACCUMULATED.
 * Kernels: bf16 mma.sync with S / P / O in warp registers, one persistent CTA loop per head (DESIGN.md 4.3). */
int esvit_window_attn_expand_bias(const float* bias_table, float* bias_ws, int nH, int ws, void* stream);
int esvit_window_attn_fwd(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws, int bias_ready,
                          void* out, float* lse, int B, int H, int W, int C, int nH, int ws, int shift, float scale,
                          void* stream);
int esvit_window_attn_bwd(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws, int bias_ready,
                          const void* out, const void* dout, const float* lse, void* dqkv, float* dbias_table,
                          float* dqkv_bias, int B, int H, int W, int C, int nH, int ws, int shift, float scale,
                          void* stream);
/* Attention probabilities (SwinTransformer.forward_selfattention, models/swin_transformer.py:766-796; softmax :141-147):
 * probs fp32 [B*nWy*nWx, nH, ws*ws, ws*ws] fully written, window w = b*nWy*nWx + wy*nWx + wx of the padded frame rolled
 * by -shift, slots row-major, rows and columns of padded slots included.  qkv / qkv_bias / bias_table / bias_ws /
 * bias_ready as for fwd; the row max and sum are computed here (the forward saves no LSE for all-padding query tiles). */
int esvit_window_attn_probs(const void* qkv, const void* qkv_bias, const float* bias_table, float* bias_ws, int bias_ready,
                            float* probs, int B, int H, int W, int C, int nH, int ws, int shift, float scale, void* stream);

/* ---- wgmma GEMM family (csrc/gemm2_wgmma.cu): every nn.Linear of the step, forward, input
 * gradient and weight gradient -------- models/swin_transformer.py:21-37,88-91,125,150,393-420; vision_transformer.py:385-418
 * 64 x BN or 128 x BN tiles (1 or 2 consumer warpgroups, BN 128 / 256); operands K-major or MN-major (the same
 * row-major matrices read "transposed" by TMA + wgmma's transpose bits: no transposed copies).
 * gemm_bf16: out[M,N] (bf16) = act(opA(a) . opB(b) + bias[N]).  a: a_mn = 0 [M,K] | a_mn = 1 [K,M];  b: b_mn = 0 [N,K]
 *   (Linear weight, forward) | b_mn = 1 [K,N] (Linear weight [out = K, in = N], input gradient).  act 0 identity, 1 exact
 *   GELU (pre != NULL also receives gelu'(pre-activation)); act 2: QuickGELU x sigmoid(1.702 x) (pre likewise; a_mn =
 *   b_mn = 0 only).  tile: 0 = automatic, else warpgroups * 1000 + BN.
 * gemm_mul_colsum2: out = (a . opB(b)) * mult; colsum[N] (fp32) += column sums of out (caller zero-fills).  The fc2
 *   input gradient fused with the GELU backward of fc1 (mult = gelu'(pre-activation) from gemm_bf16 act 1) and the fc1
 *   bias gradient.  ws fp32 [160 * N]: caller-owned scratch (per-CTA partial column sums, folded into colsum).
 * gemm_wgrad: dw[N,K] (fp32) (+)= dy[T,N]^T . x[T,K], split over T, deterministic fold of fp32 partial tiles held in ws
 *   (esvit_gemm_wgrad_ws_floats(N, K) fp32 elements); dw and ws 16-byte aligned (else ESVIT_ERR_BAD_ARG).  All of
 *   M / N / K / T multiples of 8. */
int esvit_gemm_bf16(const void* a, const void* b, const float* bias, void* out, void* pre, long long M, int N, int K,
                    int a_mn, int b_mn, int act, int tile, void* stream);
int esvit_gemm_mul_colsum2(const void* a, const void* b, const void* mult, void* out, float* colsum, float* ws,
                           long long M, int N, int K, int b_mn, int tile, void* stream);
int esvit_gemm_wgrad_ws_floats(int N, int K);
int esvit_gemm_wgrad(const void* dy, const void* x, float* dw, float* ws, long long T, int N, int K, int accumulate,
                     int tile, void* stream);
/* mlp_fwd: y[M,C] (bf16) = GELU(x[M,C] . w1[4C,C]^T + b1) . w2[C,4C]^T + b2 in one back-to-back wgmma kernel: the hidden
 *   activation stays on chip.  h, gelu_grad [M,4C] bf16: both NULL (no-grad forward) or both set (they receive GELU(pre)
 *   and gelu'(pre) for the backward).  Bit-identical to gemm_bf16 act 1 followed by gemm_bf16 act 0.  C in {96, 128, 192}
 *   (other C: status 1001); biases fp32 or NULL; matrices 16-byte aligned. */
int esvit_mlp_fwd(const void* x, const void* w1, const float* b1, const void* w2, const float* b2, void* y, void* h,
                  void* gelu_grad, long long M, int C, void* stream);

/* ---- DINOHead pieces ------------------------------------------------------ models/vision_transformer.py:403-417
 * l2norm: y = x / max(||x||, eps) rows (bf16); weight_norm: w(bf16) = v * g / ||v||_row (fp32 v [K,D], g [K]). */
int esvit_l2norm_fwd(const void* x, void* y, float* inv, float eps, long long R, int D, void* stream);
int esvit_l2norm_bwd(const void* x, const void* dy, const float* inv, void* dx, long long R, int D, void* stream);
int esvit_weight_norm_fwd(const float* v, const float* g, void* w, float* norm, long long K, int D, void* stream);
/* dw: bf16 [K,D], the gradient of w; dv fp32 [K,D]; dg fp32 [K] or NULL */
int esvit_weight_norm_bwd(const float* v, const float* g, const float* norm, const void* dw, float* dv, float* dg,
                          long long K, int D, void* stream);

/* ---- DINOLoss / DDINOLoss ---------------------------------------------------- main_esvit.py:620-648, :683-750
 * row_lse: lse[r] = log sum_k exp((x[r,k] - center[k]) * inv_temp)   (center NULL for student rows).
 * dino_ce_fwd: row_loss[r] = n_r*lse_s[r] - sum_j <softmax((t[trow[r][j]]-center)*inv_temp_t), s[r]*inv_tau_s>;
 *   lse_s[r] = LSE(s[r]*inv_tau_s) is an OUTPUT (computed in the same pass, kept for the backward)
 * dino_ce_bwd: ds[r] = gscale[0]*w[r]*inv_tau_s * (n_r*softmax(s[r]*inv_tau_s) - sum_j q_j)   (bf16 out)
 * trow int32 [R,2], -1 = no pair.  s/t bf16 [R,K]/[Rt,K], K % 8 == 0.
 * order int32 [R] or NULL: CTA i works on row order[i] (a permutation; image-major keeps the paired teacher rows in L2). */
int esvit_row_lse(const void* x, const float* center, float inv_temp, float* lse, long long R, int K, void* stream);
int esvit_dino_ce_fwd(const void* s, const void* t, const float* center, float* lse_s, const float* lse_t,
                      const int* trow, const int* order, float inv_temp_t, float inv_tau_s, float* row_loss, long long R,
                      int K, void* stream);
int esvit_dino_ce_bwd(const void* s, const void* t, const float* center, const float* lse_s, const float* lse_t,
                      const int* trow, const int* order, const float* w, const float* gscale, float inv_temp_t,
                      float inv_tau_s, void* ds, long long R, int K, void* stream);
int esvit_weighted_sum(const float* v, const float* w, int R, float* out, void* stream);
/* The same loss with the teacher probabilities stored once per teacher row (every teacher row is paired with ~3.5 student
 * rows; recomputing its exponentials per pairing made both CE kernels SFU-bound):
 * row_softmax_q: lse[r] as esvit_row_lse, q[r,k] = 2^12 * softmax((x[r] - center) * inv_temp)_k in fp16 [R,K]
 *   (K <= esvit_row_softmax_q_max_k()).
 * dino_ce_q_fwd / bwd: esvit_dino_ce_fwd / bwd with q (that fp16 tensor) in place of (t, center, lse_t, inv_temp_t). */
int esvit_row_softmax_q_max_k(void);
int esvit_row_softmax_q(const void* x, const float* center, float inv_temp, float* lse, void* q, long long R, int K,
                        void* stream);
int esvit_dino_ce_q_fwd(const void* s, const void* q, float* lse_s, const int* trow, const int* order, float inv_tau_s,
                        float* row_loss, long long R, int K, void* stream);
int esvit_dino_ce_q_bwd(const void* s, const void* q, const float* lse_s, const int* trow, const int* order,
                        const float* w, const float* gscale, float inv_tau_s, void* ds, long long R, int K, void* stream);
/* Mixup targets (main_esvit.py:638-641): targets fp32 [ncrops, B, B] (T_v[j, b], teacher sample j, student sample b),
 * finite and non-negative; q the fp16 [2B, K] output of esvit_row_softmax_q.  For student row r = (v, b):
 *   C_r = sum_{iq != v} sum_j T_v[j, b],   q_out[r] = sum_{iq != v} sum_j T_v[j, b] * q[iq*B + j] / C_r  (0 where C_r = 0)
 *   w[r] = C_r * w_scale
 * so esvit_dino_ce_q_fwd / bwd on q_out with trow[r] = (r, -1) and this w compute the mixup loss when w_scale =
 * 1 / (n_terms * B).  q_out fp16 [ncrops*B, K] in the same 2^12-scaled format; ws: fp16 [2 * ncrops*B *
 * esvit_mixup_q_kpad(B)] scratch. */
int esvit_mixup_q_kpad(int B);
int esvit_mixup_q(const float* targets, const void* q, int ncrops, int B, int K, float w_scale, void* ws, float* w,
                  void* q_out, void* stream);

/* ---- update_center ----------------------------------------------------------- main_esvit.py:650-660, :752-770
 * colsum: out[k] = sum_r t[r,k] (deterministic two-stage); workspace fp32 [esvit_colsum_workspace_rows()*K].
 * center_ema: center_out = center*m + (colsum/rows_total)*(1-m)  (after the caller's SUM all-reduce of colsum);
 * out-of-place like the reference's rebinding, because the loss backward still reads the old center.  momentum is the
 * double the reference holds: m and 1 - m are each rounded to fp32 from it, as ATen rounds a Python scalar. */
int esvit_colsum_workspace_rows(void);
int esvit_colsum(const void* t, long long R, int K, float* workspace, float* out, void* stream);
int esvit_center_ema(const float* center, const float* colsum, float rows_total, double momentum, float* center_out,
                     int K, void* stream);

/* ---- DDINOLoss region match -------------------------------------------------------- main_esvit.py:735-736
 * normalize_rows: y = x / max(||x||, eps), fp32 [R,P].
 * region_match: for every student region token of every crop v != iq, the FIRST arg-max over the Tg teacher tokens
 * of view iq (same image) of the cosine similarity.  sn fp32 [Rs,P] rows ordered (crop, image, token) with 2 global
 * crops of Tg tokens then ncrops-2 local crops of Tl tokens; tn fp32 [2*B*Tg, P].
 * idx_out int64 [2, ncrops, B, Tg] (slots of v == iq or i >= T_v untouched); trow int32 [Rs,2] teacher region rows.
 * Teacher rows that do not fit shared memory at once (Tg*P*4 > 220 KB, ViT) are streamed in chunks; same indices. */
int esvit_normalize_rows(const float* x, float* y, long long R, int P, float eps, void* stream);
int esvit_region_match(const float* sn, const float* tn, int B, int ncrops, int Tg, int Tl, int P,
                       long long* idx_out, int* trow, void* stream);

/* ---- ViT whole-sequence attention, head dim 64 ------------------------ models/vision_transformer.py:83-95
 * qkv bf16 [B*L, 3C] (qkv GEMM output incl. bias; channels [q|k|v][head][64]), C = nH*64 (else ESVIT_ERR_BAD_ARG),
 * out bf16 [B*L, C] in (attn @ v).transpose(1, 2).reshape(B, L, C) order, lse fp32 [B, nH, L] (natural log).
 * bwd: dout bf16 [B*L, C]; dvec fp32 [B*nH*L] workspace; dqkv bf16 [B*L, 3C] fully written (no atomics). */
int esvit_mhsa_fwd(const void* qkv, void* out, float* lse, int B, int L, int C, int nH, float scale, void* stream);
int esvit_mhsa_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv,
                   int B, int L, int C, int nH, float scale, void* stream);

/* ---- ViT token embedding ------------------------------------------ models/vision_transformer.py:124-139, 233-251
 * patches: img fp32 [B,3,S,S] -> bf16 [B*N, 3p^2], N = (S/p)^2, columns in the conv weight's (c, ky, kx) order (p even).
 * tokens_fwd: x fp32 [B, 1+N, D] = cat(cls, pe bf16 [B*N, D]) + pos fp32 [1+N, D].
 * tokens_bwd: g fp32 [B, 1+N, D] -> dpe bf16 [B*N, D], dpos fp32 [1+N, D] (written); dbias, dcls fp32 [D] written
 *   (accumulate = 0) or added to (accumulate = 1).  Fixed summation order, no atomics.
 * split: dir 0: x fp32 [B, 1+N, D] -> cls [B, D], region [B*N, D]; dir 1: gradients of cls / region (either may be
 *   null = zero) -> x. */
int esvit_vit_patches(const float* img, void* patches, int B, int S, int p, void* stream);
int esvit_vit_tokens_fwd(const void* pe, const float* cls, const float* pos, float* x, int B, int N, int D, void* stream);
int esvit_vit_tokens_bwd(const float* g, void* dpe, float* dpos, float* dbias, float* dcls, int accumulate, int B, int N,
                         int D, void* stream);
int esvit_vit_split(float* x, float* cls, float* region, int B, int N, int D, int dir, void* stream);

/* ---- CvT (models/cvt_v4_transformer.py) ------------------------------------------------------------------------------
 * conv_im2col: x fp32 NCHW [B, C, H, W] (nchw = 1) or token-major [B*H*W, C] (nchw = 0) -> rows bf16 [B*Ho*Wo, Kp] of a
 *   k x k / stride / pad conv in the weight's (c, ky, kx) order, columns >= C*k*k zero; Kp % 8 == 0.
 * conv_col2im: the transpose: drows bf16 [B*Ho*Wo, Kp] -> dx fp32 token-major [B*H*W, C] (written), fixed-order gather.
 * mhsa_win_fwd / _bwd: esvit_mhsa_fwd / _bwd over the w x w windows of the zero-padded map (Hp, Wp = H, W rounded up to
 *   multiples of w; any 1 <= w <= min(H, W), ceil(w*w / 64) query and key tiles per window; B * windows <= 65535 and
 *   B*Hp*Wp <= INT_MAX) at head dim 64 or 32: C = nH*64 or C = nH*32 (else ESVIT_ERR_BAD_ARG), channels
 *   [q|k|v][head][C / nH]: qkv / dqkv bf16 [B*Hp*Wp, 3C], out / dout bf16 [B*H*W, C] (padded rows not stored / read as
 *   zero), lse / dvec fp32 [B * windows, nH, w*w].
 * dwbn_*: depthwise 3x3 conv (pad 1, no bias; w fp32 [C, 9]) of y bf16 [B*H*W, C] zero-padded to Hp x Wp, then
 *   BatchNorm2d; C % 64 == 0.  fwd_stats: z bf16 [B*Hp*Wp, C] (conv output), sums fp64 [2C + 1] = (sum z, sum z^2, count).
 *   fwd_apply: stat fp32 [4C] = (mean, rstd, gamma rstd, beta - mean gamma rstd) from sums (train: run_mean / run_var /
 *   nbt updated in place when given) or from run_mean / run_var (train = 0); out bf16 [N, C] = z * stat[2] + stat[3].
 *   bwd_stats: sums fp64 [2C + 1] = (sum dy, sum dy xhat, count); dbeta / dgamma fp32 [C] += the local sums.
 *   bwd_apply: dx bf16 [B*H*W, C] (written), dw fp32 [C, 9] += filter gradient; coef fp32 [3C] scratch.
 *   part: fp32 scratch of ceil(B*Hp*Wp / 256) * 9 * C floats.  No floating-point atomics. */
int esvit_conv_im2col(const float* x, void* rows, int nchw, int B, int C, int H, int W, int k, int stride, int pad, int Kp,
                      void* stream);
int esvit_conv_col2im(const void* rows, float* dx, int B, int C, int H, int W, int k, int stride, int pad, int Kp,
                      void* stream);
int esvit_mhsa_win_fwd(const void* qkv, void* out, float* lse, int B, int H, int W, int w, int C, int nH, float scale,
                       void* stream);
int esvit_mhsa_win_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* dvec, void* dqkv,
                       int B, int H, int W, int w, int C, int nH, float scale, void* stream);
int esvit_dwbn_fwd_stats(const void* y, const float* w, void* z, float* part, double* sums, int B, int H, int W, int Hp,
                         int Wp, int C, void* stream);
int esvit_dwbn_fwd_apply(const void* z, const float* gamma, const float* beta, const double* sums, float* run_mean,
                         float* run_var, long long* nbt, float* stat, void* out, long long N, int C, int train,
                         float momentum, float eps, void* stream);
int esvit_dwbn_bwd_stats(const void* dy, const void* z, const float* stat, float* part, double* sums, float* dgamma,
                         float* dbeta, long long N, int C, void* stream);
int esvit_dwbn_bwd_apply(const void* dy, const void* z, const void* y, const float* w, const float* stat,
                         const double* sums, float* coef, void* dx, float* part, float* dw, int B, int H, int W, int Hp,
                         int Wp, int C, int train, void* stream);

/* ---- DINOHead(use_bn=True) (models/vision_transformer.py:389-397): Linear -> BatchNorm1d -> exact GELU ------------------
 * z bf16 [N, C] is the bias-GEMM output, C % 64 == 0.  The statistics, running-statistics and coefficient arithmetic is
 * the dwbn_* one.  fwd_stats: sums fp64 [2C + 1] = (sum z, sum z^2, count N).  fwd_apply: stat fp32 [4C] as dwbn_fwd_apply
 * (train: run_mean / run_var / nbt updated in place when given; train = 0: the running statistics), out bf16 [N, C] =
 * gelu(z * stat[2] + stat[3]).  bwd_stats: with dh = dy gelu'(z * stat[2] + stat[3]), sums fp64 [2C + 1] = (sum dh,
 * sum dh xhat, count); dbeta / dgamma fp32 [C] += the local sums.  bwd_apply: dz bf16 [N, C] (written) = the BN input
 * gradient, dbias fp32 [C] += column sums of dz; coef fp32 [3C] scratch.  part: fp32 scratch of ceil(N / 256) * 2 * C
 * floats.  A SyncBatchNorm all-reduces `sums` between *_stats and *_apply.  No floating-point atomics. */
int esvit_headbn_fwd_stats(const void* z, float* part, double* sums, long long N, int C, void* stream);
int esvit_headbn_fwd_apply(const void* z, const float* gamma, const float* beta, const double* sums, float* run_mean,
                           float* run_var, long long* nbt, float* stat, void* out, long long N, int C, int train,
                           float momentum, float eps, void* stream);
int esvit_headbn_bwd_stats(const void* dy, const void* z, const float* stat, float* part, double* sums, float* dgamma,
                           float* dbeta, long long N, int C, void* stream);
int esvit_headbn_bwd_apply(const void* dy, const void* z, const float* stat, const double* sums, float* coef, void* dz,
                           float* part, float* dbias, long long N, int C, int train, void* stream);

/* ---- Vision Longformer (layers/longformer2d.py Long2DSCSelfAttention, W = 7, one global token, head dim 32) --------
 * Per image N = 1 + nx*ny token rows, row 0 the global token: q bf16 [B*N, C] (unscaled), kv bf16 [B*N, 2C] as [k|v],
 * out / dout / dq bf16 [B*N, C], dkv bf16 [B*N, 2C]; C = 32 nH.  mode int32 [1] in device memory: 0 = all nine
 * neighbour chunks, 1..8 = the own chunk and the reference's mode_dict chunk, -1 = the own chunk only; a value outside
 * -1..8 is clamped into that range.  bias / dbias fp32 [nH, 49, 442] (column
 * 0: local -> global, 1 + j*49 + r: key r of neighbour chunk j; columns of chunks the mode skips are not read and their
 * gradient is 0); bias_g / dbias_g fp32 [nH, N] (the global row).  lse / dvec fp32 [B, nH, chunks, 49], lse_g fp32 [B,
 * nH]; ws fp32 scratch of esvit_vil_sc_ws_floats(B, nx, ny, nH) elements.  dbias / dbias_g are written.  No
 * floating-point atomics. */
int esvit_vil_sc_ws_floats(int B, int nx, int ny, int nH);
int esvit_vil_sc_fwd(const void* q, const void* kv, const float* bias, const float* bias_g, const int* mode, void* out,
                     float* lse, float* lse_g, int B, int nx, int ny, int nH, float scale, void* stream);
int esvit_vil_sc_bwd(const void* q, const void* kv, const float* bias, const float* bias_g, const int* mode,
                     const void* out, const void* dout, const float* lse, const float* lse_g, float* dvec, float* ws,
                     void* dq, void* dkv, float* dbias, float* dbias_g, int B, int nx, int ny, int nH, float scale,
                     void* stream);

/* ---- Vision Longformer dense stages, embedding and bias assembly (vil_dense.cu) ------------------------------------
 * vil_dense_fwd / _bwd: multi-head attention at head dim 32 with an additive fp32 bias [nH, L, L] (vision_longformer.py
 *   Attention.forward :86-131), L <= 256.  qkv / dqkv bf16 [B*L, 3C] ([q|k|v][head][32]), out / dout bf16 [B*L, C],
 *   lse / dvec fp32 [B, nH, L], part fp32 scratch [esvit_vil_dense_parts(B), nH, L, L]; dbias fp32 [nH, L, L] is written
 *   (sum over the images of dS, fixed order).  No floating-point atomics.
 * vil_im2col: rows bf16 [B*(H/p)*(W/p), Kp] of the p x p / p conv over per-image token rows x fp32 [B*N, Cin] whose
 *   H*W map rows start at row off of each image (the global rows skipped); column c*p*p + ky*p + kx.  col2im: dx fp32
 *   [B*N, Cin] fully written (0 on the global rows).
 * vil_cls_cat_fwd: out fp32 [B*(1+n), C] = per image cat(cls [C], y rows [n, C]).  _bwd: dy = the patch rows of g;
 *   dcls (+)= sum over the images of the global rows of g (accumulate != 0 adds to dcls).  C % 4 == 0.
 * vil_bias_spmv: y[r] = sum_k val[k] * src(col[k]) over k in [rowptr[r], rowptr[r+1]) in order (CSR, int32), with
 *   src(c) = s0[c] for c < n0, s1[c - n0] for c < n0 + n1, else s2[c - n0 - n1].  The relative-position bias gathers and
 *   bicubic resizes, and their transposes (fixed-order gather-sums), are such maps. */
int esvit_vil_dense_parts(int B);
int esvit_vil_dense_fwd(const void* qkv, const float* bias, void* out, float* lse, int B, int L, int C, int nH,
                        float scale, void* stream);
int esvit_vil_dense_bwd(const void* qkv, const float* bias, const void* out, const void* dout, const float* lse,
                        float* dvec, float* part, void* dqkv, float* dbias, int B, int L, int C, int nH, float scale,
                        void* stream);
int esvit_vil_im2col(const float* x, void* rows, int B, int N, int off, int Cin, int H, int W, int p, int Kp,
                     void* stream);
int esvit_vil_col2im(const void* drows, float* dx, int B, int N, int off, int Cin, int H, int W, int p, int Kp,
                     void* stream);
int esvit_vil_cls_cat_fwd(const float* y, const float* cls, float* out, int B, int n, int C, void* stream);
int esvit_vil_cls_cat_bwd(const float* g, float* dy, float* dcls, int B, int n, int C, int accumulate, void* stream);
int esvit_vil_bias_spmv(const int* rowptr, const int* col, const float* val, const float* s0, const float* s1,
                        const float* s2, int n0, int n1, float* y, int nrows, void* stream);

/* ---- optimiser-side multi-tensor kernels (host arrays of device pointers) ----------------------------------
 * ema_multi: teacher = teacher*m + student*(1-m), bit-exact with main_esvit.py:587-590.
 * clip_multi: per-tensor L2 clip of utils.py:106-115; sumsq_ws double[n] workspace; norms fp32[n] or NULL. */
int esvit_ema_multi(void* const* teacher, const void* const* student, const long long* numel, int n, double momentum,
                    void* stream);
int esvit_clip_multi(void* const* grads, const long long* numel, int n, float clip, double* sumsq_ws, float* norms,
                     void* stream);
/* Fused optimiser pass, CUDA-graph friendly (every step-varying scalar is read from device memory):
 * grad_sumsq_multi: sumsq[i] = ||grads[i]||^2 (double[n], zeroed inside).
 * adamw_ema_multi: per-tensor clip (utils.py:106-115) folded into torch.optim.AdamW's update (main_esvit.py:411) and the
 *   teacher EMA (main_esvit.py:587-590, bit-exact two-rounding form) in one sweep.
 *   hyper fp32[8] = {lr, wd(group 0), beta1, beta2, eps, ema_m, 1-ema_m, clip(<=0: off)};
 *   state fp32[2n] = per tensor {step count, flags: bit0 weight-decayed, bit1 skip (= reference's p.grad=None)};
 *   teacher may be NULL; param_bf16 / teacher_bf16 (arrays or entries may be NULL) receive bf16 copies of the updated
 *   values = the GEMM operands of the next step, so no per-step cast kernels are needed. */
int esvit_grad_sumsq_multi(void* const* grads, const long long* numel, int n, double* sumsq, void* stream);
int esvit_adamw_ema_multi(void* const* params, const void* const* grads, void* const* exp_avg, void* const* exp_avg_sq,
                          void* const* teacher, void* const* param_bf16, void* const* teacher_bf16,
                          const long long* numel, int n, const float* hyper, float* state, const double* sumsq,
                          void* stream);
/* SGD-momentum / LARS counterpart of adamw_ema_multi (main_esvit.py:412-415), same conventions:
 * lars_sums_multi: sums double[3n] (zeroed inside), planar {sum g^2 | sum p^2 | sum g*p}; params (array or entries) may
 *   be NULL, then only sum g^2 of that tensor is formed.  SGD uses grad_sumsq_multi instead.
 * sgd_ema_multi: per-tensor clip, coupled weight decay d = c*g + wd*p, LARS trust ratio, momentum buffer
 *   buf = momentum*buf + d (torch.optim.SGD dampening 0 / utils.LARS mu), p -= lr*buf, teacher EMA, bf16 shadows.
 *   hyper fp32[8] = {lr, wd(group 0), momentum, eta, ema_m, 1-ema_m, clip(<=0: off), unused};
 *   state fp32[2n] = per tensor {steps taken, flags: bit0 weight-decayed, bit1 skip, bit2 LARS trust ratio (p.dim()!=1)};
 *   sums = grad_sumsq_multi's double[n], or lars_sums_multi's double[3n] when any bit2 is set. */
int esvit_lars_sums_multi(const void* const* grads, const void* const* params, const long long* numel, int n,
                          double* sums, void* stream);
int esvit_sgd_ema_multi(void* const* params, const void* const* grads, void* const* momentum_buf, void* const* teacher,
                        void* const* param_bf16, void* const* teacher_bf16, const long long* numel, int n,
                        const float* hyper, float* state, const double* sums, void* stream);

/* ---- exact weighted k-NN classifier over frozen features ---------------------------------------- eval_knn.py:193-232
 * knn_prep: xb bf16 [R_pad, D] = bf16(x fp32 [R, D]) with rows >= R zero; norm fp32 [R] = ||x_r||; max_norm fp32 [1]
 *   ACCUMULATED as the maximum norm (integer atomicMax on its bit pattern; caller zero-fills).  D % 8 == 0.
 * knn_select: per test row r (rows int32 [nrows] or NULL = rows 0..nrows-1): S bf16 [., ld] = a . b^T from
 *   esvit_gemm_bf16; a fp32 [., D] test rows with norms a_norm; b fp32 [N, D] train rows with max norm max_norm[0].
 *   Finds the k-th largest bf16 value tau of S[r, 0:N], collects the columns with S >= tau - 2 delta_r
 *   (delta_r = (3u + 4u^2 + D 2^-23) a_norm[r] max_norm, u = 2^-8) into cand_idx / cand_val [nrows, cap] (scratch),
 *   rescores them in fp32 and writes the exact fp32 top-k by (value desc, index asc) to sims fp32 [., k] and idx int64
 *   [., k].  count int32 [.] receives the candidate count; rows with count > cap are not written (rerun with cap >= count).
 * knn_vote: per test row, scores[c] = sum of exp(sims / T) over the neighbours of train class c (rank order); hits int64
 *   [2] ACCUMULATES (top-1, top-5) hits of test_labels by (score desc, class asc).  num_classes <= 11264. */
int esvit_knn_prep(const float* x, void* xb, float* norm, float* max_norm, long long R, long long R_pad, int D,
                   void* stream);
int esvit_knn_select(const void* S, long long ld, const float* a, const float* b, const float* a_norm,
                     const float* max_norm, const int* rows, int nrows, int N, int D, int k, int cap, int* cand_idx,
                     float* cand_val, int* count, float* sims, long long* idx, void* stream);
int esvit_knn_vote(const float* sims, const long long* idx, const long long* train_labels, const long long* test_labels,
                   long long M, int k, float T, int num_classes, long long* hits, void* stream);

/* ---- multi-crop augmentation (DataAugmentationDINO) on decoded uint8 images ---------------- datasets/build.py:203-261
 * Pillow's arithmetic for RandomResizedCrop(bicubic) / hflip / ColorJitter / RandomGrayscale / ImageFilter.GaussianBlur /
 * ImageOps.solarize, then ToTensor + Normalize, for every crop of a batch (esvit_b200/augment.py builds the arguments).
 * params fp64 [ncrops, 18] (augment.PARAM_FIELDS); meta int64 [ncrops, 9]: source byte offset into src (uint8 HWC), source
 * H, W, output size S, byte offset into tmp (uint8 [h, S, 3] per crop), int32 offset into coef (S * (4 + kh + kv) per
 * crop), horizontal / vertical tap counts kh = 2 ceil(2 max(1, w / S)) + 1 and kv (same with h), fp32 output address of
 * the crop's [3, S, S].  Every offset is 64-bit.
 * coeffs: both axes' bounds and 22-bit fixed-point bicubic coefficients of every crop into coef; max_S = max S.
 * resize_h: the horizontal pass of every box row (flip applied) into tmp; max_pixels = max over crops of h * S.
 * color: crops [crop0, crop0 + ncrops), all of output size S <= 241: vertical pass, colour ops, blur, solarize, normalize
 *   with norm fp32 [6] = (mean[3], std[3]); the fp32 crop is written with streaming stores. */
int esvit_augment_coeffs(const double* params, const long long* meta, int* coef, int ncrops, int max_S, void* stream);
int esvit_augment_resize_h(const unsigned char* src, const double* params, const long long* meta, const int* coef,
                           unsigned char* tmp, int ncrops, long long max_pixels, void* stream);
int esvit_augment_color(const double* params, const long long* meta, const int* coef, const unsigned char* tmp,
                        const float* norm, int crop0, int ncrops, int S, void* stream);

/* ---- evaluation transforms on decoded uint8 images ---------------------------- eval_linear.py:50-61, eval_knn.py:48-53
 * RandomResizedCrop(224, bilinear) + RandomHorizontalFlip, or Resize(256, bicubic) + CenterCrop(224), then ToTensor +
 * Normalize, with Pillow's arithmetic, for one crop per image (esvit_b200/augment.py EvalAugment builds the arguments).
 * Each image's crop box is resized to (rh, rw) and only the S x S output window at (oy, ox) is computed.
 * rec fp64 [nimg, 11] (augment.EVAL_FIELDS: box top, left, h, w, rh, rw, oy, ox, S, flip, Pillow resample code 2 / 3);
 * meta int64 [nimg, 8]: source byte offset into src (uint8 HWC), source W, first box row y0 the window's vertical taps
 * read and their row count, byte offset into tmp (uint8 [rows, S, 3] per image), int32 offset into coef
 * (S * (4 + kh + kv) per image), horizontal / vertical tap counts kh = 2 ceil(support * max(1, w / rw)) + 1 and kv
 * (same with h / rh), support 1 (bilinear) or 2 (bicubic).
 * eval_coeffs: both axes' window bounds and 22-bit fixed-point coefficients into coef.
 * eval_resize_h: the horizontal pass (flip applied) of box rows [y0, y0 + rows) into tmp; max_pixels = max rows * S.
 * eval_resize_v: the vertical pass, ToTensor + Normalize with norm fp32 [6] = (mean[3], std[3]) into out fp32
 *   [nimg, 3, S, S], S^2 < 2^31. */
int esvit_augment_eval_coeffs(const double* rec, const long long* meta, int* coef, int nimg, int S, void* stream);
int esvit_augment_eval_resize_h(const unsigned char* src, const double* rec, const long long* meta, const int* coef,
                                unsigned char* tmp, int nimg, int S, long long max_pixels, void* stream);
int esvit_augment_eval_resize_v(const long long* meta, const int* coef, const unsigned char* tmp, const float* norm,
                                float* out, int nimg, int S, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ESVIT_B200_H */
