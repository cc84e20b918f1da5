"""nn.Linear layers of the training step on the wgmma GEMM family (csrc/gemm2_wgmma.cu).

Every GEMM of a Linear - forward, input gradient, weight gradient - is one esvit_b200 kernel:

  forward          y  = x . W^T + b            esvit_gemm_bf16   (A, B K-major; bias / GELU epilogue)
  input gradient   dx = dy . W                 esvit_gemm_bf16   (B = W [out, in] read AS IT LIES, MN-major)
  weight gradient  dW = dy^T . x   (fp32)      esvit_gemm_wgrad  (A = dy, B = x read as they lie, both MN-major; split-K
                                                                  partials folded deterministically)

so there are no transposed weight copies, no bf16 -> fp32 gradient cast kernels and no library split-K reductions.  The
fp32 weight gradient goes straight to the fp32 master parameter; bias gradients are produced by the CONSUMER kernel of the
layer's output (window attention / residual add + LN / GELU-backward epilogue), see LinearFn.

Reference: Mlp / WindowAttention.qkv / .proj / PatchMerging.reduction (models/swin_transformer.py:21-37, 88-91, 125, 150,
393-420) and DINOHead (models/vision_transformer.py:385-418)."""
from __future__ import annotations

from typing import Optional

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import ops

Tensor = torch.Tensor
BF16 = torch.bfloat16
F32 = torch.float32


def _wgrad(key, dy2: Tensor, x2: Tensor, shape):
    """fp32 weight gradient; several calls for the same weight inside one backward (the per-resolution-group loop)
    accumulate into the first call's buffer and only the first hands it to autograd (cf. ops._acc)."""
    d = ops._Arena.accs
    if d is None:
        return ops.gemm_wgrad(dy2, x2).view(shape)
    buf = d.get(key)
    if buf is not None and tuple(buf.shape) == tuple(shape):
        ops.gemm_wgrad(dy2, x2, out=buf, accumulate=True)
        return None
    buf = d[key] = ops.gemm_wgrad(dy2, x2).view(shape)
    return buf.view(shape)


class LinearFn(Function):
    """y = x @ W^T (+ b).  wp: the fp32 master weight (receives the fp32 gradient), w16: its bf16 copy (GEMM operand),
    bias: fp32 [N] or None - added in the GEMM epilogue; its GRADIENT is left to the consumer kernel."""

    @staticmethod
    def forward(ctx, x, wp, w16, bias):
        y = ops.gemm(x, w16, bias)
        ctx.save_for_backward(x, w16)
        ctx.wkey = ("w", wp.data_ptr())
        ctx.wshape = tuple(wp.shape)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w16 = ctx.saved_tensors
        g = ops._chk(g, BF16, "g")
        N, K = w16.shape
        g2 = g.reshape(-1, N)
        dx = ops.gemm(g2, w16, None, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = _wgrad(ctx.wkey, g2, x.reshape(-1, K), ctx.wshape) if ctx.needs_input_grad[1] else None
        return dx, dw, None, None


class LinearColsumFn(LinearFn):
    """LinearFn whose bias gradient is the column sums of dy (ops.colsum), for a Linear whose consumer kernel does not
    produce it: the last Linear of DINOHead(use_bn=True), read by the row L2 normalisation."""

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        dx, dw, _, _ = LinearFn.backward(ctx, g)
        db = ops.colsum(g.reshape(-1, g.shape[-1]).contiguous()) if ctx.needs_input_grad[3] else None
        return dx, dw, None, db


class MlpFn(Function):
    """fc2(gelu(fc1(x))) (models/swin_transformer.py:31-35).  forward at C in ops.MLP_FUSED_C (Swin stages 0-1): ONE
    back-to-back kernel (esvit_mlp_fwd) writes y and, when a gradient is needed, h and gelu'; at other C: h, gelu' from ONE
    GEMM (bias + exact GELU epilogue), y = h . W2^T + b2.  act 2 (CvT's QuickGELU FeedForward) always takes the two-GEMM
    path with the QuickGELU epilogue; its derivative is the stored multiplier, so the backward is the same.  backward: d(pre) = (dy . W2) * gelu' with the fc1 bias gradient
    as column sums, all in one GEMM epilogue; dx = d(pre) . W1; dW1, dW2 in fp32.  b2's gradient is produced by the consumer (residual add + LN backward)."""

    @staticmethod
    def forward(ctx, x, w1p, w1, b1, w2p, w2, b2, act: int = 1):
        need = any(ctx.needs_input_grad)  # (grad mode is always off inside Function.forward: needs_input_grad is the signal)
        C = x.shape[-1]
        if act == 1 and C in ops.MLP_FUSED_C and w1.shape[0] == 4 * C:
            # one back-to-back kernel: h goes to HBM only when the backward needs it, and is never read back here
            if need:
                y, h, pre = ops.mlp_fwd(x, w1, b1, w2, b2, want_h=True)
            else:
                y, h, pre = ops.mlp_fwd(x, w1, b1, w2, b2), None, None
        else:
            if need:
                h, pre = ops.gemm(x, w1, b1, act=act, want_pre=True)
            else:
                h, pre = ops.gemm(x, w1, b1, act=act), None
            y = ops.gemm(h, w2, b2)
        ctx.save_for_backward(x, w1, w2, pre, h)
        ctx.keys = (("w", w1p.data_ptr()), tuple(w1p.shape), ("w", w2p.data_ptr()), tuple(w2p.shape))
        ctx.bias_meta = (b1.shape, b1.device, b1.data_ptr())
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w1, w2, pre, h = ctx.saved_tensors
        k1, s1, k2, s2 = ctx.keys
        g = ops._chk(g, BF16, "g")
        Cc, Nh = g.shape[-1], pre.shape[-1]
        g2 = g.reshape(-1, Cc)
        dw2 = _wgrad(k2, g2, h.reshape(-1, Nh), s2) if ctx.needs_input_grad[4] else None
        db1, first = ops._acc(("bias", ctx.bias_meta[2]), tuple(ctx.bias_meta[0]), ctx.bias_meta[1])
        dpre = ops.gemm_mul_colsum(g2, w2, pre.reshape(-1, Nh), db1, b_mn=True)      # W2 [C, 4C] read as it lies
        dx = ops.gemm(dpre, w1, None, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        dw1 = _wgrad(k1, dpre, x.reshape(-1, x.shape[-1]), s1) if ctx.needs_input_grad[1] else None
        return dx, dw1, None, (db1 if first else None), dw2, None, None, None


class HeadMlpFn(Function):
    """The MLP of DINOHead without BN (models/vision_transformer.py:385-403, 414-415): n >= 1 Linears with a GELU after
    every one but the last.  forward(x, wp_1, w16_1, b_1, ..., wp_n, w16_n, b_n) (master weight, its bf16 copy, bias per
    layer): every GELU in its GEMM's epilogue, and every GELU backward (+ its bias gradient) in the next layer's
    input-gradient GEMM epilogue.  At n = 1 this computes what LinearColsumFn computes."""

    @staticmethod
    def forward(ctx, x, *params):
        need = any(ctx.needs_input_grad)  # (grad mode is always off inside Function.forward: needs_input_grad is the signal)
        ws, bs = params[1::3], params[2::3]
        hs, pres = [x], []
        for w, b in zip(ws[:-1], bs[:-1]):
            if need:
                h, p = ops.gemm(hs[-1], w, b, act=1, want_pre=True)
            else:
                h, p = ops.gemm(hs[-1], w, b, act=1), None
            hs.append(h)
            pres.append(p)
        y = ops.gemm(hs[-1], ws[-1], bs[-1])
        ctx.save_for_backward(*hs, *ws, *pres)
        ctx.shapes = [tuple(wp.shape) for wp in params[0::3]]
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        n = len(ctx.shapes)
        saved = ctx.saved_tensors
        hs, ws, pres = saved[:n], saved[n:2 * n], saved[2 * n:]
        g = ops._chk(g, BF16, "g")
        d = g.reshape(-1, g.shape[-1])
        grads = [None] * (3 * n)   # (dW, None, db) per layer
        db = ops.colsum(d)
        for i in reversed(range(n)):
            grads[3 * i] = ops.gemm_wgrad(d, hs[i].reshape(-1, hs[i].shape[-1])).view(ctx.shapes[i])
            grads[3 * i + 2] = db
            if i:
                db = torch.zeros(ctx.shapes[i - 1][0], dtype=F32, device=g.device)
                d = ops.gemm_mul_colsum(d, ws[i], pres[i - 1].reshape(-1, pres[i - 1].shape[-1]), db, b_mn=True)
        dx = ops.gemm(d, ws[0], None, b_mn=True).view(hs[0].shape) if ctx.needs_input_grad[0] else None
        return (dx, *grads)


class LastLayerFn(Function):
    """logits = x @ W_eff^T with W_eff = weight_norm(v, g) in bf16 [K, D] (models/vision_transformer.py:404-417).
    backward: dx = dlogits . W_eff (MN-major B, contraction over the 65536 prototypes), dW_eff = dlogits^T . x in fp32."""

    @staticmethod
    def forward(ctx, x, w_eff):
        y = ops.gemm(x, w_eff, None)
        ctx.save_for_backward(x, w_eff)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        g = ops._chk(g, BF16, "g")
        Kp, Dm = w.shape
        g2 = g.reshape(-1, Kp)
        dx = ops.gemm(g2, w, None, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = ops.gemm_wgrad(g2, x.reshape(-1, Dm)).view(Kp, Dm) if ctx.needs_input_grad[1] else None
        return dx, dw
