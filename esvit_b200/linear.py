"""nn.Linear layers of the training step on the wgmma GEMM family (csrc/gemm2_wgmma.cu).

Every GEMM of a Linear - forward, input gradient, weight gradient - is one esvit_b200 kernel:

  forward          y  = x . W^T + b            esvit_gemm_bf16   (A, B K-major; bias / GELU epilogue)
  input gradient   dx = dy . W                 esvit_gemm_bf16   (B = W [out, in] read AS IT LIES, MN-major)
  weight gradient  dW = dy^T . x   (fp32)      esvit_gemm_wgrad  (A = dy, B = x read as they lie, both MN-major; split-K
                                                                  partials folded deterministically)

so there are no transposed weight copies, no bf16 -> fp32 gradient cast kernels and no library split-K reductions.  The
fp32 weight gradient goes straight to the fp32 master parameter; bias gradients are produced by the CONSUMER kernel of the
layer's output (window attention / residual add + LN / GELU-backward epilogue), see ops.LinearBiasFn.

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


class MlpFn(Function):
    """fc2(gelu(fc1(x))) (models/swin_transformer.py:31-35).  forward: h, gelu' from ONE GEMM (bias + exact GELU epilogue),
    y = h . W2^T + b2.  backward: d(pre) = (dy . W2) * gelu' with the fc1 bias gradient as column sums, all in one GEMM
    epilogue; dx = d(pre) . W1; dW1, dW2 in fp32.  b2's gradient is produced by the consumer (residual add + LN backward)."""

    @staticmethod
    def forward(ctx, x, w1p, w1, b1, w2p, w2, b2):
        need = any(ctx.needs_input_grad)  # (grad mode is always off inside Function.forward: needs_input_grad is the signal)
        if need:
            h, pre = ops.gemm(x, w1, b1, act=1, want_pre=True)
        else:
            h, pre = ops.gemm(x, w1, b1, act=1), None
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
        return dx, dw1, None, (db1 if first else None), dw2, None, None


class HeadMlpFn(Function):
    """The 3-layer MLP of DINOHead (models/vision_transformer.py:385-403, 414-415): Linear-GELU-Linear-GELU-Linear, with
    both GELUs in GEMM epilogues and both GELU backwards (+ their bias gradients) in the next layer's input-gradient
    GEMM epilogue."""

    @staticmethod
    def forward(ctx, x, w1p, w1, b1, w2p, w2, b2, w3p, w3, b3):
        need = any(ctx.needs_input_grad)  # (grad mode is always off inside Function.forward: needs_input_grad is the signal)
        if need:
            h1, p1 = ops.gemm(x, w1, b1, act=1, want_pre=True)
            h2, p2 = ops.gemm(h1, w2, b2, act=1, want_pre=True)
        else:
            h1, p1 = ops.gemm(x, w1, b1, act=1), None
            h2, p2 = ops.gemm(h1, w2, b2, act=1), None
        y = ops.gemm(h2, w3, b3)
        ctx.save_for_backward(x, w1, w2, w3, h1, p1, h2, p2)
        ctx.shapes = (tuple(w1p.shape), tuple(w2p.shape), tuple(w3p.shape))
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w1, w2, w3, h1, p1, h2, p2 = ctx.saved_tensors
        s1, s2, s3 = ctx.shapes
        g = ops._chk(g, BF16, "g")
        g3 = g.reshape(-1, g.shape[-1])
        dev = g.device
        db3 = ops.colsum(g3)
        dw3 = ops.gemm_wgrad(g3, h2.reshape(-1, h2.shape[-1])).view(s3)
        db2 = torch.zeros(s2[0], dtype=F32, device=dev)
        d2 = ops.gemm_mul_colsum(g3, w3, p2.reshape(-1, p2.shape[-1]), db2, b_mn=True)
        dw2 = ops.gemm_wgrad(d2, h1.reshape(-1, h1.shape[-1])).view(s2)
        db1 = torch.zeros(s1[0], dtype=F32, device=dev)
        d1 = ops.gemm_mul_colsum(d2, w2, p1.reshape(-1, p1.shape[-1]), db1, b_mn=True)
        dw1 = ops.gemm_wgrad(d1, x.reshape(-1, x.shape[-1])).view(s1)
        dx = ops.gemm(d1, w1, None, b_mn=True).view(x.shape) if ctx.needs_input_grad[0] else None
        return dx, dw1, None, db1, dw2, None, db2, dw3, None, db3


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
