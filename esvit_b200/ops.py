"""torch.autograd.Function wrappers over the esvit_b200 C ABI (one entry point per kernel).

PyTorch is used here for device memory (caching allocator), the current CUDA stream and autograd bookkeeping;
all arithmetic of these ops happens in the hand-written sm_90a kernels.  There is no fallback path: every op
requires CUDA tensors and the built library.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib, shadow

Tensor = torch.Tensor
BF16 = torch.bfloat16
F32 = torch.float32


def _p(t: Optional[Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _po(t: Tensor, off_elems: int):
    """pointer to element `off_elems` of a contiguous tensor (one resolution group inside a concatenated buffer)"""
    return ctypes.c_void_p(t.data_ptr() + off_elems * t.element_size())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Arena:
    """One zero-filled fp32 buffer per training step from which the backward kernels' small ACCUMULATED outputs
    (dgamma / dbeta / bias gradients / rel-pos-table gradients) are carved: one memset per step instead of ~340 tiny
    fill kernels.  Regions are never handed out twice, so a stale arena is still correct (just smaller)."""
    buf: Optional[Tensor] = None
    off = 0
    accs: Optional[dict] = None  # live only between begin_step() and end_step(): parameter -> its accumulator
    warned = False


def begin_step(device, nfloats: int = 1 << 22) -> None:
    """Call right before ONE backward() (engine.SelfDistillStep does), end_step() right after; optional - without it
    ops fall back to torch.zeros per accumulator."""
    _Arena.buf = torch.zeros(nfloats, dtype=F32, device=device)
    _Arena.off = 0
    _Arena.accs = {}


def end_step() -> None:
    _Arena.accs = None


def _acc(key, shape, device) -> Tuple[Tensor, bool]:
    """Accumulated-gradient buffer of one parameter for THIS backward pass -> (buffer, first).  The backbone runs once per
    resolution group (global / local crops) through the same weights; both backward kernels += into the same
    zero-filled buffer and only the first call hands it to autograd (later calls return None for that input), so no
    separate gradient-accumulation kernels run.  Valid because autograd holds the first tensor by reference until every
    contribution to the leaf has been produced, and the kernels are ordered on one stream.  Outside
    begin_step()/end_step() every call gets a fresh buffer."""
    d = _Arena.accs
    if d is None:
        return _zeros(shape, device), True
    t = d.get(key)
    if t is not None and tuple(t.shape) == tuple(shape):
        return t, False
    t = d[key] = _zeros(shape, device)
    return t.view(t.shape), True  # a fresh alias: autograd adopts it as .grad instead of cloning (sole reference)


def _zeros(shape, device) -> Tensor:
    n = 1
    for d in shape:
        n *= int(d)
    buf = _Arena.buf
    n16 = (n + 3) & ~3  # keep every region 16-byte aligned (vectorised optimiser reads)
    if buf is not None and buf.device == torch.device(device) and _Arena.off + n16 <= buf.numel():
        v = buf[_Arena.off:_Arena.off + n].view(*shape)
        _Arena.off += n16
        return v
    if buf is not None and not _Arena.warned:
        _Arena.warned = True
        import warnings
        warnings.warn("esvit_b200: gradient-accumulator arena exhausted (%d floats); falling back to per-tensor torch.zeros - "
                      "pass a larger nfloats to ops.begin_step" % buf.numel())
    return torch.zeros(*shape, dtype=F32, device=device)


def _chk(t: Optional[Tensor], dtype, name: str) -> Optional[Tensor]:
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"esvit_b200 op input `{name}` must be a CUDA tensor (no CPU fallback exists)")
    if t.dtype != dtype:
        raise TypeError(f"`{name}` must be {dtype}, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------------------------
# residual add + LayerNorm


def _add_ln_fwd(x, delta, keep, tps, gamma, beta, eps, want_y, y_bf16):
    ref = x if x is not None else delta  # x = None: xout = fp32(delta), the start of a residual stream
    T, C = ref.numel() // ref.shape[-1], ref.shape[-1]
    xout = torch.empty(ref.shape, dtype=F32, device=ref.device) if delta is not None else None
    y = mean = rstd = None
    if want_y:
        y = torch.empty(ref.shape, dtype=BF16 if y_bf16 else F32, device=ref.device)
        mean = torch.empty(T, dtype=F32, device=ref.device)
        rstd = torch.empty(T, dtype=F32, device=ref.device)
    _lib.call("esvit_add_ln_fwd", _p(x), _p(delta), _p(keep), tps, _p(gamma), _p(beta), eps, _p(xout), _p(y),
              1 if y_bf16 else 0, _p(mean), _p(rstd), T, C, _stream())
    return (xout if delta is not None else x), y, mean, rstd


class AddLayerNormFn(Function):
    """(x, delta, delta_bias, keep) -> (xout = x + keep*delta, y = LN(xout)).
    keep: per-sample DropPath scale or None.  delta_bias (fp32 [C] parameter or None) is the bias the producing GEMM
    already added to delta in its epilogue: it is only routed here so that ITS GRADIENT (column sums of ddelta) comes
    out of this backward kernel instead of a separate reduction."""

    @staticmethod
    def forward(ctx, x, delta, dbias, keep, gamma, beta, eps: float, y_bf16: bool):
        x = _chk(x, F32, "x")
        delta = _chk(delta, BF16, "delta")
        dbias = _chk(dbias, F32, "delta_bias")
        keep = _chk(keep, F32, "keep")
        gamma, beta = _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        ref = x if x is not None else delta  # x = None: the stream starts here as fp32(delta) (after PatchMerging)
        tps = ref.numel() // ref.shape[-1] // ref.shape[0]
        xout, y, mean, rstd = _add_ln_fwd(x, delta, keep, tps, gamma, beta, eps, True, y_bf16)
        ctx.save_for_backward(xout, mean, rstd, gamma, keep)
        ctx.tps, ctx.y_bf16, ctx.has_dbias, ctx.has_x = tps, y_bf16, dbias is not None, x is not None
        return xout, y

    @staticmethod
    @once_differentiable
    def backward(ctx, g_xout, g_y):
        xout, mean, rstd, gamma, keep = ctx.saved_tensors
        T, C = xout.numel() // xout.shape[-1], xout.shape[-1]
        g_xout = _chk(g_xout, F32, "g_xout") if g_xout is not None else None
        if g_y is not None:
            g_y = _chk(g_y, BF16 if ctx.y_bf16 else F32, "g_y")
        dx = torch.empty_like(xout) if ctx.has_x else None
        ddelta = torch.empty(xout.shape, dtype=BF16, device=xout.device)
        acc, first = _acc(("add_ln", gamma.data_ptr()), (3, C), xout.device)  # dgamma | dbeta | ddelta_bias
        _lib.call("esvit_add_ln_bwd", _p(g_y), 1 if ctx.y_bf16 else 0, _p(g_xout), _p(xout), _p(mean), _p(rstd),
                  _p(gamma), _p(keep), ctx.tps, _p(dx), _p(ddelta), _p(acc[0]), _p(acc[1]),
                  _p(acc[2]) if ctx.has_dbias else None, T, C, _stream())
        if not first:
            return dx, ddelta, None, None, None, None, None, None
        return dx, ddelta, (acc[2] if ctx.has_dbias else None), None, acc[0], acc[1], None, None


class LayerNormFn(Function):
    """x fp32 -> y = LN(x) (bf16 or fp32)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps: float, y_bf16: bool):
        x = _chk(x, F32, "x")
        gamma, beta = _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        _, y, mean, rstd = _add_ln_fwd(x, None, None, 1, gamma, beta, eps, True, y_bf16)
        ctx.save_for_backward(x, mean, rstd, gamma)
        ctx.y_bf16 = y_bf16
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g_y):
        x, mean, rstd, gamma = ctx.saved_tensors
        T, C = x.numel() // x.shape[-1], x.shape[-1]
        g_y = _chk(g_y, BF16 if ctx.y_bf16 else F32, "g_y")
        dx = torch.empty_like(x)
        acc, first = _acc(("ln", gamma.data_ptr()), (2, C), x.device)
        _lib.call("esvit_add_ln_bwd", _p(g_y), 1 if ctx.y_bf16 else 0, None, _p(x), _p(mean), _p(rstd), _p(gamma),
                  None, 1, _p(dx), None, _p(acc[0]), _p(acc[1]), None, T, C, _stream())
        return (dx, acc[0], acc[1], None, None) if first else (dx, None, None, None, None)


class LayerNormResidFn(Function):
    """x fp32 -> (x, y = LN(x)): the start of a residual stream whose input is also the shortcut (the first block after
    PatchEmbed).  Handing x out as an OUTPUT makes autograd deliver the shortcut's gradient to this backward, where the
    add_ln backward kernel adds it to the LN input gradient (dxo) - otherwise x has two consumers and autograd sums the
    two full-size fp32 gradients with a separate add kernel (112 us for Swin-T at B = 64)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps: float, y_bf16: bool):
        x = _chk(x, F32, "x")
        gamma, beta = _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        _, y, mean, rstd = _add_ln_fwd(x, None, None, 1, gamma, beta, eps, True, y_bf16)
        ctx.save_for_backward(x, mean, rstd, gamma)
        ctx.y_bf16 = y_bf16
        return x.view(x.shape), y

    @staticmethod
    @once_differentiable
    def backward(ctx, g_x, g_y):
        x, mean, rstd, gamma = ctx.saved_tensors
        T, C = x.numel() // x.shape[-1], x.shape[-1]
        g_x = _chk(g_x, F32, "g_x") if g_x is not None else None
        if g_y is None:
            return g_x, None, None, None, None
        g_y = _chk(g_y, BF16 if ctx.y_bf16 else F32, "g_y")
        dx = torch.empty_like(x)
        acc, first = _acc(("ln", gamma.data_ptr()), (2, C), x.device)
        _lib.call("esvit_add_ln_bwd", _p(g_y), 1 if ctx.y_bf16 else 0, _p(g_x), _p(x), _p(mean), _p(rstd), _p(gamma),
                  None, 1, _p(dx), None, _p(acc[0]), _p(acc[1]), None, T, C, _stream())
        return (dx, acc[0], acc[1], None, None) if first else (dx, None, None, None, None)


class ResidualAddFn(Function):
    """xout = x + keep * delta (fp32 + bf16), no norm; delta_bias only receives its gradient (see AddLayerNormFn)."""

    @staticmethod
    def forward(ctx, x, delta, dbias, keep):
        x, delta, keep = _chk(x, F32, "x"), _chk(delta, BF16, "delta"), _chk(keep, F32, "keep")
        dbias = _chk(dbias, F32, "delta_bias")
        tps = x.numel() // x.shape[-1] // x.shape[0]
        xout, _, _, _ = _add_ln_fwd(x, delta, keep, tps, None, None, 0.0, False, False)
        ctx.save_for_backward(keep)
        ctx.tps, ctx.has_dbias = tps, dbias is not None
        ctx.dbias_ptr = dbias.data_ptr() if dbias is not None else 0
        return xout

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (keep,) = ctx.saved_tensors
        g = _chk(g, F32, "g")
        T, C = g.numel() // g.shape[-1], g.shape[-1]
        ddelta = torch.empty(g.shape, dtype=BF16, device=g.device)
        db, first = _acc(("res", ctx.dbias_ptr), (C,), g.device) if ctx.has_dbias else (None, True)
        _lib.call("esvit_add_ln_bwd", None, 0, _p(g), None, None, None, None, _p(keep), ctx.tps, None, _p(ddelta),
                  None, None, _p(db), T, C, _stream())
        return g, ddelta, (db if first else None), None


def add_layer_norm(x: Tensor, delta: Optional[Tensor], keep: Optional[Tensor], gamma: Tensor, beta: Tensor,
                   eps: float, y_bf16: bool = True, delta_bias: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    if delta is None:
        if x.requires_grad and torch.is_grad_enabled():
            return LayerNormResidFn.apply(x, gamma, beta, eps, y_bf16)
        return x, LayerNormFn.apply(x, gamma, beta, eps, y_bf16)
    return AddLayerNormFn.apply(x, delta, delta_bias, keep, gamma, beta, eps, y_bf16)  # x may be None: xout = fp32(delta)


def residual_add(x: Tensor, delta: Optional[Tensor], keep: Optional[Tensor],
                 delta_bias: Optional[Tensor] = None) -> Tensor:
    return x if delta is None else ResidualAddFn.apply(x, delta, delta_bias, keep)


# ------------------------------------------------------------------------------------------------------------
class PatchEmbedGroupsFn(Function):
    """imgs fp32 [B_g, 3, H_g, W_g], one per resolution group -> LN(conv4x4/4) of every group written into ONE token
    buffer fp32 [sum_g B_g (H_g/4)(W_g/4), E] (the concatenated residual stream of the Swin forward): no torch.cat of
    the groups' outputs (267 MB copied per step for Swin-T at B = 64) and no split of the gradient."""

    @staticmethod
    def forward(ctx, w, bias, gamma, beta, eps: float, *imgs):
        w, bias = _chk(w, F32, "w"), _chk(bias, F32, "bias")
        gamma, beta = _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        imgs = [_chk(im, F32, "img") for im in imgs]
        E = w.shape[0]
        if tuple(w.shape[1:]) != (3, 4, 4) or any(im.shape[1] != 3 for im in imgs):
            raise ValueError("PatchEmbed kernel supports in_chans=3, patch_size=4")
        rows = [im.shape[0] * (im.shape[2] // 4) * (im.shape[3] // 4) for im in imgs]
        T = sum(rows)
        dev = imgs[0].device
        out = torch.empty(T, E, dtype=F32, device=dev)
        mean = torch.empty(T, dtype=F32, device=dev)
        rstd = torch.empty(T, dtype=F32, device=dev)
        r0 = 0
        for im, n in zip(imgs, rows):
            B, _, H, W = im.shape
            _lib.call("esvit_patch_embed_fwd", _p(im), _p(w), _p(bias), _p(gamma), _p(beta), eps, _p(out[r0:]),
                      _p(mean[r0:]), _p(rstd[r0:]), B, H, W, E, _stream())
            r0 += n
        ctx.save_for_backward(w, bias, gamma, mean, rstd, *imgs)
        ctx.rows = rows
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        w, bias, gamma, mean, rstd = ctx.saved_tensors[:5]
        imgs = ctx.saved_tensors[5:]
        E = w.shape[0]
        g = _chk(g, F32, "g")
        dw, first = _acc(("pe_w", w.data_ptr()), tuple(w.shape), w.device)
        acc, _ = _acc(("pe_b", w.data_ptr()), (3, E), w.device)
        r0 = 0
        for im, n in zip(imgs, ctx.rows):
            B, _, H, W = im.shape
            _lib.call("esvit_patch_embed_bwd", _p(im), _p(w), _p(bias), _p(gamma), _p(mean[r0:]), _p(rstd[r0:]),
                      _p(g[r0:]), _p(dw), _p(acc[0]), _p(acc[1]), _p(acc[2]), B, H, W, E, _stream())
            r0 += n
        none = (None,) * len(imgs)
        return ((dw, acc[0], acc[1], acc[2], None) if first else (None, None, None, None, None)) + none


def cat_adjacent(ts):
    """torch.cat(ts) along dim 0 - as a VIEW when the tensors already lie back to back in one storage (the engine's
    static crop buffers do: the 2 global / 8 local crops of a step), so the multi-crop forward copies nothing."""
    ts = list(ts)
    if len(ts) == 1:
        return ts[0]
    t0 = ts[0]
    ok = all(t.shape == t0.shape and t.dtype == t0.dtype and t.device == t0.device and t.is_contiguous()
             and not t.requires_grad for t in ts)
    if ok:
        st, n = t0.untyped_storage(), t0.numel()
        ok = all(t.untyped_storage().data_ptr() == st.data_ptr() and t.storage_offset() == t0.storage_offset() + i * n
                 for i, t in enumerate(ts))
    if not ok:
        return torch.cat(ts)
    shape = (t0.shape[0] * len(ts),) + tuple(t0.shape[1:])
    return torch.as_strided(t0, shape, t0.stride(), t0.storage_offset())


# ------------------------------------------------------------------------------------------------------------
ATTN_WS_FLOATS = 8192  # per head; include/esvit_b200.h (expanded bias for ws 7, bias-gradient accumulator for ws 14)


class WindowAttentionGroupsFn(Function):
    """Shifted-window attention over resolution groups stored back to back in ONE token-major tensor: qkv bf16 [T, 3C]
    (qkv GEMM output incl. bias), group g = (B, H, W, row0) = rows [row0, row0 + B*H*W) holding B maps of H x W tokens
    -> attention output bf16 [T, C] in token order (pad / roll / partition / reverse folded in).  One kernel launch per
    group on pointer offsets (no slicing / concatenation copies).  qkv_bias (fp32 [3C] parameter) supplies the value of
    padded slots and receives the COMPLETE qkv-bias gradient from the backward kernel (column sums of dq/dk/dv); the
    table / qkv-bias gradients of all groups accumulate into the same buffers.  bias_exp: the table already expanded
    for this step by expand_rel_pos_bias (shared by every call and by the backward), or None: each call expands into
    its own scratch."""

    @staticmethod
    def forward(ctx, qkv, qkv_bias, bias_table, groups, num_heads: int, ws: int, shift: int, scale: float, bias_exp):
        qkv = _chk(qkv, BF16, "qkv")
        qkv_bias = _chk(qkv_bias, F32, "qkv_bias")
        bias_table = _chk(bias_table, F32, "relative_position_bias_table")
        T, C3 = qkv.shape
        C = C3 // 3
        assert sum(B * H * W for B, H, W, _ in groups) == T
        qb = shadow.lookup(qkv_bias)
        if qb is None:
            qb = qkv_bias.detach().to(BF16)
        out = torch.empty(T, C, dtype=BF16, device=qkv.device)
        lse_off, n = [], 0
        for B, H, W, _ in groups:
            lse_off.append(n)
            n += B * (-(-H // ws)) * (-(-W // ws)) * num_heads * ws * ws
        lse = torch.empty(n, dtype=F32, device=qkv.device)
        ready = 1 if (bias_exp is not None and ws == 7) else 0
        bws = bias_exp if ready else torch.empty(num_heads * ATTN_WS_FLOATS, dtype=F32, device=qkv.device)
        for (B, H, W, r0), lo in zip(groups, lse_off):
            _lib.call("esvit_window_attn_fwd", _po(qkv, r0 * C3), _p(qb), _p(bias_table), _p(bws), ready, _po(out, r0 * C),
                      _po(lse, lo), B, H, W, C, num_heads, ws, shift, scale, _stream())
        ctx.save_for_backward(qkv, qb, bias_table, out, lse, bws if ready else None)
        ctx.meta = (tuple(groups), tuple(lse_off), C, num_heads, ws, shift, scale)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        qkv, qb, bias_table, out, lse, bias_exp = ctx.saved_tensors
        groups, lse_off, C, nH, ws, shift, scale = ctx.meta
        g = _chk(g, BF16, "g")
        ready = 1 if bias_exp is not None else 0
        dqkv = torch.empty_like(qkv)
        dtable, first = _acc(("attn_t", bias_table.data_ptr()), tuple(bias_table.shape), qkv.device)
        dqb, _ = _acc(("attn_b", bias_table.data_ptr()), (3 * C,), qkv.device)
        bws = bias_exp if ready else torch.empty(nH * ATTN_WS_FLOATS, dtype=F32, device=qkv.device)
        for (B, H, W, r0), lo in zip(groups, lse_off):
            _lib.call("esvit_window_attn_bwd", _po(qkv, r0 * 3 * C), _p(qb), _p(bias_table), _p(bws), ready, _po(out, r0 * C),
                      _po(g, r0 * C), _po(lse, lo), _po(dqkv, r0 * 3 * C), _p(dtable), _p(dqb), B, H, W, C, nH, ws, shift,
                      scale, _stream())
        return dqkv, (dqb if first else None), (dtable if first else None), None, None, None, None, None, None


class PatchMergeLNGroupsFn(Function):
    """LN of the 2x2 gather of Swin's PatchMerging over resolution groups stored back to back: x fp32 [T, C] -> bf16
    [T', 4C] (T' = sum of B * ceil(H/2) * ceil(W/2); odd maps are zero-padded), one launch per group on pointer
    offsets."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps: float, groups):
        x, gamma, beta = _chk(x, F32, "x"), _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        T, C = x.shape
        assert sum(B * H * W for B, H, W, _ in groups) == T
        out_off, n = [], 0
        for B, H, W, _ in groups:
            out_off.append(n)
            n += B * ((H + 1) // 2) * ((W + 1) // 2)
        y = torch.empty(n, 4 * C, dtype=BF16, device=x.device)
        mean = torch.empty(n, dtype=F32, device=x.device)
        rstd = torch.empty(n, dtype=F32, device=x.device)
        for (B, H, W, r0), o0 in zip(groups, out_off):
            _lib.call("esvit_patch_merge_ln_fwd", _po(x, r0 * C), _p(gamma), _p(beta), eps, _po(y, o0 * 4 * C), _po(mean, o0),
                      _po(rstd, o0), B, H, W, C, _stream())
        ctx.save_for_backward(x, mean, rstd, gamma)
        ctx.meta = (tuple(groups), tuple(out_off))
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, mean, rstd, gamma = ctx.saved_tensors
        groups, out_off = ctx.meta
        T, C = x.shape
        g = _chk(g, BF16, "g")
        dx = torch.empty_like(x)
        acc, first = _acc(("merge", gamma.data_ptr()), (2, gamma.numel()), x.device)
        for (B, H, W, r0), o0 in zip(groups, out_off):
            _lib.call("esvit_patch_merge_ln_bwd", _po(g, o0 * 4 * C), _po(x, r0 * C), _po(mean, o0), _po(rstd, o0), _p(gamma),
                      _po(dx, r0 * C), _p(acc[0]), _p(acc[1]), B, H, W, C, _stream())
        return (dx, acc[0], acc[1], None, None) if first else (dx, None, None, None, None)


class TokenMeanGroupsFn(Function):
    """Mean over the tokens of every sample of resolution groups stored back to back: region fp32 [T, C] -> pooled
    fp32 [sum B, C]."""

    @staticmethod
    def forward(ctx, region, groups):
        region = _chk(region, F32, "region")
        T, C = region.shape
        nb = sum(B for B, _, _, _ in groups)
        pooled = torch.empty(nb, C, dtype=F32, device=region.device)
        b0 = 0
        for B, H, W, r0 in groups:
            _lib.call("esvit_token_mean_fwd", _po(region, r0 * C), _po(pooled, b0 * C), B, H * W, C, _stream())
            b0 += B
        ctx.meta = (tuple(groups), T, C)
        return pooled

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        groups, T, C = ctx.meta
        g = _chk(g, F32, "g")
        d = torch.empty(T, C, dtype=F32, device=g.device)
        b0 = 0
        for B, H, W, r0 in groups:
            _lib.call("esvit_token_mean_bwd", _po(g, b0 * C), None, _po(d, r0 * C), B, H * W, C, _stream())
            b0 += B
        return d, None


class MhsaGroupsFn(Function):
    """Whole-sequence multi-head attention at head dim 64 (models/vision_transformer.py:83-95) over several resolution
    groups stored back to back: qkv bf16 [T, 3C] (qkv GEMM output incl. bias), group g = (B, L, row0) = rows
    [row0, row0 + B*L) holding B sequences of L tokens -> bf16 [T, C].  One launch per group on pointer offsets.
    qkv_bias (fp32 [3C]) only receives its gradient: the fixed-order column sums of dqkv (esvit_colsum)."""

    @staticmethod
    def forward(ctx, qkv, qkv_bias, groups, num_heads: int, scale: float):
        qkv = _chk(qkv, BF16, "qkv")
        T, C3 = qkv.shape
        C = C3 // 3
        if sum(B * L for B, L, _ in groups) != T:
            raise ValueError(f"groups {groups} do not cover the {T} rows of qkv")
        out = torch.empty(T, C, dtype=BF16, device=qkv.device)
        lse = torch.empty(T * num_heads, dtype=F32, device=qkv.device)  # per group [B, nH, L] at row0 * nH
        for B, L, r0 in groups:
            _lib.call("esvit_mhsa_fwd", _po(qkv, r0 * C3), _po(out, r0 * C), _po(lse, r0 * num_heads), B, L, C, num_heads,
                      scale, _stream())
        ctx.save_for_backward(qkv, out, lse)
        ctx.meta = (tuple(groups), num_heads, scale, qkv_bias is not None)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        qkv, out, lse = ctx.saved_tensors
        groups, nH, scale, has_bias = ctx.meta
        g = _chk(g, BF16, "g")
        T, C3 = qkv.shape
        C = C3 // 3
        dqkv = torch.empty_like(qkv)
        dvec = torch.empty_like(lse)
        for B, L, r0 in groups:
            _lib.call("esvit_mhsa_bwd", _po(qkv, r0 * C3), _po(out, r0 * C), _po(g, r0 * C), _po(lse, r0 * nH),
                      _po(dvec, r0 * nH), _po(dqkv, r0 * C3), B, L, C, nH, scale, _stream())
        return dqkv, (colsum(dqkv) if has_bias else None), None, None, None


def mhsa(qkv: Tensor, num_heads: int, scale: float) -> Tuple[Tensor, Tensor]:
    """(out bf16 [B*L, C], lse fp32 [B, nH, L]) of MhsaGroupsFn's kernel on qkv bf16 [B, L, 3C]; not differentiable."""
    qkv = _chk(qkv, BF16, "qkv")
    B, L, C3 = qkv.shape
    out = torch.empty(B * L, C3 // 3, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, num_heads, L, dtype=F32, device=qkv.device)
    _lib.call("esvit_mhsa_fwd", _p(qkv), _p(out), _p(lse), B, L, C3 // 3, num_heads, scale, _stream())
    return out, lse


def vit_patches(imgs: Sequence[Tensor], p: int) -> Tensor:
    """fp32 [B_g, 3, S_g, S_g] crops -> the bf16 patch rows [sum_g B_g N_g, 3p^2] of all of them, back to back, in the
    conv weight's (c, ky, kx) flatten order (the input of the patch-projection GEMM)."""
    imgs = [_chk(im, F32, "img") for im in imgs]
    rows = [im.shape[0] * (im.shape[2] // p) * (im.shape[3] // p) for im in imgs]
    out = torch.empty(sum(rows), 3 * p * p, dtype=BF16, device=imgs[0].device)
    r0 = 0
    for im, n in zip(imgs, rows):
        B, Cin, H, W = im.shape
        if Cin != 3 or H != W or H % p != 0:
            raise ValueError(f"expected square crops [B, 3, S, S] with S a multiple of {p}, got {tuple(im.shape)}")
        _lib.call("esvit_vit_patches", _p(im), _po(out, r0 * 3 * p * p), B, H, p, _stream())
        r0 += n
    return out


class VitTokensGroupsFn(Function):
    """The ViT residual stream of several resolution groups, back to back in ONE fp32 tensor [sum_g B_g (1+N_g), D]:
    sequence b of group g = cat(cls_token, pe[b]) + pos_g (models/vision_transformer.py:237-240).
    pe bf16 [sum_g B_g N_g, D] is the patch-projection GEMM output (bias included); groups = ((B, N), ...);
    pos: one fp32 [1, 1+N_g, D] tensor per group.  bias (fp32 [D]) only receives its gradient (column sums of the patch
    rows' gradient)."""

    @staticmethod
    def forward(ctx, pe, bias, cls_token, groups, *pos):
        pe, cls = _chk(pe, BF16, "pe"), _chk(cls_token, F32, "cls_token")
        pos = [_chk(q, F32, "pos_embed") for q in pos]
        D = pe.shape[-1]
        T = sum(B * (N + 1) for B, N in groups)
        x = torch.empty(T, D, dtype=F32, device=pe.device)
        p0 = x0 = 0
        for (B, N), q in zip(groups, pos):
            if q.numel() != (N + 1) * D:
                raise ValueError(f"pos_embed of {q.numel()} values for {N} patches of width {D}")
            _lib.call("esvit_vit_tokens_fwd", _po(pe, p0 * D), _p(cls), _p(q), _po(x, x0 * D), B, N, D, _stream())
            p0 += B * N
            x0 += B * (N + 1)
        ctx.meta = (tuple(groups), D, pe.shape[0], tuple(tuple(q.shape) for q in pos))
        return x

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        groups, D, npe, pos_shapes = ctx.meta
        g = _chk(g, F32, "g")
        dpe = torch.empty(npe, D, dtype=BF16, device=g.device)
        dbias = torch.empty(D, dtype=F32, device=g.device)
        dcls = torch.empty(1, 1, D, dtype=F32, device=g.device)
        dpos, p0, x0 = [], 0, 0
        for gi, ((B, N), shp) in enumerate(zip(groups, pos_shapes)):
            d = torch.empty(shp, dtype=F32, device=g.device)
            _lib.call("esvit_vit_tokens_bwd", _po(g, x0 * D), _po(dpe, p0 * D), _p(d), _p(dbias), _p(dcls),
                      1 if gi else 0, B, N, D, _stream())
            dpos.append(d)
            p0 += B * N
            x0 += B * (N + 1)
        return (dpe, dbias, dcls, None) + tuple(dpos)


class VitSplitGroupsFn(Function):
    """x fp32 [sum_g B_g (1+N_g), D] (the final norm's output) -> (cls rows [sum_g B_g, D], region rows
    [sum_g B_g N_g, D]), group-major then image-major as the reference concatenates them; groups = ((B, N), ...)."""

    @staticmethod
    def forward(ctx, x, groups):
        x = _chk(x, F32, "x")
        D = x.shape[-1]
        nb = sum(B for B, _ in groups)
        cls = torch.empty(nb, D, dtype=F32, device=x.device)
        region = torch.empty(sum(B * N for B, N in groups), D, dtype=F32, device=x.device)
        _vit_split(x, cls, region, groups, 0)
        ctx.meta = (tuple(groups), tuple(x.shape))
        return cls, region

    @staticmethod
    @once_differentiable
    def backward(ctx, g_cls, g_region):
        groups, shape = ctx.meta
        g_cls = _chk(g_cls, F32, "g_cls")
        g_region = _chk(g_region, F32, "g_region")
        dx = torch.empty(shape, dtype=F32, device=(g_cls if g_cls is not None else g_region).device)
        _vit_split(dx, g_cls, g_region, groups, 1)
        return dx, None


def _vit_split(x, cls, region, groups, direction):
    D = x.shape[-1]
    x0 = b0 = q0 = 0
    for B, N in groups:
        _lib.call("esvit_vit_split", _po(x, x0 * D), _po(cls, b0 * D) if cls is not None else None,
                  _po(region, q0 * D) if region is not None else None, B, N, D, direction, _stream())
        x0 += B * (N + 1)
        b0 += B
        q0 += B * N


@torch.no_grad()
def window_attention_probs(qkv: Tensor, qkv_bias: Tensor, bias_table: Tensor, H: int, W: int, num_heads: int, ws: int,
                           shift: int, scale: float, bias_exp: Optional[Tensor] = None) -> Tensor:
    """The attention probabilities of the WindowAttentionGroupsFn call on the one group (B, H, W, 0) of qkv bf16
    [B, H*W, 3C] with the same other arguments, fp32
    [B*nWy*nWx, nH, ws*ws, ws*ws] in the reference's layout (the `attn` that WindowAttention.forward returns,
    models/swin_transformer.py:141-152): windows of the padded frame rolled by -shift, rows and columns of padded slots
    included.  Not differentiable."""
    qkv = _chk(qkv, BF16, "qkv")
    qkv_bias = _chk(qkv_bias, F32, "qkv_bias")
    bias_table = _chk(bias_table.detach(), F32, "relative_position_bias_table")
    B, L, C3 = qkv.shape
    if L != H * W:
        raise ValueError(f"qkv has {L} tokens per sample, expected H * W = {H * W}")
    C = C3 // 3
    qb = shadow.lookup(qkv_bias)
    if qb is None:
        qb = qkv_bias.detach().to(BF16)
    nwin = B * (-(-H // ws)) * (-(-W // ws))
    probs = torch.empty(nwin, num_heads, ws * ws, ws * ws, dtype=F32, device=qkv.device)
    ready = 1 if (bias_exp is not None and ws == 7) else 0
    bws = bias_exp if ready else torch.empty(num_heads * ATTN_WS_FLOATS, dtype=F32, device=qkv.device)
    _lib.call("esvit_window_attn_probs", _p(qkv), _p(qb), _p(bias_table), _p(bws), ready, _p(probs), B, H, W, C,
              num_heads, ws, shift, scale, _stream())
    return probs


def expand_rel_pos_bias(bias_table: Tensor, num_heads: int, ws: int) -> Optional[Tensor]:
    """ws = 7: the rel-pos bias table expanded ONCE for all attention calls (both crop groups, forward and backward) that
    use it this step -> fp32 [nH*4096] to pass as WindowAttentionGroupsFn's bias_exp; ws = 14: None (staged per CTA)."""
    if ws != 7:
        return None
    bias_table = _chk(bias_table.detach(), F32, "relative_position_bias_table")
    bws = torch.empty(num_heads * 4096, dtype=F32, device=bias_table.device)
    _lib.call("esvit_window_attn_expand_bias", _p(bias_table), _p(bws), num_heads, ws, _stream())
    return bws


class GeluFn(Function):
    @staticmethod
    def forward(ctx, x):
        x = _chk(x, BF16, "x")
        y = torch.empty_like(x)
        _lib.call("esvit_gelu_fwd", _p(x), _p(y), x.numel(), _stream())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        g = _chk(g, BF16, "g")
        dx = torch.empty_like(x)
        _lib.call("esvit_gelu_bwd", _p(x), _p(g), _p(dx), x.numel(), _stream())
        return dx


class BiasGeluFn(Function):
    """y = gelu(x) for x bf16 [..., N] that already holds the producing GEMM's bias; `bias` (fp32 [N] parameter) only
    receives its gradient = column sums of dx, computed inside the GELU backward kernel."""

    @staticmethod
    def forward(ctx, x, bias):
        x = _chk(x, BF16, "x")
        y = torch.empty_like(x)
        _lib.call("esvit_gelu_fwd", _p(x), _p(y), x.numel(), _stream())
        ctx.save_for_backward(x)
        ctx.bias_meta = (bias.shape, bias.device, bias.data_ptr())
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        g = _chk(g, BF16, "g")
        N = x.shape[-1]
        dx = torch.empty_like(x)
        db, first = _acc(("bias", ctx.bias_meta[2]), tuple(ctx.bias_meta[0]), ctx.bias_meta[1])
        _lib.call("esvit_gelu_bwd_dbias", _p(x), _p(g), _p(dx), _p(db), x.numel() // N, N, _stream())
        return dx, (db if first else None)


GEMM_COLSUM_WS_ROWS = 160  # include/esvit_b200.h: esvit_gemm_mul_colsum scratch rows


def gemm_bias_act(a: Tensor, w: Tensor, bias: Optional[Tensor], act: int = 0, want_pre: bool = False):
    """wgmma/TMA GEMM: act(a @ w^T + bias) -> bf16 [M, N] (and gelu'(a @ w^T + bias) when act != 0 and want_pre)."""
    a, w = _chk(a, BF16, "a"), _chk(w, BF16, "w")
    bias = _chk(bias, F32, "bias")
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    out = torch.empty(*a.shape[:-1], N, dtype=BF16, device=a.device)
    pre = torch.empty_like(out) if (act and want_pre) else None
    _lib.call("esvit_gemm_bias_act", _p(a), _p(w), _p(bias), _p(out), _p(pre), M, N, K, act, _stream())
    return (out, pre) if (act and want_pre) else out


def gemm(a: Tensor, b: Tensor, bias: Optional[Tensor] = None, act: int = 0, want_pre: bool = False, a_mn: bool = False,
         b_mn: bool = False, tile: int = 0):
    """wgmma/TMA GEMM: act(opA(a) @ opB(b) + bias) -> bf16 [M, N].
    a: [..., K] (a_mn: [K, M]);  b: [N, K] (b_mn: [K, N] - a Linear weight read as it lies for the input gradient)."""
    a, b = _chk(a, BF16, "a"), _chk(b, BF16, "b")
    bias = _chk(bias, F32, "bias")
    if a_mn:
        K, M = a.shape
        lead = (M,)
    else:
        K = a.shape[-1]
        M = a.numel() // K
        lead = tuple(a.shape[:-1])
    N = b.shape[1] if b_mn else b.shape[0]
    assert (b.shape[0] if b_mn else b.shape[1]) == K, (a.shape, b.shape)
    out = torch.empty(*lead, N, dtype=BF16, device=a.device)
    pre = torch.empty_like(out) if (act and want_pre) else None
    _lib.call("esvit_gemm_bf16", _p(a), _p(b), _p(bias), _p(out), _p(pre), M, N, K, 1 if a_mn else 0, 1 if b_mn else 0, act,
              tile, _stream())
    return (out, pre) if (act and want_pre) else out


def gemm_mul_colsum(a: Tensor, b: Tensor, mult: Tensor, colsum: Tensor, b_mn: bool = False, tile: int = 0) -> Tensor:
    """out = (a @ opB(b)) * mult (bf16); colsum (fp32 [N]) += column sums of out."""
    a, b, mult = _chk(a, BF16, "a"), _chk(b, BF16, "b"), _chk(mult, BF16, "mult")
    K = a.shape[-1]
    M = a.numel() // K
    N = b.shape[1] if b_mn else b.shape[0]
    out = torch.empty_like(mult)
    ws = torch.empty(GEMM_COLSUM_WS_ROWS * N, dtype=F32, device=a.device)
    _lib.call("esvit_gemm_mul_colsum2", _p(a), _p(b), _p(mult), _p(out), _p(colsum), _p(ws), M, N, K, 1 if b_mn else 0, tile,
              _stream())
    return out


MLP_FUSED_C = (96, 128, 192)  # include/esvit_b200.h: the widths esvit_mlp_fwd serves


def mlp_fwd(x: Tensor, w1: Tensor, b1: Optional[Tensor], w2: Tensor, b2: Optional[Tensor], want_h: bool = False):
    """y = GELU(x @ w1^T + b1) @ w2^T + b2 -> bf16 [..., C] in one kernel, equal to gemm(gemm(x, w1, b1, act=1), w2, b2).
    C = x.shape[-1] in MLP_FUSED_C, w1 [4C, C], w2 [C, 4C].  want_h: return (y, h, gelu'(pre)) for the backward."""
    x, w1, w2 = _chk(x, BF16, "x"), _chk(w1, BF16, "w1"), _chk(w2, BF16, "w2")
    b1, b2 = _chk(b1, F32, "b1"), _chk(b2, F32, "b2")
    C = x.shape[-1]
    M = x.numel() // C
    assert tuple(w1.shape) == (4 * C, C) and tuple(w2.shape) == (C, 4 * C), (x.shape, w1.shape, w2.shape)
    y = torch.empty_like(x)
    h = torch.empty(*x.shape[:-1], 4 * C, dtype=BF16, device=x.device) if want_h else None
    pre = torch.empty_like(h) if want_h else None
    _lib.call("esvit_mlp_fwd", _p(x), _p(w1), _p(b1), _p(w2), _p(b2), _p(y), _p(h), _p(pre), M, C, _stream())
    return (y, h, pre) if want_h else y


_wgrad_ws = {}


def gemm_wgrad(dy: Tensor, x: Tensor, out: Optional[Tensor] = None, accumulate: bool = False, tile: int = 0) -> Tensor:
    """dw[N, K] (fp32) (+)= dy[T, N]^T @ x[T, K]: the weight gradient of a Linear straight in fp32 (no bf16 round trip,
    no cast kernel, no transposes); deterministic split-K."""
    dy, x = _chk(dy, BF16, "dy"), _chk(x, BF16, "x")
    N, K = dy.shape[-1], x.shape[-1]
    T = dy.numel() // N
    assert x.numel() // K == T
    if out is None:
        out = torch.empty(N, K, dtype=F32, device=dy.device)
        accumulate = False
    key = (dy.device, N, K)
    ws = _wgrad_ws.get(key)
    if ws is None:
        n = _lib.load().esvit_gemm_wgrad_ws_floats(N, K)
        if n <= 0:
            raise ValueError("esvit_gemm_wgrad: weight too large for the split-K workspace")
        ws = _wgrad_ws[key] = torch.empty(n, dtype=F32, device=dy.device)
    _lib.call("esvit_gemm_wgrad", _p(dy), _p(x), _p(out), _p(ws), T, N, K, 1 if accumulate else 0, tile, _stream())
    return out


class LinearGeluFn(Function):
    """gelu(x @ w^T + b) as ONE wgmma/TMA kernel (esvit_gemm_bias_act): the GEMM epilogue adds the bias, applies the
    exact GELU and also emits gelu'(pre-activation), so the [T, 4C] hidden tensor is written once and never re-read in
    the forward and the backward's dh = dy * gelu' (+ bias gradient) is a pure streaming kernel; dx / dw are library
    GEMMs."""

    @staticmethod
    def forward(ctx, x, w, bias):
        out, pre = gemm_bias_act(x, w, bias, act=1, want_pre=True)
        ctx.save_for_backward(x, w, pre)
        ctx.bias_meta = (bias.shape, bias.device, bias.data_ptr())
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w, pre = ctx.saved_tensors  # pre = gelu'(x @ w^T + b)
        g = _chk(g, BF16, "g")
        N = pre.shape[-1]
        dh = torch.empty_like(pre)
        db, first = _acc(("bias", ctx.bias_meta[2]), tuple(ctx.bias_meta[0]), ctx.bias_meta[1])
        _lib.call("esvit_mul_bwd_dbias", _p(pre), _p(g), _p(dh), _p(db), pre.numel() // N, N, _stream())
        dh2 = dh.reshape(-1, N)
        dx = (dh2 @ w).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = dh2.t() @ x.reshape(-1, x.shape[-1]) if ctx.needs_input_grad[1] else None
        return dx, dw, (db if first else None)




class MlpFn(Function):
    """fc2(gelu(fc1(x))) of the Swin MLP (models/swin_transformer.py:31-35) with both GELU passes inside wgmma GEMM
    epilogues.  forward: h, gelu' = esvit_gemm_bias_act(x, w1, b1) (one kernel), y = h @ w2^T + b2 (library GEMM).
    backward: d(pre) = (dy @ w2) * gelu' and the fc1 bias gradient come out of ONE kernel (esvit_gemm_mul_colsum, w2t =
    w2^T bf16 [4C, C]); the hidden-sized dh tensor of the unfused chain (GEMM -> multiply kernel) is never written.
    fc2's bias gradient is produced by the consumer (residual add + LN backward), as for LinearBiasFn."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, w2t):
        h, pre = gemm_bias_act(x, w1, b1, act=1, want_pre=True)
        with torch.autocast("cuda", enabled=False):
            y = torch.nn.functional.linear(h, w2, b2)
        ctx.save_for_backward(x, w1, pre, h, w2t)
        ctx.bias_meta = (b1.shape, b1.device, b1.data_ptr())
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w1, pre, h, w2t = ctx.saved_tensors
        g = _chk(g, BF16, "g")
        C, N = g.shape[-1], pre.shape[-1]
        g2 = g.reshape(-1, C)
        M = g2.shape[0]
        dw2 = g2.t() @ h.reshape(-1, N) if ctx.needs_input_grad[3] else None
        dpre = torch.empty_like(pre)
        db1, first = _acc(("bias", ctx.bias_meta[2]), tuple(ctx.bias_meta[0]), ctx.bias_meta[1])
        ws = torch.empty(GEMM_COLSUM_WS_ROWS * N, dtype=F32, device=g.device)
        _lib.call("esvit_gemm_mul_colsum", _p(g2), _p(w2t), _p(pre), _p(dpre), _p(db1), _p(ws), M, N, C, _stream())
        d2 = dpre.reshape(-1, N)
        dx = (d2 @ w1).view(x.shape) if ctx.needs_input_grad[0] else None
        dw1 = d2.t() @ x.reshape(-1, x.shape[-1]) if ctx.needs_input_grad[1] else None
        return dx, dw1, (db1 if first else None), dw2, None, None


class LinearBiasFn(Function):
    """y = x @ w^T + b as ONE library GEMM (bias in the cuBLASLt epilogue).  The backward produces dx and dw with two
    library GEMMs and NO bias gradient: the consumer kernel (window attention / GELU / add+LN backward) column-sums
    it for free, which removes the reference's per-layer `grad.sum(0)` reduction kernels (10 % of the first profile)."""

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        with torch.autocast("cuda", enabled=False):
            return torch.nn.functional.linear(x, w, b)

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        g2 = g.reshape(-1, g.shape[-1])
        dx = (g2 @ w).view(x.shape) if ctx.needs_input_grad[0] else None
        dw = g2.t() @ x.reshape(-1, x.shape[-1]) if ctx.needs_input_grad[1] else None
        return dx, dw, None


class L2NormFn(Function):
    @staticmethod
    def forward(ctx, x, eps: float):
        x = _chk(x, BF16, "x")
        R, Dm = x.numel() // x.shape[-1], x.shape[-1]
        y = torch.empty_like(x)
        inv = torch.empty(R, dtype=F32, device=x.device)
        _lib.call("esvit_l2norm_fwd", _p(x), _p(y), _p(inv), eps, R, Dm, _stream())
        ctx.save_for_backward(x, inv)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, inv = ctx.saved_tensors
        g = _chk(g, BF16, "g")
        R, Dm = x.numel() // x.shape[-1], x.shape[-1]
        dx = torch.empty_like(x)
        _lib.call("esvit_l2norm_bwd", _p(x), _p(g), _p(inv), _p(dx), R, Dm, _stream())
        return dx, None


class WeightNormFn(Function):
    """(v fp32 [K,D], g fp32 [K,1]) -> w bf16 [K,D] = v * g / ||v||_row."""

    @staticmethod
    def forward(ctx, v, g):
        v, g = _chk(v, F32, "weight_v"), _chk(g, F32, "weight_g")
        K, Dm = v.shape
        w = torch.empty(K, Dm, dtype=BF16, device=v.device)
        norm = torch.empty(K, dtype=F32, device=v.device)
        _lib.call("esvit_weight_norm_fwd", _p(v), _p(g), _p(w), _p(norm), K, Dm, _stream())
        ctx.save_for_backward(v, g, norm)
        return w

    @staticmethod
    @once_differentiable
    def backward(ctx, gw):
        v, g, norm = ctx.saved_tensors
        f32 = gw.dtype == F32  # fp32 from esvit_gemm_wgrad, bf16 from a library GEMM
        gw = _chk(gw, F32 if f32 else BF16, "gw")
        K, Dm = v.shape
        dv = torch.empty_like(v)
        dg = torch.empty_like(g) if ctx.needs_input_grad[1] else None
        _lib.call("esvit_weight_norm_bwd", _p(v), _p(g), _p(norm), _p(gw), 1 if f32 else 0, _p(dv), _p(dg), K, Dm, _stream())
        return dv, dg


# ------------------------------------------------------------------------------------------------------------
# losses


def row_lse(x: Tensor, center: Optional[Tensor], inv_temp: float) -> Tensor:
    x = _chk(x, BF16, "logits")
    R, K = x.shape
    lse = torch.empty(R, dtype=F32, device=x.device)
    _lib.call("esvit_row_lse", _p(x), _p(center), inv_temp, _p(lse), R, K, _stream())
    return lse


def ce_q_enabled(K: int) -> bool:
    """The CE kernels run on teacher probabilities stored once per teacher row (fp16, esvit_row_softmax_q) unless
    ESVIT_CE_Q=0 or a row of K logits does not fit one CTA's shared memory."""
    import os
    return os.environ.get("ESVIT_CE_Q", "1") != "0" and K <= _lib.load().esvit_row_softmax_q_max_k()


def row_softmax_q(x: Tensor, center: Tensor, inv_temp: float) -> Tuple[Tensor, Tensor]:
    """(lse fp32 [R] as row_lse, q fp16 [R, K] = 2^12 * softmax((x - center) * inv_temp)): ONE pass over the teacher rows."""
    x, center = _chk(x, BF16, "teacher logits"), _chk(center, F32, "center")
    R, K = x.shape
    lse = torch.empty(R, dtype=F32, device=x.device)
    q = torch.empty(R, K, dtype=torch.float16, device=x.device)
    _lib.call("esvit_row_softmax_q", _p(x), _p(center), inv_temp, _p(lse), _p(q), R, K, _stream())
    return lse, q


class DinoCEFn(Function):
    """loss = sum_r w[r] * ( n_r * LSE(s_r / tau) - sum_j <softmax((t[trow[r,j]] - center) / temp), s_r / tau> ).

    s bf16 [R,K] (grad), t bf16 [Rt,K], center fp32 [K], trow int32 [R,2], w fp32 [R].
    lse_t = None (the default path): the teacher probabilities are computed ONCE per teacher row and stored in fp16
    (row_softmax_q), the CE kernels stream them; lse_t = row_lse(t, center, inv_temp_t): every pairing recomputes the
    teacher exponentials from the logits (the round-1 kernels)."""

    @staticmethod
    def forward(ctx, s, t, center, lse_t, trow, w, inv_temp_t: float, inv_tau_s: float, order=None):
        s, t = _chk(s, BF16, "student logits"), _chk(t, BF16, "teacher logits")
        center, w = _chk(center, F32, "center"), _chk(w, F32, "w")
        trow = _chk(trow, torch.int32, "trow")
        order = _chk(order, torch.int32, "order")
        R, K = s.shape
        lse_s = torch.empty(R, dtype=F32, device=s.device)  # written by the CE kernel itself (one pass over s)
        row_loss = torch.empty(R, dtype=F32, device=s.device)
        ctx.use_q = lse_t is None
        if ctx.use_q:
            _, q = row_softmax_q(t, center, inv_temp_t)
            _lib.call("esvit_dino_ce_q_fwd", _p(s), _p(q), _p(lse_s), _p(trow), _p(order), inv_tau_s, _p(row_loss), R, K,
                      _stream())
            ctx.save_for_backward(s, q, lse_s, trow, w, order)
        else:
            lse_t = _chk(lse_t, F32, "lse_t")
            _lib.call("esvit_dino_ce_fwd", _p(s), _p(t), _p(center), _p(lse_s), _p(lse_t), _p(trow), _p(order), inv_temp_t,
                      inv_tau_s, _p(row_loss), R, K, _stream())
            ctx.save_for_backward(s, t, center, lse_s, lse_t, trow, w, order)
        loss = torch.empty((), dtype=F32, device=s.device)
        _lib.call("esvit_weighted_sum", _p(row_loss), _p(w), R, _p(loss), _stream())
        ctx.temps = (inv_temp_t, inv_tau_s)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        inv_temp_t, inv_tau_s = ctx.temps
        gs = _chk(g.reshape(1).to(F32), F32, "g")
        if ctx.use_q:
            s, q, lse_s, trow, w, order = ctx.saved_tensors
            R, K = s.shape
            ds = torch.empty_like(s)
            _lib.call("esvit_dino_ce_q_bwd", _p(s), _p(q), _p(lse_s), _p(trow), _p(order), _p(w), _p(gs), inv_tau_s, _p(ds),
                      R, K, _stream())
        else:
            s, t, center, lse_s, lse_t, trow, w, order = ctx.saved_tensors
            R, K = s.shape
            ds = torch.empty_like(s)
            _lib.call("esvit_dino_ce_bwd", _p(s), _p(t), _p(center), _p(lse_s), _p(lse_t), _p(trow), _p(order), _p(w),
                      _p(gs), inv_temp_t, inv_tau_s, _p(ds), R, K, _stream())
        return ds, None, None, None, None, None, None, None, None


_colsum_ws = {}


def colsum(t: Tensor, out: Optional[Tensor] = None) -> Tensor:
    """fp32 column sums of a bf16 [R, K] matrix (deterministic)."""
    t = _chk(t, BF16, "teacher logits")
    R, K = t.shape
    key = (t.device, K)
    ws = _colsum_ws.get(key)
    if ws is None:
        rows = _lib.load().esvit_colsum_workspace_rows()
        ws = _colsum_ws[key] = torch.empty(rows * K, dtype=F32, device=t.device)
    if out is None:
        out = torch.empty(K, dtype=F32, device=t.device)
    _lib.call("esvit_colsum", _p(t), R, K, _p(ws), _p(out), _stream())
    return out


def center_ema(center: Tensor, colsum_total: Tensor, rows_total: int, momentum: float,
               out: Optional[Tensor] = None) -> Tensor:
    """out = center*m + (colsum/rows)*(1-m); out defaults to a new tensor, out=center updates in place."""
    assert center.is_cuda and center.dtype == F32 and center.is_contiguous()
    if out is None:
        out = torch.empty_like(center)
    _lib.call("esvit_center_ema", _p(center), _p(colsum_total), float(rows_total), momentum, _p(out), center.numel(),
              _stream())
    return out


def normalize_rows(x: Tensor, eps: float = 1e-12) -> Tensor:
    x = _chk(x, F32, "features")
    y = torch.empty_like(x)
    _lib.call("esvit_normalize_rows", _p(x), _p(y), x.shape[0], x.shape[1], eps, _stream())
    return y


def region_match(s_fea: Tensor, t_fea: Tensor, B: int, ncrops: int, Tg: int, Tl: int) -> Tuple[Tensor, Tensor]:
    """Cosine arg-max of every student region token against the teacher view's tokens of the same image.

    Returns (idx int64 [2, ncrops, B, Tg] with -1 in unused slots, trow int32 [Rs, 2] teacher region row per iq)."""
    sn, tn = normalize_rows(s_fea), normalize_rows(t_fea)
    P = sn.shape[1]
    Rs = sn.shape[0]
    assert Rs == B * (2 * Tg + (ncrops - 2) * Tl) and tn.shape[0] == 2 * B * Tg
    idx = torch.full((2, ncrops, B, Tg), -1, dtype=torch.int64, device=sn.device)
    trow = torch.empty(Rs, 2, dtype=torch.int32, device=sn.device)
    _lib.call("esvit_region_match", _p(sn), _p(tn), B, ncrops, Tg, Tl, P, _p(idx), _p(trow), _stream())
    return idx, trow


# ------------------------------------------------------------------------------------------------------------
# CvT (models/cvt_v4_transformer.py): conv token embedding, depthwise conv + BatchNorm, window attention at head dim 64.
# A window group g = (B, H, W, w, row0, prow0): B maps of H x W tokens at rows [row0, row0 + B*H*W) of the token-major
# stream, their zero-padded Hp x Wp maps (multiples of the window w) at rows [prow0, prow0 + B*Hp*Wp) of the padded
# buffers (the depthwise + BN output and the qkv GEMM output).


def win_padded(H: int, W: int, w: int) -> Tuple[int, int]:
    return -(-H // w) * w, -(-W // w) * w


def conv_out_size(S: int, k: int, stride: int, pad: int) -> int:
    return (S + 2 * pad - k) // stride + 1


class ConvEmbedFn(Function):
    """Conv2d(Cin, Cout, k, stride, pad) of ConvEmbed (:349-382) over every resolution group as ONE GEMM: the patch rows
    bf16 [sum B*Ho*Wo, Kp] (esvit_conv_im2col) . w16^T + bias -> bf16 [sum B*Ho*Wo, Cout], groups back to back.
    Source: `imgs` (fp32 NCHW crops, one tensor per group; no input gradient) or x fp32 token-major [T, Cin] with
    groups ((B, H, W, row0), ...).  w16 bf16 [Cout, Kp]: the weight flattened in (c, ky, kx) order, K padded to a multiple
    of 8 with zero columns.  bias (fp32 [Cout]) gets its gradient from the consumer (the fused add + LN).  backward: the
    fp32 weight gradient (padding columns dropped) and, for x, the col2im gather of the rows' gradient."""

    @staticmethod
    def forward(ctx, x, weight, w16, bias, imgs, groups, k: int, stride: int, pad: int):
        w16 = _chk(w16, BF16, "w16")
        Cout, Kp = w16.shape
        Cin = weight.shape[1]
        if imgs is not None:
            src = [(_chk(im, F32, "img"), 1, im.shape[0], im.shape[2], im.shape[3]) for im in imgs]
        else:
            x = _chk(x, F32, "x")
            src = [(x, 0, B, H, W, r0) for B, H, W, r0 in groups]
        n = [s[2] * conv_out_size(s[3], k, stride, pad) * conv_out_size(s[4], k, stride, pad) for s in src]
        rows = torch.empty(sum(n), Kp, dtype=BF16, device=w16.device)
        r0 = 0
        for s, ni in zip(src, n):
            t, nchw, B, H, W = s[:5]
            base = _p(t) if nchw else _po(t, s[5] * Cin)
            _lib.call("esvit_conv_im2col", base, _po(rows, r0 * Kp), nchw, B, Cin, H, W, k, stride, pad, Kp, _stream())
            r0 += ni
        y = gemm(rows, w16, bias)
        ctx.save_for_backward(rows, w16)
        ctx.meta = (tuple(weight.shape), None if imgs is not None else (tuple(x.shape), tuple(groups)), k, stride, pad)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        rows, w16 = ctx.saved_tensors
        wshape, xmeta, k, stride, pad = ctx.meta
        g = _chk(g, BF16, "g")
        Cout, Cin = wshape[0], wshape[1]
        K = Cin * k * k
        dw = None
        if ctx.needs_input_grad[1]:
            dw = gemm_wgrad(g, rows)
            dw = (dw[:, :K].contiguous() if dw.shape[1] != K else dw).view(wshape)
        dx = None
        if xmeta is not None and ctx.needs_input_grad[0]:
            xshape, groups = xmeta
            drows = gemm(g, w16, None, b_mn=True)
            Kp = drows.shape[1]
            dx = torch.empty(xshape, dtype=F32, device=g.device)
            o0 = 0
            for B, H, W, r0 in groups:
                _lib.call("esvit_conv_col2im", _po(drows, o0 * Kp), _po(dx, r0 * Cin), B, Cin, H, W, k, stride, pad, Kp,
                          _stream())
                o0 += B * conv_out_size(H, k, stride, pad) * conv_out_size(W, k, stride, pad)
        return dx, dw, None, None, None, None, None, None, None


def _bn_part(groups, C: int, device) -> Tensor:
    n = max(-(-(B * Hp * Wp) // 256) for B, H, W, w, _, _ in groups for Hp, Wp in (win_padded(H, W, w),))
    return torch.empty(n * 9 * C, dtype=F32, device=device)


class DwBnFn(Function):
    """DepthWiseConv2d.dw + .bn (:101-104) on the zero-padded maps (Attention.forward :170-180): y bf16 [T, C] (the
    PreNorm output of every window group) -> bf16 [Tp, C] of the padded maps, ready for the pw GEMM.  `bn` is the
    nn.BatchNorm2d holding gamma / beta and the running buffers; train: per-group batch statistics over the padded maps
    (the running statistics are updated in place, group by group, as the reference's per-group forward does); else the
    running statistics.  pg: the process group of a SyncBatchNorm (world size > 1) or None; the per-channel sums (and
    the count) are then all-reduced in one call per BN call, forward and backward."""

    @staticmethod
    def forward(ctx, y, weight, gamma, beta, bn, groups, train: bool, pg):
        y = _chk(y, BF16, "y")
        w = _chk(weight, F32, "weight").view(-1, 9)
        gamma, beta = _chk(gamma, F32, "gamma"), _chk(beta, F32, "beta")
        C = y.shape[1]
        Tp = sum(B * Hp * Wp for B, H, W, w_, _, _ in groups for Hp, Wp in (win_padded(H, W, w_),))
        z = torch.empty(Tp, C, dtype=BF16, device=y.device)
        out = torch.empty_like(z)
        part = _bn_part(groups, C, y.device)
        sums = torch.empty(len(groups), 2 * C + 1, dtype=torch.float64, device=y.device)
        stat = torch.empty(len(groups), 4 * C, dtype=F32, device=y.device)
        rm, rv, nbt = bn.running_mean, bn.running_var, bn.num_batches_tracked
        for i, (B, H, W, w_, r0, p0) in enumerate(groups):
            Hp, Wp = win_padded(H, W, w_)
            _lib.call("esvit_dwbn_fwd_stats", _po(y, r0 * C), _p(w), _po(z, p0 * C), _p(part), _p(sums[i]), B, H, W,
                      Hp, Wp, C, _stream())
            if train and pg is not None:
                torch.distributed.all_reduce(sums[i], group=pg)
            _lib.call("esvit_dwbn_fwd_apply", _po(z, p0 * C), _p(gamma), _p(beta), _p(sums[i]) if train else None,
                      _p(rm), _p(rv), _p(nbt) if (train and nbt is not None) else None, _p(stat[i]), _po(out, p0 * C),
                      B * Hp * Wp, C, 1 if train else 0, float(bn.momentum), float(bn.eps), _stream())
        ctx.save_for_backward(y, z, w, stat)
        ctx.meta = (tuple(groups), train, pg, tuple(weight.shape), gamma.data_ptr(), weight.data_ptr())
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        y, z, w, stat = ctx.saved_tensors
        groups, train, pg, wshape, gptr, wptr = ctx.meta
        g = _chk(g, BF16, "g")
        C = y.shape[1]
        dy = torch.empty_like(y)
        part = _bn_part(groups, C, y.device)
        bsums = torch.empty(2 * C + 1, dtype=torch.float64, device=y.device)
        coef = torch.empty(3 * C, dtype=F32, device=y.device)
        dwt, first_w = _acc(("dw", wptr), wshape, y.device)
        aff, first_a = _acc(("bn", gptr), (2, C), y.device)  # dgamma | dbeta
        for i, (B, H, W, w_, r0, p0) in enumerate(groups):
            Hp, Wp = win_padded(H, W, w_)
            N = B * Hp * Wp
            _lib.call("esvit_dwbn_bwd_stats", _po(g, p0 * C), _po(z, p0 * C), _p(stat[i]), _p(part), _p(bsums),
                      _p(aff[0]), _p(aff[1]), N, C, _stream())
            if train and pg is not None:
                torch.distributed.all_reduce(bsums, group=pg)
            _lib.call("esvit_dwbn_bwd_apply", _po(g, p0 * C), _po(z, p0 * C), _po(y, r0 * C), _p(w), _p(stat[i]),
                      _p(bsums), _p(coef), _po(dy, r0 * C), _p(part), _p(dwt), B, H, W, Hp, Wp, C, 1 if train else 0,
                      _stream())
        return (dy, dwt if first_w else None, aff[0] if first_a else None, aff[1] if first_a else None,
                None, None, None, None)


class MhsaWinGroupsFn(Function):
    """Window attention of CvT (Attention.forward :180-218; no mask, no bias) at head dim 64: qkv bf16 [Tp, 3C] of the
    padded maps (pw GEMM output incl. bias) -> the cropped output bf16 [T, C]; groups as DwBnFn's.  One launch per group.
    qkv_bias only receives its gradient: the fixed-order column sums of dqkv."""

    @staticmethod
    def forward(ctx, qkv, qkv_bias, groups, num_heads: int, scale: float):
        qkv = _chk(qkv, BF16, "qkv")
        Tp, C3 = qkv.shape
        C = C3 // 3
        T = sum(B * H * W for B, H, W, _, _, _ in groups)
        out = torch.empty(T, C, dtype=BF16, device=qkv.device)
        lse = torch.empty(Tp * num_heads, dtype=F32, device=qkv.device)  # per group [windows, nH, w*w] at prow0 * nH
        for B, H, W, w, r0, p0 in groups:
            _lib.call("esvit_mhsa_win_fwd", _po(qkv, p0 * C3), _po(out, r0 * C), _po(lse, p0 * num_heads), B, H, W, w, C,
                      num_heads, scale, _stream())
        ctx.save_for_backward(qkv, out, lse)
        ctx.meta = (tuple(groups), num_heads, scale, qkv_bias is not None)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        qkv, out, lse = ctx.saved_tensors
        groups, nH, scale, has_bias = ctx.meta
        g = _chk(g, BF16, "g")
        C3 = qkv.shape[1]
        C = C3 // 3
        dqkv = torch.empty_like(qkv)
        dvec = torch.empty_like(lse)
        for B, H, W, w, r0, p0 in groups:
            _lib.call("esvit_mhsa_win_bwd", _po(qkv, p0 * C3), _po(out, r0 * C), _po(g, r0 * C), _po(lse, p0 * nH),
                      _po(dvec, p0 * nH), _po(dqkv, p0 * C3), B, H, W, w, C, nH, scale, _stream())
        return dqkv, (colsum(dqkv) if has_bias else None), None, None, None


VIL_W = 7               # sliding-chunk size of the Vision Longformer
VIL_NB = 1 + 9 * VIL_W * VIL_W  # local bias columns: the global key, then 9 neighbour chunks of 49 keys
_vil_ws = {}  # scratch per geometry, never freed: a captured CUDA graph may still write into it


class SlidingChunkAttnFn(Function):
    """Vision Longformer attention with one global token (layers/longformer2d.py Long2DSCSelfAttention.forward
    :139-330, exact = 0, rpe, shared global weights, head dim 32): q bf16 [B*N, C] (query GEMM output over all N = 1 +
    nx*ny rows per image, unscaled), kv bf16 [B*N, 2C] -> the context bf16 [B*N, C] that feeds proj (global row 0
    first, :330).  bias fp32 [nH, 49, 442] is the dense local bias (column 0: g2l[1]; 1 + j*49 + r: key r of neighbour
    chunk j in slidingchunk_qk order), bias_g fp32 [nH, N] the global row's (g2g | g2l[0]).  mode is an int32 CUDA
    tensor [1] holding 0 (all nine chunks), 1..8 (the own chunk plus mode_dict[mode]) or -1 (the own chunk only); the
    kernels read it at run time (clamping it into -1..8), so a captured CUDA graph follows whatever was written into it
    before the replay."""

    @staticmethod
    def forward(ctx, q, kv, bias, bias_g, mode, B: int, nx: int, ny: int, num_heads: int, scale: float):
        q = _chk(q, BF16, "q")
        kv = _chk(kv, BF16, "kv")
        bias = _chk(bias, F32, "bias").contiguous()
        bias_g = _chk(bias_g, F32, "bias_g").contiguous()
        mode = _chk(mode, torch.int32, "mode")
        N, C = 1 + nx * ny, 32 * num_heads
        if q.shape != (B * N, C) or kv.shape != (B * N, 2 * C) or not q.is_contiguous() or not kv.is_contiguous():
            raise ValueError(f"q [B*N, C] = [{B * N}, {C}] and kv [B*N, 2C] contiguous required, got "
                             f"{tuple(q.shape)}, {tuple(kv.shape)}")
        if bias.shape != (num_heads, VIL_W * VIL_W, VIL_NB) or bias_g.shape != (num_heads, N) or mode.numel() != 1:
            raise ValueError("bias [nH, 49, 442], bias_g [nH, N] and a one-element mode required")
        mx, my = -(-nx // VIL_W), -(-ny // VIL_W)
        out = torch.empty(B * N, C, dtype=BF16, device=q.device)
        lse = torch.empty(B * num_heads * mx * my * VIL_W * VIL_W, dtype=F32, device=q.device)
        lse_g = torch.empty(B * num_heads, dtype=F32, device=q.device)
        _lib.call("esvit_vil_sc_fwd", _p(q), _p(kv), _p(bias), _p(bias_g), _p(mode), _p(out), _p(lse), _p(lse_g), B, nx,
                  ny, num_heads, scale, _stream())
        ctx.save_for_backward(q, kv, bias, bias_g, mode, out, lse, lse_g)
        ctx.meta = (B, nx, ny, num_heads, scale)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, kv, bias, bias_g, mode, out, lse, lse_g = ctx.saved_tensors
        B, nx, ny, nH, scale = ctx.meta
        g = _chk(g, BF16, "g").contiguous()
        ws = _vil_sc_ws(q.device, B, nx, ny, nH)
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        dvec = torch.empty_like(lse)
        dbias, dbias_g = torch.empty_like(bias), torch.empty_like(bias_g)
        _lib.call("esvit_vil_sc_bwd", _p(q), _p(kv), _p(bias), _p(bias_g), _p(mode), _p(out), _p(g), _p(lse), _p(lse_g),
                  _p(dvec), _p(ws), _p(dq), _p(dkv), _p(dbias), _p(dbias_g), B, nx, ny, nH, scale, _stream())
        return dq, dkv, dbias, dbias_g, None, None, None, None, None, None


def _vil_sc_ws(device, B: int, nx: int, ny: int, nH: int) -> Tensor:
    key = (device, B, nx, ny, nH)
    ws = _vil_ws.get(key)
    if ws is None:
        n = _lib.load().esvit_vil_sc_ws_floats(B, nx, ny, nH)
        if n <= 0:
            raise ValueError("esvit_vil_sc_bwd: problem too large for the workspace")
        ws = _vil_ws[key] = torch.empty(n, dtype=F32, device=device)
    return ws


class SlidingChunkAttnGroupsFn(Function):
    """SlidingChunkAttnFn over resolution groups stored back to back: q bf16 [T, C], kv bf16 [T, 2C] (the query / kv
    GEMM outputs incl. bias over every row of every image), group g = (B, nx, ny, row0, bias_off, bias_g_off) = rows
    [row0, row0 + B*(1 + nx*ny)).  bias: ONE fp32 vector (RelBiasFn's output) holding every group's [nH, 49, 442] local
    bias at bias_off and its [nH, N] global-row bias at bias_g_off; modes int32 [G] on the device, element g the mode
    of group g.  One esvit_vil_sc_fwd / _bwd per group on pointer offsets.  The bias gradient of group g is written into
    the same offsets of one gradient vector (the kernel writes, it does not accumulate; RelBiasFn's backward sums the
    groups in a fixed order).  q_bias / kv_bias (fp32 or None) only receive their gradients: column sums of dq / dkv."""

    @staticmethod
    def forward(ctx, q, kv, q_bias, kv_bias, bias, modes, groups, num_heads: int, scale: float):
        q, kv = _chk(q, BF16, "q"), _chk(kv, BF16, "kv")
        bias = _chk(bias, F32, "bias")
        modes = _chk(modes, torch.int32, "modes")
        T, C = q.shape
        if C != 32 * num_heads or kv.shape != (T, 2 * C):
            raise ValueError(f"q [T, 32 nH] and kv [T, 2C] required, got {tuple(q.shape)}, {tuple(kv.shape)}")
        if sum(B * (1 + nx * ny) for B, nx, ny, _, _, _ in groups) != T or modes.numel() != len(groups):
            raise ValueError(f"groups {groups} do not cover the {T} rows, or not one mode per group")
        out = torch.empty(T, C, dtype=BF16, device=q.device)
        lse_off, lse_g_off, n, ng = [], [], 0, 0
        for B, nx, ny, _, _, _ in groups:
            lse_off.append(n)
            lse_g_off.append(ng)
            n += B * num_heads * (-(-nx // VIL_W)) * (-(-ny // VIL_W)) * VIL_W * VIL_W
            ng += B * num_heads
        lse = torch.empty(n, dtype=F32, device=q.device)
        lse_g = torch.empty(ng, dtype=F32, device=q.device)
        for gi, ((B, nx, ny, r0, bo, bgo), lo, lgo) in enumerate(zip(groups, lse_off, lse_g_off)):
            _lib.call("esvit_vil_sc_fwd", _po(q, r0 * C), _po(kv, r0 * 2 * C), _po(bias, bo), _po(bias, bgo),
                      _po(modes, gi), _po(out, r0 * C), _po(lse, lo), _po(lse_g, lgo), B, nx, ny, num_heads, scale,
                      _stream())
        ctx.save_for_backward(q, kv, bias, modes, out, lse, lse_g)
        ctx.meta = (tuple(groups), tuple(lse_off), tuple(lse_g_off), num_heads, scale, q_bias is not None,
                    kv_bias is not None)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        q, kv, bias, modes, out, lse, lse_g = ctx.saved_tensors
        groups, lse_off, lse_g_off, nH, scale, has_qb, has_kvb = ctx.meta
        g = _chk(g, BF16, "g")
        C = q.shape[1]
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        dvec = torch.empty_like(lse)
        dbias = torch.zeros_like(bias)  # every group writes its own slots; the zeros cover nothing but alignment gaps
        for gi, ((B, nx, ny, r0, bo, bgo), lo, lgo) in enumerate(zip(groups, lse_off, lse_g_off)):
            ws = _vil_sc_ws(q.device, B, nx, ny, nH)
            _lib.call("esvit_vil_sc_bwd", _po(q, r0 * C), _po(kv, r0 * 2 * C), _po(bias, bo), _po(bias, bgo),
                      _po(modes, gi), _po(out, r0 * C), _po(g, r0 * C), _po(lse, lo), _po(lse_g, lgo), _po(dvec, lo),
                      _p(ws), _po(dq, r0 * C), _po(dkv, r0 * 2 * C), _po(dbias, bo), _po(dbias, bgo), B, nx, ny, nH,
                      scale, _stream())
        return (dq, dkv, colsum(dq) if has_qb else None, colsum(dkv) if has_kvb else None, dbias,
                None, None, None, None)


class DenseBiasAttnGroupsFn(Function):
    """Whole-sequence attention at head dim 32 with an additive bias (vision_longformer.py Attention.forward :86-131)
    over resolution groups stored back to back: qkv bf16 [T, 3C] (qkv GEMM output incl. bias), group g = (B, L, row0,
    bias_off) = rows [row0, row0 + B*L), bias fp32 [nH, L, L] at bias_off of ONE vector (RelBiasFn's output).  One
    esvit_vil_dense_fwd / _bwd per group; each group's bias gradient (sum over its images, fixed order) is written at the
    same offset of one gradient vector.  qkv_bias only receives its gradient: the column sums of dqkv."""

    @staticmethod
    def forward(ctx, qkv, qkv_bias, bias, groups, num_heads: int, scale: float):
        qkv, bias = _chk(qkv, BF16, "qkv"), _chk(bias, F32, "bias")
        T, C3 = qkv.shape
        C = C3 // 3
        if sum(B * L for B, L, _, _ in groups) != T:
            raise ValueError(f"groups {groups} do not cover the {T} rows of qkv")
        out = torch.empty(T, C, dtype=BF16, device=qkv.device)
        lse = torch.empty(T * num_heads, dtype=F32, device=qkv.device)  # per group [B, nH, L] at row0 * nH
        for B, L, r0, bo in groups:
            _lib.call("esvit_vil_dense_fwd", _po(qkv, r0 * C3), _po(bias, bo), _po(out, r0 * C), _po(lse, r0 * num_heads),
                      B, L, C, num_heads, scale, _stream())
        ctx.save_for_backward(qkv, bias, out, lse)
        ctx.meta = (tuple(groups), num_heads, scale, qkv_bias is not None)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        qkv, bias, out, lse = ctx.saved_tensors
        groups, nH, scale, has_bias = ctx.meta
        g = _chk(g, BF16, "g")
        C = qkv.shape[1] // 3
        dqkv = torch.empty_like(qkv)
        dvec = torch.empty_like(lse)
        dbias = torch.zeros_like(bias)
        lib = _lib.load()
        for B, L, r0, bo in groups:
            part = torch.empty(lib.esvit_vil_dense_parts(B) * nH * L * L, dtype=F32, device=qkv.device)
            _lib.call("esvit_vil_dense_bwd", _po(qkv, r0 * 3 * C), _po(bias, bo), _po(out, r0 * C), _po(g, r0 * C),
                      _po(lse, r0 * nH), _po(dvec, r0 * nH), _p(part), _po(dqkv, r0 * 3 * C), _po(dbias, bo), B, L, C, nH,
                      scale, _stream())
        return dqkv, (colsum(dqkv) if has_bias else None), dbias, None, None, None


def vil_dense_attention(qkv: Tensor, bias: Tensor, num_heads: int, scale: float) -> Tuple[Tensor, Tensor]:
    """(out bf16 [B*L, C], lse fp32 [B, nH, L]) of DenseBiasAttnGroupsFn's kernel on qkv bf16 [B, L, 3C] and bias fp32
    [nH, L, L]; not differentiable."""
    qkv, bias = _chk(qkv, BF16, "qkv"), _chk(bias, F32, "bias")
    B, L, C3 = qkv.shape
    out = torch.empty(B * L, C3 // 3, dtype=BF16, device=qkv.device)
    lse = torch.empty(B, num_heads, L, dtype=F32, device=qkv.device)
    _lib.call("esvit_vil_dense_fwd", _p(qkv), _p(bias), _p(out), _p(lse), B, L, C3 // 3, num_heads, scale, _stream())
    return out, lse


class VilStreamEmbedFn(Function):
    """PatchEmbed.proj (Conv2d p x p / p, vision_longformer.py:203-204) of stages 2-4, reading the previous stage's
    residual stream x fp32 [T, Cin] directly: group g = (B, N, off, H, W, row0) holds B images of N rows each at rows
    [row0, row0 + B*N), the H x W map rows of an image start at row `off` (the global rows before it are dropped,
    forward_features :584-592).  All groups -> one im2col buffer bf16 [sum B*(H/p)*(W/p), Kp] -> ONE GEMM with the bias
    -> bf16 [rows, Cout].  bias gets its gradient from the consumer (the fused add + LN).  backward: the fp32 weight
    gradient and dx (0 on the global rows)."""

    @staticmethod
    def forward(ctx, x, weight, w16, bias, groups, p: int):
        x, w16 = _chk(x, F32, "x"), _chk(w16, BF16, "w16")
        Cout, Kp = w16.shape
        Cin = x.shape[1]
        if tuple(weight.shape) != (Cout, Cin, p, p):
            raise ValueError(f"weight {tuple(weight.shape)} is not [{Cout}, {Cin}, {p}, {p}]")
        n = [B * (H // p) * (W // p) for B, N, off, H, W, r0 in groups]
        # the im2col writes the K = Cin*p*p columns; padding columns (Kp > K) must be zeros, not garbage
        alloc = torch.empty if Kp == Cin * p * p else torch.zeros
        rows = alloc(sum(n), Kp, dtype=BF16, device=x.device)
        o0 = 0
        for (B, N, off, H, W, r0), ni in zip(groups, n):
            _lib.call("esvit_vil_im2col", _po(x, r0 * Cin), _po(rows, o0 * Kp), B, N, off, Cin, H, W, p, Kp, _stream())
            o0 += ni
        y = gemm(rows, w16, bias)
        ctx.save_for_backward(rows, w16)
        ctx.meta = (tuple(weight.shape), tuple(x.shape), tuple(groups), tuple(n), p)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        rows, w16 = ctx.saved_tensors
        wshape, xshape, groups, n, p = ctx.meta
        g = _chk(g, BF16, "g")
        K = wshape[1] * p * p
        dw = None
        if ctx.needs_input_grad[1]:
            dw = gemm_wgrad(g, rows)
            dw = (dw[:, :K].contiguous() if dw.shape[1] != K else dw).view(wshape)
        dx = None
        if ctx.needs_input_grad[0]:
            drows = gemm(g, w16, None, b_mn=True)
            Kp, Cin = drows.shape[1], xshape[1]
            dx = torch.empty(xshape, dtype=F32, device=g.device)
            o0 = 0
            for (B, N, off, H, W, r0), ni in zip(groups, n):
                _lib.call("esvit_vil_col2im", _po(drows, o0 * Kp), _po(dx, r0 * Cin), B, N, off, Cin, H, W, p, Kp,
                          _stream())
                o0 += ni
        return dx, dw, None, None, None, None


class ClsCatGroupsFn(Function):
    """PatchEmbed's cat(cls_token, x) (vision_longformer.py:240-243) over resolution groups: y fp32 [sum B*n, C] (the
    embedding LN output, groups back to back) -> the residual stream fp32 [sum B*(1+n), C]; groups = ((B, n), ...).
    The cls_token gradient is the fixed-order sum of the global rows' gradient."""

    @staticmethod
    def forward(ctx, y, cls_token, groups):
        y, cls = _chk(y, F32, "y"), _chk(cls_token, F32, "cls_token")
        C = y.shape[1]
        out = torch.empty(sum(B * (1 + n) for B, n in groups), C, dtype=F32, device=y.device)
        y0 = x0 = 0
        for B, n in groups:
            _lib.call("esvit_vil_cls_cat_fwd", _po(y, y0 * C), _p(cls), _po(out, x0 * C), B, n, C, _stream())
            y0 += B * n
            x0 += B * (1 + n)
        ctx.meta = (tuple(groups), tuple(y.shape), tuple(cls_token.shape))
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        groups, yshape, cshape = ctx.meta
        g = _chk(g, F32, "g")
        C = yshape[1]
        dy = torch.empty(yshape, dtype=F32, device=g.device)
        dcls = torch.empty(cshape, dtype=F32, device=g.device)
        y0 = x0 = 0
        for gi, (B, n) in enumerate(groups):
            _lib.call("esvit_vil_cls_cat_bwd", _po(g, x0 * C), _po(dy, y0 * C), _p(dcls), B, n, C, 1 if gi else 0,
                      _stream())
            y0 += B * n
            x0 += B * (1 + n)
        return dy, dcls, None


class RelBiasFn(Function):
    """The relative-position biases of one ViL attention module for every resolution group, as ONE fp32 vector
    y = M . [table | g2l | g2g] (flattened parameters): M is a sparse matrix built once per geometry on the host
    (vision_longformer.bias_plan: gathers, and at other resolutions than the table's the reference's bicubic resize as
    fixed per-axis weights).  backward: d[table | g2l | g2g] = M^T . dy, a gather-sum in a fixed order per parameter
    entry (the transposed CSR), so no atomics.  plan = (M CSR (rowptr, col, val), M^T CSR, nrows) on the device."""

    @staticmethod
    def forward(ctx, table, g2l, g2g, plan):
        table = _chk(table, F32, "table")
        g2l, g2g = _chk(g2l, F32, "g2l"), _chk(g2g, F32, "g2g")
        (rp, col, val), _, nrows = plan
        n0, n1 = table.numel(), (g2l.numel() if g2l is not None else 0)
        y = torch.empty(nrows, dtype=F32, device=table.device)
        _lib.call("esvit_vil_bias_spmv", _p(rp), _p(col), _p(val), _p(table), _p(g2l), _p(g2g), n0, n1, _p(y), nrows,
                  _stream())
        ctx.plan = plan
        ctx.shapes = (tuple(table.shape), None if g2l is None else tuple(g2l.shape),
                      None if g2g is None else tuple(g2g.shape))
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        g = _chk(g, F32, "g")
        _, (rp, col, val), _ = ctx.plan
        shapes = ctx.shapes
        sizes = [0 if s is None else int(torch.Size(s).numel()) for s in shapes]
        d = torch.empty(sum(sizes), dtype=F32, device=g.device)
        _lib.call("esvit_vil_bias_spmv", _p(rp), _p(col), _p(val), _p(g), None, None, g.numel(), 0, _p(d), d.numel(),
                  _stream())
        out, o = [], 0
        for s, n in zip(shapes, sizes):
            out.append(None if s is None else d[o:o + n].view(s))
            o += n
        return out[0], out[1], out[2], None


# ------------------------------------------------------------------------------------------------------------
# optimiser-side multi-tensor ops


def _ptr_array(tensors: Sequence[Tensor]):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def _numel_array(tensors: Sequence[Tensor]):
    arr = (ctypes.c_longlong * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.numel()
    return arr


def ema_update_(teacher: Sequence[Tensor], student: Sequence[Tensor], momentum: float) -> None:
    """teacher = teacher * m + (1 - m) * student for every tensor pair; bit-exact with the reference loop."""
    assert len(teacher) == len(student)
    for k, q in zip(teacher, student):
        if not (k.is_cuda and q.is_cuda and k.dtype == F32 and q.dtype == F32 and k.is_contiguous()
                and q.is_contiguous() and k.numel() == q.numel()):
            raise RuntimeError("ema_update_: fp32 contiguous CUDA tensors of equal size required")
    _lib.call("esvit_ema_multi", _ptr_array(teacher), _ptr_array(student), _numel_array(teacher), len(teacher),
              float(momentum), _stream())


def clip_grads_(grads: Sequence[Tensor], clip: float) -> Tensor:
    """Per-tensor L2 clipping in place; returns the pre-clip norms as a device tensor (no host sync)."""
    n = len(grads)
    dev = grads[0].device
    for g in grads:
        if not (g.is_cuda and g.dtype == F32 and g.is_contiguous()):
            raise RuntimeError("clip_grads_: fp32 contiguous CUDA gradients required")
    ws = torch.empty(n, dtype=torch.float64, device=dev)
    norms = torch.empty(n, dtype=F32, device=dev)
    _lib.call("esvit_clip_multi", _ptr_array(grads), _numel_array(grads), n, float(clip), _p(ws), _p(norms), _stream())
    return norms
