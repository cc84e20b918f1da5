"""H100-native Swin backbone behind the reference's module names, signatures and state_dict keys.

Drop-in for the reference's models/swin_transformer.py on the pre-training path: same constructor arguments,
same parameter / buffer names (teacher.load_state_dict(student.state_dict()) and checkpoints interchange),
``forward(x or list_of_crops)`` returning ``head(cls)`` or the dense 4-tuple exactly as
``SwinTransformer.forward`` (models/swin_transformer.py:713-763).

Execution model (what differs from the reference, see DESIGN.md):
  * the residual stream is fp32 token-major [B, H*W, C]; every branch output is bf16;
  * ``x = shortcut + drop_path(branch)`` is fused with the NEXT LayerNorm (ops.add_layer_norm), so a block is
    LN -> qkv GEMM -> window-attention kernel -> proj GEMM -> add+LN -> fc1 GEMM -> GELU -> fc2 GEMM, with the
    trailing add deferred into the following block / PatchMerging / final norm;
  * pad, cyclic shift, window partition/reverse, the relative-position bias gather and the shift mask never
    exist as tensors - the attention kernel derives them from (H, W, window, shift);
  * the plain GEMMs (qkv, proj, fc1, fc2, reduction) are bf16 library GEMMs (torch.nn.functional.linear).
"""
from __future__ import annotations

import math
import os
from functools import partial
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import linear, ops, shadow

Tensor = torch.Tensor
BF16 = torch.bfloat16


# fc1 + bias + GELU as one wgmma/TMA GEMM (esvit_gemm_bias_act) instead of library GEMM + GELU kernel
USE_TCGEN05_FC1 = os.environ.get("ESVIT_TCGEN05_FC1", "1") != "0"
# run every per-token op (GEMMs, add+LN, MLP) ONCE over the concatenated tokens of all resolution groups of a multi-crop
# forward instead of once per group; attention / patch merging / pooling launch per group on slices of the same buffers
# (SwinTransformer._forward_fused_groups).  ESVIT_FUSE_GROUPS=0 restores the reference's per-group loop.
USE_FUSED_GROUPS = os.environ.get("ESVIT_FUSE_GROUPS", "1") != "0"
# every Linear (forward, input gradient, weight gradient) on the wgmma GEMM family (esvit_b200.linear)
# instead of library GEMMs; ESVIT_GEMM2=0 restores the library-GEMM path of round 1
USE_GEMM2 = os.environ.get("ESVIT_GEMM2", "1") != "0"


def _trunc_normal_(t: Tensor, std: float = .02) -> Tensor:
    return nn.init.trunc_normal_(t, std=std)


def _lin(x: Tensor, w: Tensor, b: Optional[Tensor]) -> Tensor:
    """bf16 library GEMM; fp32 master weights are cast per call (autograd routes the bf16 grads back to fp32)."""
    with torch.autocast("cuda", enabled=False):
        return F.linear(x, w.to(BF16), None if b is None else b.to(BF16))


class _CastCache:
    """bf16 copies of weights shared by the resolution groups of one forward call (one cast per step)."""

    def __init__(self):
        self.d: Dict[int, Tensor] = {}
        self.drop_plan = None  # [(block id, drop_prob)] of the backbone in execution order (set by the backbone)
        self.keep_prob = None  # device fp32 [2*nblk, 1]: 1 - drop_prob per DropPath call
        self.group = 0         # resolution group being run
        self._drop = {}        # (group, batch size) -> {block id: (k1, k2)}

    def drop_keeps(self, batch: int, drop_prob: float, device, key):
        tab = self._drop.get((self.group, batch))
        if tab is None:  # one draw for every block of this resolution group
            r = torch.rand(len(self.drop_plan) * 2, batch, dtype=torch.float32, device=device)
            keeps = r.add_(self.keep_prob).floor_().div_(self.keep_prob)      # timm: floor(keep_prob + U) / keep_prob
            tab = self._drop[(self.group, batch)] = {bid: (keeps[2 * i], keeps[2 * i + 1])
                                                     for i, (bid, _) in enumerate(self.drop_plan)}
        return tab[key]

    def __call__(self, p: Optional[Tensor]) -> Optional[Tensor]:
        if p is None:
            return None
        k = id(p)
        t = self.d.get(k)
        if t is None:
            t = self.d[k] = shadow.as_bf16(p)  # optimiser-maintained bf16 shadow when registered, else a cast
        return t

    def transposed(self, p: Tensor) -> Tensor:
        """bf16 W^T (contiguous) of a 2-D weight: the K-major operand of the fused input-gradient GEMM (ops.MlpFn)."""
        k = ("T", id(p))
        t = self.d.get(k)
        if t is None:
            t = self.d[k] = shadow.as_bf16(p, track_grad=False).t().contiguous()
        return t

    def expanded_bias(self, table: Tensor, num_heads: int, ws: int) -> Optional[Tensor]:
        """the rel-pos bias table expanded once per forward call (ops.expand_rel_pos_bias), shared by the crop groups."""
        k = ("B", id(table))
        if k not in self.d:
            self.d[k] = ops.expand_rel_pos_bias(table, num_heads, ws)
        return self.d[k]

    def nograd(self, p: Tensor) -> Tensor:
        k = ("ng", id(p))
        t = self.d.get(k)
        if t is None:
            t = self.d[k] = shadow.as_bf16(p, track_grad=False)
        return t


def _lin_c(x: Tensor, lin: nn.Linear, cc: Optional[_CastCache]) -> Tensor:
    """bf16 library GEMM x @ W^T + b (bias in the GEMM epilogue).  The bias GRADIENT is not computed here: the consumer
    kernel (window attention / GELU / residual add + LN backward) column-sums it, see ops.LinearBiasFn."""
    if USE_GEMM2:
        w16 = shadow.as_bf16(lin.weight, track_grad=False) if cc is None else cc.nograd(lin.weight)
        return linear.LinearFn.apply(x, lin.weight, w16, lin.bias)
    w = shadow.as_bf16(lin.weight) if cc is None else cc(lin.weight)
    if lin.bias is None:
        with torch.autocast("cuda", enabled=False):
            return F.linear(x, w)
    return ops.LinearBiasFn.apply(x, w, (shadow.as_bf16(lin.bias, False) if cc is None else cc.nograd(lin.bias)))


def drop_path_keep(batch: int, drop_prob: float, training: bool, device) -> Optional[Tensor]:
    """Per-sample stochastic-depth scale (0 or 1/keep_prob) of timm 0.3.2 DropPath; None = identity."""
    if drop_prob == 0. or not training:
        return None
    keep_prob = 1.0 - drop_prob
    r = keep_prob + torch.rand(batch, dtype=torch.float32, device=device)
    return r.floor_().div_(keep_prob)


def drop_path_keeps(batch: int, drop_prob: float, training: bool, device, cc, key):
    """The two DropPath scales of one block (attention branch, MLP branch).  Same distribution as drop_path_keep; the
    uniforms of ALL blocks of one backbone pass are drawn by one torch.rand and turned into scales by two kernels
    (registered in the pass' _CastCache) instead of four tiny kernels per DropPath call (~100 launches per step)."""
    if drop_prob == 0. or not training:
        return None, None
    if cc is None or cc.drop_plan is None:
        return (drop_path_keep(batch, drop_prob, training, device), drop_path_keep(batch, drop_prob, training, device))
    return cc.drop_keeps(batch, drop_prob, device, key)


class Mlp(nn.Module):
    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        if act_layer is not nn.GELU or drop != 0.:
            raise NotImplementedError("the fused path implements exact GELU and drop=0 (all EsViT Swin configs)")
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden_features, out_features)

    def fused(self, x: Tensor, cc: Optional[_CastCache] = None) -> Tensor:
        """x bf16 [..., C] -> fc2(gelu(fc1(x))) bf16.  fc1.bias gets its gradient from the GELU backward kernel; the
        caller must route fc2.bias through the residual-add kernel (ops.add_layer_norm / residual_add delta_bias)."""
        if USE_GEMM2 and self.fc2.bias is not None:
            cc = cc if cc is not None else _CastCache()
            return linear.MlpFn.apply(x, self.fc1.weight, cc.nograd(self.fc1.weight), self.fc1.bias, self.fc2.weight,
                                      cc.nograd(self.fc2.weight), self.fc2.bias)
        if USE_TCGEN05_FC1:
            w1 = shadow.as_bf16(self.fc1.weight) if cc is None else cc(self.fc1.weight)
            if torch.is_grad_enabled() and self.fc1.weight.requires_grad and self.fc2.bias is not None:
                cc = cc if cc is not None else _CastCache()
                return ops.MlpFn.apply(x, w1, self.fc1.bias, cc(self.fc2.weight), cc.nograd(self.fc2.bias),
                                       cc.transposed(self.fc2.weight))
            h = ops.LinearGeluFn.apply(x, w1, self.fc1.bias)
        else:
            h = ops.BiasGeluFn.apply(_lin_c(x, self.fc1, cc), self.fc1.bias)
        return _lin_c(h, self.fc2, cc)

    def forward(self, x: Tensor) -> Tensor:
        """Reference signature (standalone use; fc2.bias receives no gradient on this path - use the block)."""
        return self.fused(x.to(BF16))


class WindowAttention(nn.Module):
    """W-MSA / SW-MSA with relative position bias (models/swin_transformer.py:72-152), head_dim 32."""

    def __init__(self, dim, window_size, num_heads, qkv_bias=True, qk_scale=None, attn_drop=0., proj_drop=0.):
        super().__init__()
        self.dim = dim
        self.window_size = tuple(window_size)
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = qk_scale or head_dim ** -0.5
        if head_dim != 32 or self.window_size[0] != self.window_size[1] or attn_drop != 0. or proj_drop != 0.:
            raise NotImplementedError("kernel supports head_dim 32, square windows, no attention dropout")
        if not qkv_bias:
            raise NotImplementedError("qkv_bias=False is not used by any EsViT config")
        ws = self.window_size[0]
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * ws - 1) * (2 * ws - 1), num_heads))
        t = torch.arange(ws * ws)
        y, x = t // ws, t % ws
        idx = (y[:, None] - y[None, :] + ws - 1) * (2 * ws - 1) + (x[:, None] - x[None, :] + ws - 1)
        self.register_buffer("relative_position_index", idx)  # kept for state_dict parity; the kernel uses the closed form
        self.qkv = nn.Linear(dim, dim * 3, bias=True)
        self.proj = nn.Linear(dim, dim)
        _trunc_normal_(self.relative_position_bias_table, std=.02)

    def attend(self, y: Tensor, H: int, W: int, shift: int, cc: Optional[_CastCache] = None) -> Tensor:
        """y = norm1(x) bf16 [B, H*W, C] in token order -> proj(attention) bf16 [B, H*W, C]; proj.bias gets its gradient
        from the residual-add kernel the caller routes it through."""
        qkv = _lin_c(y, self.qkv, cc)
        ws = self.window_size[0]
        bexp = None if cc is None else cc.expanded_bias(self.relative_position_bias_table, self.num_heads, ws)
        a = ops.WindowAttentionFn.apply(qkv, self.qkv.bias, self.relative_position_bias_table, H, W, self.num_heads,
                                        ws, shift, float(self.scale), bexp)
        return _lin_c(a, self.proj, cc)

    def attend_groups(self, y: Tensor, grp, shift: int, cc: Optional[_CastCache] = None) -> Tensor:
        """attend() for the concatenated tokens [T, C] of several resolution groups grp = [(B, H, W, row0)]."""
        qkv = _lin_c(y, self.qkv, cc)
        ws = self.window_size[0]
        bexp = None if cc is None else cc.expanded_bias(self.relative_position_bias_table, self.num_heads, ws)
        a = ops.WindowAttentionGroupsFn.apply(qkv, self.qkv.bias, self.relative_position_bias_table, tuple(grp),
                                              self.num_heads, ws, shift, float(self.scale), bexp)
        return _lin_c(a, self.proj, cc)

    def forward(self, x: Tensor, mask: Optional[Tensor] = None):
        """Reference signature: x [num_windows*B, N, C] pre-partitioned windows.  Only mask=None is supported
        standalone (the shifted case is handled inside SwinTransformerBlock from the geometry); the attention
        probabilities (2nd return of the reference) are never materialised -> None."""
        if mask is not None:
            raise NotImplementedError("explicit masks are generated in-kernel; call SwinTransformerBlock instead")
        ws = self.window_size[0]
        B_, N, C = x.shape
        assert N == ws * ws
        return self.attend(x.to(BF16), ws, ws, 0), None


class SwinTransformerBlock(nn.Module):
    def __init__(self, dim, input_resolution, num_heads, window_size=7, shift_size=0, mlp_ratio=4., qkv_bias=True,
                 qk_scale=None, drop=0., attn_drop=0., drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.dim, self.input_resolution, self.num_heads = dim, input_resolution, num_heads
        self.window_size, self.shift_size, self.mlp_ratio = window_size, shift_size, mlp_ratio
        if min(self.input_resolution) <= self.window_size:  # models/swin_transformer.py:206-209
            self.shift_size = 0
            self.window_size = min(self.input_resolution)
        assert 0 <= self.shift_size < self.window_size
        self.norm1 = norm_layer(dim)
        self.attn = WindowAttention(dim, (self.window_size, self.window_size), num_heads, qkv_bias, qk_scale,
                                    attn_drop, drop)
        self.drop_prob = float(drop_path)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), act_layer=act_layer, drop=drop)

    def fused(self, x: Tensor, pending, cc: Optional[_CastCache] = None):
        """(x fp32 [B,L,C], pending=(delta bf16, keep, delta_bias) or None) -> (x, pending): the MLP branch's
        residual add (and fc2 bias) is deferred into the next fused add+LN."""
        delta, keep, dbias = pending if pending is not None else (None, None, None)
        B, L, C = (x if x is not None else delta).shape  # x None: the stream starts as fp32(delta) (after PatchMerging)
        H = W = int(math.sqrt(L))
        x, y = ops.add_layer_norm(x, delta, keep, self.norm1.weight, self.norm1.bias, self.norm1.eps, delta_bias=dbias)
        a = self.attn.attend(y, H, W, self.shift_size, cc)
        k1, k2 = drop_path_keeps(B, self.drop_prob, self.training, x.device, cc, id(self))
        x, y = ops.add_layer_norm(x, a, k1, self.norm2.weight, self.norm2.bias, self.norm2.eps,
                                  delta_bias=self.attn.proj.bias)
        z = self.mlp.fused(y, cc)
        return x, (z, k2, self.mlp.fc2.bias)

    def fused_groups(self, x: Optional[Tensor], pending, grp, cc, k1: Optional[Tensor], k2: Optional[Tensor]):
        """fused() over the concatenated tokens x fp32 [T, C] of the resolution groups grp = [(B, H, W, row0)];
        k1 / k2: per-ROW DropPath scales (fp32 [T]) or None."""
        delta, keep, dbias = pending if pending is not None else (None, None, None)
        x, y = ops.add_layer_norm(x, delta, keep, self.norm1.weight, self.norm1.bias, self.norm1.eps, delta_bias=dbias)
        a = self.attn.attend_groups(y, grp, self.shift_size, cc)
        x, y = ops.add_layer_norm(x, a, k1, self.norm2.weight, self.norm2.bias, self.norm2.eps,
                                  delta_bias=self.attn.proj.bias)
        z = self.mlp.fused(y, cc)
        return x, (z, k2, self.mlp.fc2.bias)

    def forward(self, x: Tensor):
        """Reference signature: x [B, L, C] -> (x, attn); attn probabilities are not materialised (None)."""
        x, pend = self.fused(x.float(), None)
        return ops.residual_add(x, *pend), None


class PatchMerging(nn.Module):
    def __init__(self, input_resolution, dim, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim = input_resolution, dim
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = norm_layer(4 * dim)

    def forward(self, x: Tensor, cc: Optional[_CastCache] = None) -> Tensor:
        """x fp32 [B, H*W, C] -> fp32 [B, H*W/4, 2C]."""
        B, L, C = x.shape
        H = W = int(math.sqrt(L))
        return self.fused(x, cc).float()

    def fused(self, x: Tensor, cc: Optional[_CastCache] = None) -> Tensor:
        """-> bf16 [B, H*W/4, 2C]; the caller starts the next stage's fp32 residual stream from it inside the next
        add+LN kernel (ops.add_layer_norm with x=None) instead of a separate cast pass."""
        B, L, C = x.shape
        H = W = int(math.sqrt(L))
        y = ops.PatchMergeLNFn.apply(x, self.norm.weight, self.norm.bias, self.norm.eps, H, W)
        return _lin_c(y, self.reduction, cc)


    def fused_groups(self, x: Tensor, grp, cc: Optional[_CastCache] = None):
        """fused() over concatenated groups: x fp32 [T, C] -> (bf16 [T', 2C], the groups' new geometry)."""
        y = ops.PatchMergeLNGroupsFn.apply(x, self.norm.weight, self.norm.bias, self.norm.eps, tuple(grp))
        new_grp, row0 = [], 0
        for B, H, W, _ in grp:
            Ho, Wo = (H + 1) // 2, (W + 1) // 2
            new_grp.append((B, Ho, Wo, row0))
            row0 += B * Ho * Wo
        return _lin_c(y, self.reduction, cc), new_grp


class BasicLayer(nn.Module):
    def __init__(self, dim, input_resolution, depth, num_heads, window_size, mlp_ratio=4., qkv_bias=True,
                 qk_scale=None, drop=0., attn_drop=0., drop_path=0., norm_layer=nn.LayerNorm, downsample=None):
        super().__init__()
        self.dim, self.input_resolution, self.depth = dim, input_resolution, depth
        self.blocks = nn.ModuleList([
            SwinTransformerBlock(dim=dim, input_resolution=input_resolution, num_heads=num_heads,
                                 window_size=window_size, shift_size=0 if (i % 2 == 0) else window_size // 2,
                                 mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop,
                                 attn_drop=attn_drop,
                                 drop_path=drop_path[i] if isinstance(drop_path, (list, tuple)) else drop_path,
                                 norm_layer=norm_layer) for i in range(depth)])
        self.downsample = downsample(input_resolution, dim=dim, norm_layer=norm_layer) if downsample else None

    def fused(self, x: Optional[Tensor], cc: Optional[_CastCache] = None, pend=None):
        """(x fp32 or None, pend) -> (x, pend).  After a downsample the stream is handed on as (None, (merged bf16, None,
        None)): the next stage's first add+LN turns it into the fp32 residual."""
        for blk in self.blocks:
            x, pend = blk.fused(x, pend, cc)
        if self.downsample is not None:
            x = ops.residual_add(x, *pend)
            return None, (self.downsample.fused(x, cc), None, None)
        return x, pend

    def fused_groups(self, x: Optional[Tensor], pend, grp, cc, keeps: Optional[Tensor]):
        """fused() over concatenated groups; keeps: per-row DropPath scales fp32 [2*depth, T] of this layer or None."""
        for i, blk in enumerate(self.blocks):
            k1 = k2 = None
            if keeps is not None and blk.drop_prob > 0. and blk.training:
                k1, k2 = keeps[2 * i], keeps[2 * i + 1]
            x, pend = blk.fused_groups(x, pend, grp, cc, k1, k2)
        if self.downsample is not None:
            x = ops.residual_add(x, *pend)
            m, grp = self.downsample.fused_groups(x, grp, cc)
            return None, (m, None, None), grp
        return x, pend, grp

    def forward(self, x: Tensor) -> Tensor:
        x, pend = self.fused(x.float())
        if x is None:
            return pend[0].float()
        return x if pend is None else ops.residual_add(x, *pend)

    def forward_with_features(self, x: Tensor):
        """models/swin_transformer.py:483-490: x [B, L, C] -> (x after the downsample, [output of every block]), fp32."""
        x, fea = x.float(), []
        for blk in self.blocks:
            x, pend = blk.fused(x, None)
            x = ops.residual_add(x, *pend)
            fea.append(x)
        if self.downsample is not None:
            x = self.downsample(x)
        return x, fea


class PatchEmbed(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, embed_dim=96, norm_layer=None):
        super().__init__()
        img_size = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        patch_size = (patch_size, patch_size) if isinstance(patch_size, int) else tuple(patch_size)
        if patch_size != (4, 4) or in_chans != 3 or norm_layer is None:
            raise NotImplementedError("kernel supports patch_size=4, in_chans=3, patch_norm=True (all EsViT Swin configs)")
        self.img_size, self.patch_size = img_size, patch_size
        self.patches_resolution = [img_size[0] // 4, img_size[1] // 4]
        self.num_patches = self.patches_resolution[0] * self.patches_resolution[1]
        self.in_chans, self.embed_dim = in_chans, embed_dim
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)  # parameter container
        self.norm = norm_layer(embed_dim)

    def forward(self, x: Tensor) -> Tensor:
        """x fp32 [B,3,H,W] -> fp32 [B, (H/4)(W/4), E]."""
        return ops.PatchEmbedFn.apply(x.float(), self.proj.weight, self.proj.bias, self.norm.weight, self.norm.bias,
                                      self.norm.eps)


class SwinTransformer(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, num_classes=1000, embed_dim=96, depths=[2, 2, 6, 2],
                 num_heads=[3, 6, 12, 24], window_size=7, mlp_ratio=4., qkv_bias=True, qk_scale=None, drop_rate=0.,
                 attn_drop_rate=0., drop_path_rate=0.1, norm_layer=nn.LayerNorm, ape=False, patch_norm=True,
                 use_dense_prediction=False, **kwargs):
        super().__init__()
        if ape or drop_rate != 0. or not patch_norm:
            raise NotImplementedError("ape / dropout / patch_norm=False are not used by any EsViT Swin config")
        self.num_classes = num_classes
        self.num_layers = len(depths)
        self.embed_dim = embed_dim
        self.ape, self.patch_norm = ape, patch_norm
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))
        self.mlp_ratio = mlp_ratio
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim, norm_layer)
        pr = self.patch_embed.patches_resolution
        self.patches_resolution = pr
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        self.layers = nn.ModuleList()
        for i in range(self.num_layers):
            self.layers.append(BasicLayer(
                dim=int(embed_dim * 2 ** i), input_resolution=(pr[0] // (2 ** i), pr[1] // (2 ** i)),
                depth=depths[i], num_heads=num_heads[i], window_size=window_size, mlp_ratio=mlp_ratio,
                qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop_rate, attn_drop=attn_drop_rate,
                drop_path=dpr[sum(depths[:i]):sum(depths[:i + 1])], norm_layer=norm_layer,
                downsample=PatchMerging if i < self.num_layers - 1 else None))
        self.norm = norm_layer(self.num_features)
        self.avgpool = nn.AdaptiveAvgPool1d(1)  # structural parity only; ops.TokenMeanFn does the work
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        self.use_dense_prediction = use_dense_prediction
        if self.use_dense_prediction:
            self.head_dense = None
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            _trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'absolute_pos_embed'}

    @torch.jit.ignore
    def no_weight_decay_keywords(self):
        return {'relative_position_bias_table'}

    def forward_features(self, x: Tensor, cc: Optional[_CastCache] = None):
        """models/swin_transformer.py:678-694 -> pooled fp32 [B, D] (and region fp32 [B, N, D] in dense mode)."""
        x = self.patch_embed(x)
        pend = None
        for layer in self.layers:
            x, pend = layer.fused(x, cc, pend)
        delta, keep, dbias = pend if pend is not None else (None, None, None)
        _, x_region = ops.add_layer_norm(x, delta, keep, self.norm.weight, self.norm.bias, self.norm.eps,
                                         y_bf16=False, delta_bias=dbias)
        pooled = ops.TokenMeanFn.apply(x_region)
        if self.use_dense_prediction:
            return pooled, x_region
        return pooled

    def _row_samples(self, grp, device) -> Tensor:
        """int64 [T]: the (global) sample index of every token row of the concatenated groups (cached per geometry)."""
        cache = self.__dict__.setdefault("_rs_cache", {})
        key = (tuple(grp), device)
        t = cache.get(key)
        if t is None:
            parts, b0 = [], 0
            for B, H, W, _ in grp:
                parts.append(torch.arange(b0, b0 + B, device=device).repeat_interleave(H * W))
                b0 += B
            t = cache[key] = torch.cat(parts)
        return t

    def _forward_fused_groups(self, x, groups, cc):
        """Multi-crop forward with ONE pass over the concatenated tokens of all resolution groups for every per-token op
        (same math and output order as the per-group loop of models/swin_transformer.py:713-763)."""
        imgs, grp, row0 = [], [], 0
        for s, e in groups:
            im = ops.cat_adjacent(x[s:e]).float()
            B, H, W = im.shape[0], im.shape[2] // 4, im.shape[3] // 4
            imgs.append(im)
            grp.append((B, H, W, row0))
            row0 += B * H * W
        pe = self.patch_embed
        # every group's tokens straight into the concatenated stream (fp32 [T, E]); same kernels as PatchEmbed.forward
        xa = ops.PatchEmbedGroupsFn.apply(pe.proj.weight, pe.proj.bias, pe.norm.weight, pe.norm.bias, pe.norm.eps, *imgs)
        dev = xa.device
        keeps_all = None
        if self.training and any(blk.drop_prob > 0. for layer in self.layers for blk in layer.blocks):
            kp = self._keep_prob_column(dev)                                    # [2*nblk, 1]
            r = torch.rand(kp.shape[0], sum(g[0] for g in grp), dtype=torch.float32, device=dev)
            keeps_all = r.add_(kp).floor_().div_(kp)                            # timm DropPath scale per (call, sample)
        pend, off = None, 0
        for layer in self.layers:
            depth = len(layer.blocks)
            keeps = None
            if keeps_all is not None:
                keeps = keeps_all[2 * off:2 * (off + depth)].index_select(1, self._row_samples(grp, dev))
            xa, pend, grp = layer.fused_groups(xa, pend, grp, cc, keeps)
            off += depth
        delta, keep, dbias = pend if pend is not None else (None, None, None)
        _, x_region = ops.add_layer_norm(xa, delta, keep, self.norm.weight, self.norm.bias, self.norm.eps,
                                         y_bf16=False, delta_bias=dbias)
        pooled = ops.TokenMeanGroupsFn.apply(x_region, tuple(grp))
        if self.use_dense_prediction:
            return self.head(pooled), self.head_dense(x_region), x_region, [H * W for _, H, W, _ in grp]
        return self.head(pooled)

    def _keep_prob_column(self, device) -> Tensor:
        """device fp32 [2*nblk, 1] of 1 - drop_prob (two DropPath calls per block), built once per device."""
        cache = self.__dict__.setdefault("_kp_cache", {})
        t = cache.get(device)
        if t is None:
            probs = [[1.0 - blk.drop_prob] for layer in self.layers for blk in layer.blocks for _ in range(2)]
            t = cache[device] = torch.tensor(probs, dtype=torch.float32).to(device)
        return t

    def forward_return_n_last_blocks(self, x: Tensor, n: int = 1, return_patch_avgpool: bool = False, depth=[]):
        """models/swin_transformer.py:799-837 (eval_linear.py's probe features): fp32 [B, sum C_i], the token means of
        the outputs of the last n blocks in execution order; outputs of last-stage blocks go through the final norm
        first.  return_patch_avgpool is ignored, as in the reference.  `depth` must equal the model's depths.

        Runs the fused path of forward_features: only a tapped block's output is materialised (residual_add), and the
        stream continues from it; the last block's normed output is the final add+LN output itself."""
        depths = [len(layer.blocks) for layer in self.layers]
        if [int(d) for d in depth] != depths:
            raise ValueError(f"depth {list(depth)} does not match the model's depths {depths}")
        total = sum(depths)
        if not 1 <= int(n) <= total:
            raise ValueError(f"n must be in [1, {total}], got {n}")
        start, last = total - int(n), len(self.layers) - 1
        cc = _CastCache()
        x = self.patch_embed(x)
        pend, out, b = None, [], 0
        for i, layer in enumerate(self.layers):
            for j, blk in enumerate(layer.blocks):
                x, pend = blk.fused(x, pend, cc)
                if b >= start and not (i == last and j == len(layer.blocks) - 1):
                    x, pend = ops.residual_add(x, *pend), None
                    y = ops.LayerNormFn.apply(x, self.norm.weight, self.norm.bias, self.norm.eps, False) if i == last else x
                    out.append(ops.TokenMeanFn.apply(y))
                b += 1
            if layer.downsample is not None:
                if pend is not None:
                    x = ops.residual_add(x, *pend)
                x, pend = None, (layer.downsample.fused(x, cc), None, None)
        delta, keep, dbias = pend if pend is not None else (None, None, None)
        _, x_region = ops.add_layer_norm(x, delta, keep, self.norm.weight, self.norm.bias, self.norm.eps,
                                         y_bf16=False, delta_bias=dbias)
        out.append(ops.TokenMeanFn.apply(x_region))
        return torch.cat(out, dim=-1)

    def forward_feature_maps(self, x: Tensor):
        d = self.use_dense_prediction
        self.use_dense_prediction = True
        try:
            return self.forward_features(x)
        finally:
            self.use_dense_prediction = d

    def forward(self, x):
        """Multi-crop forward (models/swin_transformer.py:713-763): consecutive same-resolution crops are
        concatenated on the batch axis and run once; outputs are concatenated crop-major."""
        if not isinstance(x, list):
            x = [x]
        cc = _CastCache()
        if self.training:
            cc.drop_plan = [(id(blk), blk.drop_prob) for layer in self.layers for blk in layer.blocks]
            cc.keep_prob = self._keep_prob_column(x[0].device)
        groups, start = [], 0
        for i in range(1, len(x) + 1):
            if i == len(x) or x[i].shape[-1] != x[start].shape[-1]:
                groups.append((start, i))
                start = i
        if USE_FUSED_GROUPS:
            return self._forward_fused_groups(x, groups, cc)
        if self.use_dense_prediction:
            cls_l, fea_l, npatch = [], [], []
            for gi, (s, e) in enumerate(groups):
                cc.group = gi
                pooled, region = self.forward_features(ops.cat_adjacent(x[s:e]), cc)
                B, N, C = region.shape
                cls_l.append(pooled)
                fea_l.append(region.reshape(B * N, C))
                npatch.append(N)
            output_cls = torch.cat(cls_l) if len(cls_l) > 1 else cls_l[0]
            output_fea = torch.cat(fea_l) if len(fea_l) > 1 else fea_l[0]
            return self.head(output_cls), self.head_dense(output_fea), output_fea, npatch
        outs = []
        for gi, (s, e) in enumerate(groups):
            cc.group = gi
            outs.append(self.forward_features(torch.cat(x[s:e]) if e - s > 1 else x[s], cc))
        return self.head(torch.cat(outs) if len(outs) > 1 else outs[0])


def get_cls_model(config, is_teacher=False, use_dense_prediction=False, **kwargs):
    """Same contract as models/swin_transformer.py:947-978 (yacs config in, nn.Module out)."""
    spec = config.MODEL.SPEC
    return SwinTransformer(
        img_size=config.TRAIN.IMAGE_SIZE[0], in_chans=3, num_classes=config.MODEL.NUM_CLASSES,
        patch_size=spec['PATCH_SIZE'], embed_dim=spec['DIM_EMBED'], depths=spec['DEPTHS'],
        num_heads=spec['NUM_HEADS'], window_size=spec['WINDOW_SIZE'], mlp_ratio=spec['MLP_RATIO'],
        qkv_bias=spec['QKV_BIAS'], drop_rate=spec['DROP_RATE'], attn_drop_rate=spec['ATTN_DROP_RATE'],
        drop_path_rate=0.0 if is_teacher else spec['DROP_PATH_RATE'], norm_layer=partial(nn.LayerNorm, eps=1e-6),
        ape=spec['USE_APE'], patch_norm=spec['PATCH_NORM'], use_dense_prediction=use_dense_prediction)
