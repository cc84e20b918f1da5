"""H100-native Swin backbone behind the reference's module names, signatures and state_dict keys.

Drop-in for the reference's models/swin_transformer.py on the pre-training path: same constructor arguments,
same parameter / buffer names (teacher.load_state_dict(student.state_dict()) and checkpoints interchange),
``forward(x or list_of_crops)`` returning ``head(cls)`` or the dense 4-tuple exactly as
``SwinTransformer.forward`` (models/swin_transformer.py:713-763).

Execution model (what differs from the reference, see DESIGN.md):
  * every entry point runs one path: the resolution groups of a call (one group per crop size; a plain batch is one
    group) are stored back to back in ONE fp32 token-major residual stream [T, C], described by the geometry
    grp = ((B, H, W, row0), ...); every per-token op runs once over all of them; every branch output is bf16;
  * ``x = shortcut + drop_path(branch)`` is fused with the NEXT LayerNorm (ops.add_layer_norm), so a block is
    LN -> qkv GEMM -> window-attention kernel -> proj GEMM -> add+LN -> fc1 GEMM -> GELU -> fc2 GEMM, with the
    trailing add deferred into the following block / PatchMerging / final norm;
  * pad, cyclic shift, window partition/reverse, the relative-position bias gather and the shift mask never
    exist as tensors - the attention kernel derives them from (H, W, window, shift);
  * the plain GEMMs (qkv, proj, fc1, fc2, reduction) run on the wgmma GEMM family (esvit_b200.linear).
"""
from __future__ import annotations

import math
from functools import partial
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

from . import backbone, linear, ops, shadow
from .backbone import MultiCropBackbone, _CastCache

Tensor = torch.Tensor
BF16 = torch.bfloat16


def _trunc_normal_(t: Tensor, std: float = .02) -> Tensor:
    return nn.init.trunc_normal_(t, std=std)


def _lin_c(x: Tensor, lin: nn.Linear, cc: Optional[_CastCache]) -> Tensor:
    """x @ W^T + b on the wgmma GEMM family (bias in the GEMM epilogue).  The bias GRADIENT is not computed here: the
    consumer kernel (window attention / residual add + LN backward) column-sums it, see linear.LinearFn."""
    w16 = shadow.as_bf16(lin.weight) if cc is None else cc.nograd(lin.weight)
    return linear.LinearFn.apply(x, lin.weight, w16, lin.bias)


def _one_group(x: Tensor):
    """a [B, H*W, C] batch of square maps as the stream of one resolution group -> (x [B*H*W, C], grp)"""
    B, L, C = x.shape
    H = int(math.sqrt(L))
    return x.reshape(B * L, C), ((B, H, H, 0),)


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
        """x bf16 [..., C] -> fc2(gelu(fc1(x))) bf16.  fc1.bias gets its gradient from the fused GELU backward (see
        linear.MlpFn); the caller must route fc2.bias through the residual-add kernel (ops.add_layer_norm /
        residual_add delta_bias)."""
        cc = cc if cc is not None else _CastCache()
        return linear.MlpFn.apply(x, self.fc1.weight, cc.nograd(self.fc1.weight), self.fc1.bias, self.fc2.weight,
                                  cc.nograd(self.fc2.weight), self.fc2.bias)

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

    def attend(self, y: Tensor, grp, shift: int, cc: Optional[_CastCache] = None,
               maps: Optional[List[Tensor]] = None) -> Tensor:
        """y = norm1(x) bf16 [T, C] in token order of the resolution groups grp = ((B, H, W, row0), ...) ->
        proj(attention) bf16 [T, C]; proj.bias gets its gradient from the residual-add kernel the caller routes it
        through.  maps: a list to append the attention probabilities to (ops.window_attention_probs, fp32
        [B*nW, nH, N, N]; one group only), or None."""
        qkv = _lin_c(y, self.qkv, cc)
        ws = self.window_size[0]
        bexp = None if cc is None else cc.expanded_bias(self.relative_position_bias_table, self.num_heads, ws)
        a = ops.WindowAttentionGroupsFn.apply(qkv, self.qkv.bias, self.relative_position_bias_table, tuple(grp),
                                              self.num_heads, ws, shift, float(self.scale), bexp)
        if maps is not None:
            (B, H, W, _), = grp
            maps.append(ops.window_attention_probs(qkv.view(B, H * W, -1), self.qkv.bias,
                                                   self.relative_position_bias_table, H, W, self.num_heads, ws, shift,
                                                   float(self.scale), bexp))
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
        return self.attend(x.to(BF16).reshape(B_ * N, C), ((B_, ws, ws, 0),), 0).view(B_, N, C), None


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

    def fused(self, x: Optional[Tensor], pending, grp, cc: Optional[_CastCache], k1: Optional[Tensor],
              k2: Optional[Tensor], maps: Optional[List[Tensor]] = None):
        """backbone.pre_norm_block over the resolution groups grp = ((B, H, W, row0), ...); x None: the stream starts
        after PatchMerging.  maps: see WindowAttention.attend."""
        return backbone.pre_norm_block(x, pending, self.norm1,
                                       lambda y: self.attn.attend(y, grp, self.shift_size, cc, maps), self.norm2,
                                       self.attn.proj.bias, lambda y: self.mlp.fused(y, cc), self.mlp.fc2.bias, k1, k2)

    def forward(self, x: Tensor):
        """Reference signature: x [B, L, C] -> (x, attn); attn probabilities are not materialised (None)."""
        xs, grp = _one_group(x.float())
        xs, pend = self.fused(xs, None, grp, None, *backbone.block_keeps(self, x.shape[0], x.shape[1], x.device))
        return ops.residual_add(xs, *pend).view(x.shape), None


class PatchMerging(nn.Module):
    def __init__(self, input_resolution, dim, norm_layer=nn.LayerNorm):
        super().__init__()
        self.input_resolution, self.dim = input_resolution, dim
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = norm_layer(4 * dim)

    def forward(self, x: Tensor) -> Tensor:
        """x fp32 [B, H*W, C] -> fp32 [B, ceil(H/2)*ceil(W/2), 2C]."""
        xs, grp = _one_group(x)
        m, _ = self.fused(xs, grp)
        return m.float().view(x.shape[0], -1, m.shape[-1])

    def fused(self, x: Tensor, grp, cc: Optional[_CastCache] = None):
        """x fp32 [T, C] of the resolution groups grp = ((B, H, W, row0), ...) -> (bf16 [T', 2C], the groups' new
        geometry); the caller starts the next stage's fp32 residual stream from it inside the next add+LN kernel
        (ops.add_layer_norm with x=None) instead of a separate cast pass."""
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

    def fused(self, x: Optional[Tensor], pend, grp, cc: Optional[_CastCache], keeps: Optional[Sequence[Tensor]],
              maps: Optional[Sequence[Optional[List[Tensor]]]] = None, taps=None):
        """(x fp32 [T, C] or None, pend) over the resolution groups grp = ((B, H, W, row0), ...) -> (x, pend, grp after
        the downsample).  After a downsample the stream is handed on as (None, (merged bf16, None, None)): the next
        stage's first add+LN turns it into the fp32 residual.  keeps: per-row DropPath scales [2*depth][T] of this
        layer or None.  Per block j: maps[j] is the list its attention probabilities are appended to, or None;
        taps: see backbone.tap, called with grp."""
        for j, blk in enumerate(self.blocks):
            k1 = k2 = None
            if keeps is not None and blk.drop_prob > 0. and blk.training:
                k1, k2 = keeps[2 * j], keeps[2 * j + 1]
            x, pend = blk.fused(x, pend, grp, cc, k1, k2, None if maps is None else maps[j])
            x, pend = backbone.tap(taps, j, x, pend, grp)
        if self.downsample is not None:
            if pend is not None:
                x = ops.residual_add(x, *pend)
            m, grp = self.downsample.fused(x, grp, cc)
            return None, (m, None, None), grp
        return x, pend, grp

    def _forward(self, x: Tensor, maps=None, taps=None) -> Tensor:
        """x [B, L, C] as one group through fused() -> fp32 [B, L', C'] after the downsample"""
        B, L, _ = x.shape
        keeps = [k for blk in self.blocks for k in backbone.block_keeps(blk, B, L, x.device)]
        xs, grp = _one_group(x.float())
        xs, pend, _ = self.fused(xs, None, grp, None, keeps, maps, taps)
        if xs is None:  # after the downsample: the merged bf16 tokens
            xs = pend[0].float()
        elif pend is not None:
            xs = ops.residual_add(xs, *pend)
        return xs.view(B, -1, xs.shape[-1])

    def forward(self, x: Tensor) -> Tensor:
        return self._forward(x)

    def forward_with_attention(self, x: Tensor):
        """models/swin_transformer.py:492-499: x [B, L, C] -> (x after the downsample, [attention probabilities of
        every block, fp32 [B*nW, nH, N, N]]).  The probabilities do not require grad."""
        maps = []
        return self._forward(x, maps=[maps] * len(self.blocks)), maps

    def forward_with_features(self, x: Tensor):
        """models/swin_transformer.py:483-490: x [B, L, C] -> (x after the downsample, [output of every block]), fp32."""
        B, L, _ = x.shape
        fea = []
        y = self._forward(x, taps=[lambda xs, grp: fea.append(xs.view(B, L, -1))] * len(self.blocks))
        return y, fea


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

    def fused(self, imgs: Sequence[Tensor]):
        """fp32 crops, one [B_g, 3, S_g, S_g] tensor per resolution group -> (the residual stream fp32 [T, E] with the
        groups back to back, grp = ((B, H, W, row0), ...))."""
        grp, row0 = [], 0
        for im in imgs:
            B, H, W = im.shape[0], im.shape[2] // 4, im.shape[3] // 4
            grp.append((B, H, W, row0))
            row0 += B * H * W
        x = ops.PatchEmbedGroupsFn.apply(self.proj.weight, self.proj.bias, self.norm.weight, self.norm.bias,
                                         self.norm.eps, *imgs)
        return x, grp

    def forward(self, x: Tensor) -> Tensor:
        """x fp32 [B,3,H,W] -> fp32 [B, (H/4)(W/4), E]."""
        xs, _ = self.fused([x.float()])
        return xs.view(x.shape[0], -1, xs.shape[-1])


class SwinTransformer(MultiCropBackbone):
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
        self.avgpool = nn.AdaptiveAvgPool1d(1)  # structural parity only; ops.TokenMeanGroupsFn does the work
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

    def _depths(self) -> List[int]:
        return [len(layer.blocks) for layer in self.layers]

    def _run(self, x, taps=None, maps=None):
        """The backbone with ONE pass over the concatenated tokens of all resolution groups for every per-token op (same
        math and output order as the per-group loop of models/swin_transformer.py:713-763).  x: fp32 crops, one
        [B_g, 3, S_g, S_g] tensor per group, or patch-embedded tokens fp32 [B, L, C] (one group) -> (stream fp32 [T, C]
        or None, pending (delta, keep, delta_bias) or None, the last stage's grp = ((B, H, W, row0), ...)).
        taps / maps: None or one entry per block in execution order, see BasicLayer.fused."""
        cc = _CastCache()
        x, grp = _one_group(x) if isinstance(x, Tensor) else self.patch_embed.fused(x)
        dev = x.device
        probs = [blk.drop_prob for layer in self.layers for blk in layer.blocks for _ in range(2)]
        scales = backbone.drop_path_scales(self, probs, sum(g[0] for g in grp), dev)
        pend, b = None, 0
        for layer in self.layers:
            d = len(layer.blocks)
            keeps = backbone.drop_path_rows(self, None if scales is None else scales[2 * b:2 * (b + d)],
                                            [(B, H * W) for B, H, W, _ in grp], dev)
            x, pend, grp = layer.fused(x, pend, grp, cc, keeps, None if maps is None else maps[b:b + d],
                                       None if taps is None else taps[b:b + d])
            b += d
        return x, pend, grp

    def _features(self, imgs: List[Tensor], taps=None):
        """-> (pooled fp32 [sum B, D], region fp32 [T, D] = the final norm's tokens, tokens per image of each group)"""
        x, pend, grp = self._run(imgs, taps)
        region = self._final_norm(x, pend)
        return ops.TokenMeanGroupsFn.apply(region, tuple(grp)), region, [H * W for _, H, W, _ in grp]

    def _tap_feature(self, i: int, x: Tensor, grp) -> Tensor:
        """models/swin_transformer.py:799-837: the token mean of a block's output"""
        return ops.TokenMeanGroupsFn.apply(x, tuple(grp))

    def _attention_maps(self, x, last: bool):
        """_run's input -> the last block's attention probabilities (last) or every block's in execution order; only
        the blocks asked for compute them."""
        nblk = sum(len(layer.blocks) for layer in self.layers)
        maps = []
        self._run(x, maps=[None] * (nblk - 1) + [maps] if last else [maps] * nblk)
        return maps[0] if last else maps

    @torch.no_grad()
    def forward_selfattention(self, x: Tensor, n: int = 1):
        """models/swin_transformer.py:766-778 (analyze_models.py's attention maps): images fp32 [B, 3, S, S] -> the last
        block's attention probabilities if n == 1, else the list of every block's in execution order.  Each is fp32
        [B*nW, nH, N, N] with the block's window (N = ws*ws) and windows in the reference's window_partition order of
        the padded, rolled map; rows and columns of padded slots are included."""
        if x.dim() != 4 or x.shape[2] != x.shape[3] or x.shape[2] % 4 != 0:
            raise ValueError(f"expected square images [B, 3, S, S] with S a multiple of 4, got {tuple(x.shape)}")
        return self._attention_maps([x.float()], n == 1)

    def _check_tokens(self, x: Tensor) -> Tensor:
        side = math.isqrt(x.shape[1]) if x.dim() == 3 else 0
        if x.dim() != 3 or side * side != x.shape[1] or x.shape[2] != self.embed_dim:
            raise ValueError(f"expected patch-embedded tokens [B, S*S, {self.embed_dim}], got {tuple(x.shape)}")
        return x.float()

    @torch.no_grad()
    def forward_last_selfattention(self, x: Tensor) -> Tensor:
        """models/swin_transformer.py:780-787: patch-embedded tokens [B, L, C] -> the last block's probabilities."""
        return self._attention_maps(self._check_tokens(x), True)

    @torch.no_grad()
    def forward_all_selfattention(self, x: Tensor) -> List[Tensor]:
        """models/swin_transformer.py:789-796: patch-embedded tokens [B, L, C] -> every block's probabilities in execution
        order (sum(depths) tensors)."""
        return self._attention_maps(self._check_tokens(x), False)

    def forward_feature_maps(self, x: Tensor):
        d = self.use_dense_prediction
        self.use_dense_prediction = True
        try:
            return self.forward_features(x)
        finally:
            self.use_dense_prediction = d


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
