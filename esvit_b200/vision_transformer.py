"""ViT / DeiT backbones and DINOHead behind the reference's signatures and state_dict keys
(models/vision_transformer.py).

VisionTransformer / Block / Attention / PatchEmbed / deit_tiny / deit_small / vit_base take the reference's constructor
arguments and hold the reference's parameters (``cls_token``, ``pos_embed``, ``patch_embed.proj.*``,
``blocks.i.{norm1,attn.qkv,attn.proj,norm2,mlp.fc1,mlp.fc2}.*``, ``norm.*``).  Execution follows the Swin port
(swin_transformer.py): fp32 residual stream token-major [T, D], bf16 branches, the residual add + DropPath fused into the
next LayerNorm, every Linear on the wgmma GEMM family, and every per-token op run ONCE over the tokens of all resolution
groups of a multi-crop forward.  The attention core is esvit_mhsa_fwd / _bwd (csrc/mhsa.cu), the token embedding
csrc/vit_embed.cu.

DINOHead (:384-418): mlp.{0,2,4} Linear(+exact GELU) -> L2 normalise -> weight-normed Linear(bottleneck, out_dim,
bias=False), with parameters ``mlp.N.{weight,bias}``, ``last_layer.weight_g`` [K,1], ``last_layer.weight_v`` [K,D].
The three MLP GEMMs and the last-layer GEMM are bf16 library GEMMs; GELU, the row normalisation and the
weight-norm reparameterisation (fwd + bwd) are esvit_b200 kernels.  Output logits are bf16 [rows, out_dim]
(what the reference produces under autocast); the losses consume them without an fp32 copy.
"""
from __future__ import annotations

import math
from functools import partial
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import linear, ops, shadow
from .swin_transformer import USE_GEMM2, Mlp, _CastCache, _lin_c, drop_path_keep

Tensor = torch.Tensor

BF16 = torch.bfloat16


class _WeightNormLinear(nn.Module):
    """Parameter container with the names nn.utils.weight_norm(nn.Linear(..., bias=False)) registers."""

    def __init__(self, in_features: int, out_features: int):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        lin = nn.Linear(in_features, out_features, bias=False)  # same default init stream as the reference
        self.weight_g = nn.Parameter(lin.weight.detach().norm(2, dim=1, keepdim=True))
        self.weight_v = nn.Parameter(lin.weight.detach().clone())

    def effective_weight(self) -> torch.Tensor:
        return ops.WeightNormFn.apply(self.weight_v, self.weight_g)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if USE_GEMM2:
            return linear.LastLayerFn.apply(x, self.effective_weight())
        with torch.autocast("cuda", enabled=False):
            return F.linear(x, self.effective_weight())


class DINOHead(nn.Module):
    def __init__(self, in_dim, out_dim, use_bn=False, norm_last_layer=True, nlayers=3, hidden_dim=2048,
                 bottleneck_dim=256):
        super().__init__()
        if use_bn:
            raise NotImplementedError("use_bn_in_head is False in every EsViT recipe")
        nlayers = max(nlayers, 1)
        if nlayers == 1:
            self.mlp = nn.Linear(in_dim, bottleneck_dim)
        else:
            layers = [nn.Linear(in_dim, hidden_dim), nn.GELU()]
            for _ in range(nlayers - 2):
                layers += [nn.Linear(hidden_dim, hidden_dim), nn.GELU()]
            layers.append(nn.Linear(hidden_dim, bottleneck_dim))
            self.mlp = nn.Sequential(*layers)
        self.apply(self._init_weights)
        self.last_layer = _WeightNormLinear(bottleneck_dim, out_dim)
        self.last_layer.weight_g.data.fill_(1)
        if norm_last_layer:
            self.last_layer.weight_g.requires_grad = False

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x.to(BF16)
        mods = [self.mlp] if isinstance(self.mlp, nn.Linear) else list(self.mlp)
        lins = [m for m in mods if isinstance(m, nn.Linear)]
        if USE_GEMM2 and len(lins) == 3 and len(mods) == 5:
            args = []
            for m in lins:
                args += [m.weight, shadow.as_bf16(m.weight, track_grad=False), m.bias]
            x = linear.HeadMlpFn.apply(x, *args)
            return self.last_layer(ops.L2NormFn.apply(x, 1e-12))
        with torch.autocast("cuda", enabled=False):
            for i, m in enumerate(mods):
                if not isinstance(m, nn.Linear):
                    continue
                if i + 1 < len(mods) and isinstance(mods[i + 1], nn.GELU):
                    # GEMM with bias epilogue; exact GELU kernel whose backward also yields the bias gradient
                    x = ops.BiasGeluFn.apply(
                        ops.LinearBiasFn.apply(x, shadow.as_bf16(m.weight), shadow.as_bf16(m.bias, False)), m.bias)
                else:
                    x = F.linear(x, shadow.as_bf16(m.weight), shadow.as_bf16(m.bias))
        x = ops.L2NormFn.apply(x, 1e-12)
        return self.last_layer(x)


# ---------------------------------------------------------------------------------------------------------------------
# ViT backbone (models/vision_transformer.py:71-381)


class Attention(nn.Module):
    """models/vision_transformer.py:71-95 with head dim 64 (every ViT / DeiT of the reference)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0.):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        if head_dim * num_heads != dim or head_dim != 64 or attn_drop != 0. or proj_drop != 0.:
            raise NotImplementedError("the attention kernel supports head_dim 64 and no attention / projection dropout")
        self.scale = qk_scale or head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)

    def attend_groups(self, y: Tensor, grp, cc: Optional[_CastCache] = None) -> Tensor:
        """y = norm1(x) bf16 [T, C] of the sequences grp = ((B, L, row0), ...) -> proj(attention) bf16 [T, C]; proj.bias
        gets its gradient from the residual-add kernel the caller routes it through."""
        qkv = _lin_c(y, self.qkv, cc)
        a = ops.MhsaGroupsFn.apply(qkv, self.qkv.bias, tuple(grp), self.num_heads, float(self.scale))
        return _lin_c(a, self.proj, cc)

    def forward(self, x: Tensor):
        """Reference signature: x [B, N, C] -> (bf16 [B, N, C], None); the probabilities are not materialised, and
        proj.bias receives no gradient on this standalone path (use the block)."""
        B, N, C = x.shape
        return self.attend_groups(x.to(torch.bfloat16).reshape(B * N, C), ((B, N, 0),)).view(B, N, C), None


class Block(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop=0., attn_drop=0.,
                 drop_path=0., act_layer=nn.GELU, norm_layer=nn.LayerNorm):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                              proj_drop=drop)
        self.drop_prob = float(drop_path)
        self.norm2 = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), act_layer=act_layer, drop=drop)

    def fused_groups(self, x: Optional[Tensor], pending, grp, cc, k1: Optional[Tensor], k2: Optional[Tensor]):
        """(x fp32 [T, C], pending = (delta bf16, keep, delta_bias) or None) -> (x, pending): the MLP branch's residual
        add is deferred into the next fused add+LN.  k1 / k2: per-ROW DropPath scales fp32 [T] or None."""
        delta, keep, dbias = pending if pending is not None else (None, None, None)
        x, y = ops.add_layer_norm(x, delta, keep, self.norm1.weight, self.norm1.bias, self.norm1.eps, delta_bias=dbias)
        a = self.attn.attend_groups(y, grp, cc)
        x, y = ops.add_layer_norm(x, a, k1, self.norm2.weight, self.norm2.bias, self.norm2.eps,
                                  delta_bias=self.attn.proj.bias)
        z = self.mlp.fused(y, cc)
        return x, (z, k2, self.mlp.fc2.bias)

    def forward(self, x: Tensor, return_attention: bool = False) -> Tensor:
        """Reference signature (:110-116): x [B, N, C] -> fp32 [B, N, C]."""
        if return_attention:
            raise NotImplementedError("ViT attention maps are not implemented (forward_selfattention)")
        B, N, C = x.shape
        k1 = k2 = None
        if self.training and self.drop_prob > 0.:
            k1 = drop_path_keep(B, self.drop_prob, True, x.device).repeat_interleave(N)
            k2 = drop_path_keep(B, self.drop_prob, True, x.device).repeat_interleave(N)
        xs, pend = self.fused_groups(x.float().reshape(B * N, C), None, ((B, N, 0),), _CastCache(), k1, k2)
        return ops.residual_add(xs, *pend).view(B, N, C)


class PatchEmbed(nn.Module):
    """models/vision_transformer.py:124-139: Conv2d(3, D, p, stride p) as a patch gather + GEMM."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768):
        super().__init__()
        if in_chans != 3 or patch_size % 2 != 0:
            raise NotImplementedError("the patch kernels support in_chans=3 and an even patch size")
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size // patch_size) * (img_size // patch_size)
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)

    def embed(self, imgs: Sequence[Tensor], cc: Optional[_CastCache] = None) -> Tensor:
        """fp32 crops [B_g, 3, S_g, S_g] -> patch projections bf16 [sum_g B_g N_g, D] (bias included), back to back.
        proj.bias gets its gradient from the consumer (ops.VitTokensGroupsFn)."""
        w = self.proj.weight
        w16 = (shadow.as_bf16(w, track_grad=False) if cc is None else cc.nograd(w)).view(w.shape[0], -1)
        return linear.LinearFn.apply(ops.vit_patches(imgs, self.patch_size), w, w16, self.proj.bias)

    def forward(self, x: Tensor) -> Tensor:
        """x fp32 [B, 3, S, S] -> fp32 [B, N, D] (bf16 GEMM output; proj.bias receives no gradient on this path)."""
        B = x.shape[0]
        pe = self.embed([x.float()])
        return pe.float().view(B, -1, pe.shape[-1])


class VisionTransformer(nn.Module):
    """models/vision_transformer.py:142-360."""

    def __init__(self, img_size=[224], patch_size=16, in_chans=3, num_classes=0, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=False, qk_scale=None, drop_rate=0., attn_drop_rate=0.,
                 drop_path_rate=0., norm_layer=nn.LayerNorm, use_dense_prediction=False, **kwargs):
        super().__init__()
        if drop_rate != 0.:
            raise NotImplementedError("dropout is not used by any EsViT ViT config")
        self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size=img_size[0], patch_size=patch_size, in_chans=in_chans,
                                      embed_dim=embed_dim)
        num_patches = self.patch_embed.num_patches
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, num_patches + 1, embed_dim))
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]
        self.blocks = nn.ModuleList([
            Block(dim=embed_dim, num_heads=num_heads, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias, qk_scale=qk_scale,
                  drop=drop_rate, attn_drop=attn_drop_rate, drop_path=dpr[i], norm_layer=norm_layer)
            for i in range(depth)])
        self.norm = norm_layer(embed_dim)
        self.head = nn.Linear(embed_dim, num_classes) if num_classes > 0 else nn.Identity()
        self.use_dense_prediction = use_dense_prediction
        if self.use_dense_prediction:
            self.head_dense = None
        nn.init.trunc_normal_(self.pos_embed, std=.02)
        nn.init.trunc_normal_(self.cls_token, std=.02)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def interpolate_pos_encoding(self, x, pos_embed):
        """:271-285, the reference's call: bicubic resampling of the patch positions by scale_factor (parameter-sized
        plumbing, differentiated by torch)."""
        npatch = x.shape[1] - 1
        N = pos_embed.shape[1] - 1
        if npatch == N:
            return pos_embed
        class_emb = pos_embed[:, 0]
        pos_embed = pos_embed[:, 1:]
        dim = x.shape[-1]
        pos_embed = F.interpolate(
            pos_embed.reshape(1, int(math.sqrt(N)), int(math.sqrt(N)), dim).permute(0, 3, 1, 2),
            scale_factor=math.sqrt(npatch / N), mode='bicubic')
        pos_embed = pos_embed.permute(0, 2, 3, 1).reshape(1, -1, dim)
        return torch.cat((class_emb.unsqueeze(0), pos_embed), dim=1)

    # ---- the fused path ---------------------------------------------------------------------------------------
    def _embed(self, imgs: List[Tensor], cc: _CastCache):
        """fp32 crops (one tensor per resolution group) -> (residual stream fp32 [T, D], sequences ((B, 1+N, row0), ...),
        token groups ((B, N), ...))."""
        p = self.patch_embed.patch_size
        for im in imgs:
            if im.dim() != 4 or im.shape[2] != im.shape[3] or im.shape[2] % p != 0:
                raise ValueError(f"expected square images [B, 3, S, S] with S a multiple of {p}, got {tuple(im.shape)}")
        pe = self.patch_embed.embed(imgs, cc)
        tg = tuple((im.shape[0], (im.shape[2] // p) ** 2) for im in imgs)
        D = self.embed_dim
        pos = [self.interpolate_pos_encoding(torch.empty(0, N + 1, D, device="meta"), self.pos_embed) for _, N in tg]
        x = ops.VitTokensGroupsFn.apply(pe, self.patch_embed.proj.bias, self.cls_token, tg, *pos)
        grp, r0 = [], 0
        for B, N in tg:
            grp.append((B, N + 1, r0))
            r0 += B * (N + 1)
        return x, tuple(grp), tg

    def _keeps(self, grp, device) -> Optional[Tensor]:
        """per-row DropPath scales fp32 [2*depth, T] (timm: floor(keep_prob + U) / keep_prob per (call, sample)), drawn
        by one torch.rand as SwinTransformer._run does; None when no block drops."""
        if not self.training or not any(blk.drop_prob > 0. for blk in self.blocks):
            return None
        cache = self.__dict__.setdefault("_kp_cache", {})
        kp = cache.get(device)
        if kp is None:
            kp = cache[device] = torch.tensor([[1.0 - blk.drop_prob] for blk in self.blocks for _ in range(2)],
                                              dtype=torch.float32).to(device)
        rows = self.__dict__.setdefault("_rs_cache", {})
        rs = rows.get((grp, device))
        if rs is None:
            if len(rows) >= 8:  # a handful of crop geometries per run; keep the cache from growing with odd batches
                rows.clear()
            parts, b0 = [], 0
            for B, L, _ in grp:
                parts.append(torch.arange(b0, b0 + B, device=device).repeat_interleave(L))
                b0 += B
            rs = rows[(grp, device)] = torch.cat(parts)
        r = torch.rand(kp.shape[0], sum(g[0] for g in grp), dtype=torch.float32, device=device)
        return r.add_(kp).floor_().div_(kp).index_select(1, rs)

    def _final_norm(self, x: Tensor, pend) -> Tensor:
        delta, keep, dbias = pend if pend is not None else (None, None, None)
        _, y = ops.add_layer_norm(x, delta, keep, self.norm.weight, self.norm.bias, self.norm.eps, y_bf16=False,
                                  delta_bias=dbias)
        return y

    def _run(self, imgs: List[Tensor]):
        """-> (cls fp32 [sum B, D], region fp32 [sum B*N, D], token groups)."""
        cc = _CastCache()
        x, grp, tg = self._embed(imgs, cc)
        keeps = self._keeps(grp, x.device)
        pend = None
        for i, blk in enumerate(self.blocks):
            k1 = k2 = None
            if keeps is not None and blk.drop_prob > 0.:
                k1, k2 = keeps[2 * i], keeps[2 * i + 1]
            x, pend = blk.fused_groups(x, pend, grp, cc, k1, k2)
        cls, region = ops.VitSplitGroupsFn.apply(self._final_norm(x, pend), tg)
        return cls, region, tg

    def forward(self, x):
        """Multi-crop forward (:186-231): consecutive same-resolution crops form one group; the outputs are
        concatenated group-major exactly as the reference's per-group loop concatenates them."""
        if not isinstance(x, list):
            x = [x]
        groups, start = [], 0
        for i in range(1, len(x) + 1):
            if i == len(x) or x[i].shape[-1] != x[start].shape[-1]:
                groups.append((start, i))
                start = i
        cls, region, tg = self._run([ops.cat_adjacent(x[s:e]).float() for s, e in groups])
        if self.use_dense_prediction:
            return self.head(cls), self.head_dense(region), region, [N for _, N in tg]
        return self.head(cls)

    def forward_features(self, x: Tensor):
        """:233-251 -> cls fp32 [B, D] (and the region tokens fp32 [B, N, D] in dense mode)."""
        cls, region, tg = self._run([x.float()])
        if self.use_dense_prediction:
            return cls, region.view(tg[0][0], tg[0][1], -1)
        return cls

    def forward_feature_maps(self, x: Tensor) -> Tensor:
        """:253-269 -> the final norm's output fp32 [B, 1+N, D]."""
        cc = _CastCache()
        xs, grp, tg = self._embed([x.float()], cc)
        pend = None
        for blk in self.blocks:
            xs, pend = blk.fused_groups(xs, pend, grp, cc, None, None)
        return self._final_norm(xs, pend).view(tg[0][0], tg[0][1] + 1, -1)

    def forward_return_n_last_blocks(self, x: Tensor, n: int = 1, return_patch_avgpool: bool = False, depths=[]):
        """:339-360 (eval_linear.py's probe features): the final norm's cls row after each of the last n blocks,
        concatenated, plus the mean of the last block's normed patch tokens when return_patch_avgpool.  `depths` is
        ignored, as in the reference.  A tapped block's output is materialised (residual_add) and the stream continues
        from it."""
        depth = len(self.blocks)
        if not 1 <= int(n) <= depth:
            raise ValueError(f"n must be in [1, {depth}], got {n}")
        cc = _CastCache()
        xs, grp, tg = self._embed([x.float()], cc)
        out, pend, region = [], None, None
        for i, blk in enumerate(self.blocks):
            xs, pend = blk.fused_groups(xs, pend, grp, cc, None, None)
            if depth - i <= int(n):
                xs, pend = ops.residual_add(xs, *pend), None
                y = ops.LayerNormFn.apply(xs, self.norm.weight, self.norm.bias, self.norm.eps, False)
                cls, region = ops.VitSplitGroupsFn.apply(y, tg)
                out.append(cls)
        if return_patch_avgpool:
            B, N = tg[0]
            out.append(ops.TokenMeanGroupsFn.apply(region, ((B, 1, N, 0),)))
        return torch.cat(out, dim=-1)

    def forward_selfattention(self, x, n=1):
        raise NotImplementedError("ViT attention maps (forward_selfattention) are not implemented by esvit_b200")

    def forward_last_selfattention(self, x):
        raise NotImplementedError("ViT attention maps (forward_last_selfattention) are not implemented by esvit_b200")

    def forward_all_selfattention(self, x):
        raise NotImplementedError("ViT attention maps (forward_all_selfattention) are not implemented by esvit_b200")


def deit_tiny(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=192, depth=12, num_heads=3, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def deit_small(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=384, depth=12, num_heads=6, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)


def vit_base(patch_size=16, **kwargs):
    return VisionTransformer(patch_size=patch_size, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4, qkv_bias=True,
                             norm_layer=partial(nn.LayerNorm, eps=1e-6), **kwargs)
