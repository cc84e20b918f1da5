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
With use_bn=True each hidden Linear is followed by a real nn.BatchNorm1d (``mlp.{1,4}.*``; so utils.has_batchnorms and
nn.SyncBatchNorm.convert_sync_batchnorm work unchanged) and the MLP runs as ops.HeadBnGeluFn units.
Without BN the MLP of any depth is one linear.HeadMlpFn (GELUs in the GEMM epilogues) and the last layer one
linear.LastLayerFn; the row normalisation and the weight-norm reparameterisation (fwd + bwd) are esvit_b200 kernels.
Output logits are bf16 [rows, out_dim] (what the reference produces under autocast); the losses consume them without
an fp32 copy.
"""
from __future__ import annotations

import math
from functools import partial
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.modules.batchnorm import _BatchNorm

from . import backbone, linear, ops, shadow
from .backbone import MultiCropBackbone, _CastCache
from .cvt_v4_transformer import _sync_group
from .swin_transformer import Mlp, _lin_c

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
        return linear.LastLayerFn.apply(x, self.effective_weight())


class DINOHead(nn.Module):
    def __init__(self, in_dim, out_dim, use_bn=False, norm_last_layer=True, nlayers=3, hidden_dim=2048,
                 bottleneck_dim=256):
        super().__init__()
        nlayers = max(nlayers, 1)
        if nlayers == 1:
            self.mlp = nn.Linear(in_dim, bottleneck_dim)
        else:
            bn = [nn.BatchNorm1d(hidden_dim)] if use_bn else []
            layers = [nn.Linear(in_dim, hidden_dim)] + bn + [nn.GELU()]
            for _ in range(nlayers - 2):
                bn = [nn.BatchNorm1d(hidden_dim)] if use_bn else []
                layers += [nn.Linear(hidden_dim, hidden_dim)] + bn + [nn.GELU()]
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
        if any(isinstance(m, _BatchNorm) for m in mods):
            x = self._mlp_bn(x, mods)
        else:
            args = []
            for m in mods:
                if isinstance(m, nn.Linear):
                    args += [m.weight, shadow.as_bf16(m.weight), m.bias]
            x = linear.HeadMlpFn.apply(x, *args)
        return self.last_layer(ops.L2NormFn.apply(x, 1e-12))

    @staticmethod
    def _mlp_bn(x: Tensor, mods) -> Tensor:
        """the use_bn MLP: each Linear -> BatchNorm1d / SyncBatchNorm -> GELU is one ops.HeadBnGeluFn; the BN module's
        mode decides (train: batch statistics over all rows, running statistics updated; eval: running statistics)."""
        i = 0
        while i < len(mods):
            lin = mods[i]
            w16 = shadow.as_bf16(lin.weight)
            if i + 1 < len(mods) and isinstance(mods[i + 1], _BatchNorm):
                bn = mods[i + 1]
                train = bn.training or not bn.track_running_stats
                if train and bn.track_running_stats and bn.momentum is None:
                    raise NotImplementedError("BatchNorm1d(momentum=None) (cumulative running average) is not implemented")
                x = ops.HeadBnGeluFn.apply(x, lin.weight, w16, lin.bias, bn.weight, bn.bias, bn, train, _sync_group(bn))
                i += 3  # Linear, BN, GELU
            else:
                x = linear.LinearColsumFn.apply(x, lin.weight, w16, lin.bias)
                i += 1
        return x


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
        """backbone.pre_norm_block over the sequences grp = ((B, L, row0), ...)"""
        return backbone.pre_norm_block(x, pending, self.norm1, lambda y: self.attn.attend_groups(y, grp, cc),
                                       self.norm2, self.attn.proj.bias, lambda y: self.mlp.fused(y, cc),
                                       self.mlp.fc2.bias, k1, k2)

    def forward(self, x: Tensor, return_attention: bool = False) -> Tensor:
        """Reference signature (:110-116): x [B, N, C] -> fp32 [B, N, C]."""
        if return_attention:
            raise NotImplementedError("ViT attention maps are not implemented (forward_selfattention)")
        B, N, C = x.shape
        k1, k2 = backbone.block_keeps(self, B, N, x.device)
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
        w16 = (shadow.as_bf16(w) if cc is None else cc.nograd(w)).view(w.shape[0], -1)
        return linear.LinearFn.apply(ops.vit_patches(imgs, self.patch_size), w, w16, self.proj.bias)

    def forward(self, x: Tensor) -> Tensor:
        """x fp32 [B, 3, S, S] -> fp32 [B, N, D] (bf16 GEMM output; proj.bias receives no gradient on this path)."""
        B = x.shape[0]
        pe = self.embed([x.float()])
        return pe.float().view(B, -1, pe.shape[-1])


class VisionTransformer(MultiCropBackbone):
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

    def _depths(self) -> List[int]:
        return [len(self.blocks)]

    def _run(self, imgs: List[Tensor], taps=None):
        """-> (stream fp32 [T, D], pending delta, token groups ((B, N), ...)); taps: see backbone.tap, called with the
        token groups."""
        cc = _CastCache()
        x, grp, tg = self._embed(imgs, cc)
        probs = [blk.drop_prob for blk in self.blocks for _ in range(2)]
        scales = backbone.drop_path_scales(self, probs, sum(g[0] for g in grp), x.device)
        keeps = backbone.drop_path_rows(self, scales, [(B, L) for B, L, _ in grp], x.device)
        pend = None
        for i, blk in enumerate(self.blocks):
            k1 = k2 = None
            if keeps is not None and blk.drop_prob > 0.:
                k1, k2 = keeps[2 * i], keeps[2 * i + 1]
            x, pend = blk.fused_groups(x, pend, grp, cc, k1, k2)
            x, pend = backbone.tap(taps, i, x, pend, tg)
        return x, pend, tg

    def _features(self, imgs: List[Tensor], taps=None):
        """-> (cls fp32 [sum B, D], region fp32 [sum B*N, D] = the final norm's patch tokens, patches per image)"""
        x, pend, tg = self._run(imgs, taps)
        cls, region = ops.VitSplitGroupsFn.apply(self._final_norm(x, pend), tg)
        return cls, region, [N for _, N in tg]

    def _tap_feature(self, i: int, x: Tensor, tg) -> Tensor:
        """:339-360: the cls row of a block's normed output"""
        return ops.VitSplitGroupsFn.apply(x, tg)[0]

    def forward_feature_maps(self, x: Tensor) -> Tensor:
        """:253-269 -> the final norm's output fp32 [B, 1+N, D]."""
        xs, pend, _ = self._run([x.float()])
        return self._final_norm(xs, pend).view(x.shape[0], -1, xs.shape[-1])

    def forward_return_n_last_blocks(self, x: Tensor, n: int = 1, return_patch_avgpool: bool = False, depths=[]):
        """:339-360 (eval_linear.py's probe features): the final norm's cls row after each of the last n blocks,
        concatenated, plus the mean of the last block's normed patch tokens when return_patch_avgpool.  `depths` is
        ignored, as in the reference."""
        out, region = self._last_blocks(x, n, self._depths())
        if return_patch_avgpool:
            B = x.shape[0]
            out.append(ops.TokenMeanGroupsFn.apply(region, ((B, 1, region.shape[0] // B, 0),)))
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
