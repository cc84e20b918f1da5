"""Functional fp32 restatement of the reference ViT backbone (models/vision_transformer.py) over a reference state_dict.

TEST INFRASTRUCTURE.  Plain PyTorch, no modules: every function cites the reference lines it follows.
"""
from __future__ import annotations

import math
from typing import List, Sequence

import torch
import torch.nn.functional as F

EPS = 1e-6  # norm_layer=partial(nn.LayerNorm, eps=1e-6), models/vision_transformer.py:363-381


def pos_encoding(pos_embed: torch.Tensor, npatch: int) -> torch.Tensor:
    """interpolate_pos_encoding :271-285"""
    N = pos_embed.shape[1] - 1
    if npatch == N:
        return pos_embed
    dim = pos_embed.shape[-1]
    side = int(math.sqrt(N))
    p = F.interpolate(pos_embed[:, 1:].reshape(1, side, side, dim).permute(0, 3, 1, 2),
                      scale_factor=math.sqrt(npatch / N), mode="bicubic")
    return torch.cat((pos_embed[:, 0].unsqueeze(0), p.permute(0, 2, 3, 1).reshape(1, -1, dim)), dim=1)


def embed(sd: dict, x: torch.Tensor, patch: int) -> torch.Tensor:
    """PatchEmbed :136-139 + forward_features :234-241 -> [B, 1+N, D]"""
    t = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch).flatten(2).transpose(1, 2)
    t = torch.cat((sd["cls_token"].expand(x.shape[0], -1, -1), t), dim=1)
    return t + pos_encoding(sd["pos_embed"], t.shape[1] - 1)


def attention(sd: dict, pre: str, x: torch.Tensor, nH: int) -> torch.Tensor:
    """Attention.forward :83-95"""
    B, N, C = x.shape
    qkv = F.linear(x, sd[pre + "qkv.weight"], sd.get(pre + "qkv.bias"))
    qkv = qkv.reshape(B, N, 3, nH, C // nH).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    attn = ((q @ k.transpose(-2, -1)) * (C // nH) ** -0.5).softmax(dim=-1)
    return F.linear((attn @ v).transpose(1, 2).reshape(B, N, C), sd[pre + "proj.weight"], sd[pre + "proj.bias"])


def block(sd: dict, i: int, x: torch.Tensor, nH: int, keep=None) -> torch.Tensor:
    """Block.forward :110-116; keep: (k1, k2) per-sample DropPath scales [B] or None"""
    pre = f"blocks.{i}."
    C = x.shape[-1]
    k1, k2 = keep if keep is not None else (None, None)
    y = attention(sd, pre + "attn.", F.layer_norm(x, (C,), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], EPS), nH)
    x = x + (y if k1 is None else y * k1[:, None, None])
    h = F.layer_norm(x, (C,), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], EPS)
    h = F.linear(F.gelu(F.linear(h, sd[pre + "mlp.fc1.weight"], sd[pre + "mlp.fc1.bias"])),
                 sd[pre + "mlp.fc2.weight"], sd[pre + "mlp.fc2.bias"])
    return x + (h if k2 is None else h * k2[:, None, None])


def depth_of(sd: dict) -> int:
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))


def feature_maps(sd: dict, x: torch.Tensor, patch: int, nH: int, keeps=None) -> torch.Tensor:
    """forward_feature_maps :253-269 -> norm(x) [B, 1+N, D]; keeps: per block (k1, k2) or None"""
    t = embed(sd, x, patch)
    for i in range(depth_of(sd)):
        t = block(sd, i, t, nH, None if keeps is None else keeps[i])
    return F.layer_norm(t, (t.shape[-1],), sd["norm.weight"], sd["norm.bias"], EPS)


def forward_dense(sd: dict, crops: Sequence[torch.Tensor], patch: int, nH: int, keeps=None):
    """VisionTransformer.forward :186-217 without the heads -> (cls [sum B, D], region [sum B*N, D], npatch).
    keeps: per resolution group, per block (k1, k2) DropPath scales [B_g], or None"""
    cls, fea, npatch = [], [], []
    start = 0
    sides = [c.shape[-1] for c in crops]
    for end in range(1, len(crops) + 1):
        if end == len(crops) or sides[end] != sides[start]:
            y = feature_maps(sd, torch.cat(list(crops[start:end])), patch, nH,
                             None if keeps is None else keeps[len(npatch)])
            B, L, C = y.shape
            cls.append(y[:, 0])
            fea.append(y[:, 1:].reshape(B * (L - 1), C))
            npatch.append(L - 1)
            start = end
    return torch.cat(cls), torch.cat(fea), npatch


def n_last_blocks(sd: dict, x: torch.Tensor, patch: int, nH: int, n: int, avgpool: bool) -> torch.Tensor:
    """forward_return_n_last_blocks :339-360"""
    t = embed(sd, x, patch)
    D = depth_of(sd)
    out: List[torch.Tensor] = []
    norm = lambda z: F.layer_norm(z, (z.shape[-1],), sd["norm.weight"], sd["norm.bias"], EPS)  # noqa: E731
    for i in range(D):
        t = block(sd, i, t, nH)
        if D - i <= n:
            out.append(norm(t)[:, 0])
    if avgpool:
        out.append(norm(t)[:, 1:].mean(dim=1))
    return torch.cat(out, dim=-1)


def multicrop_forward(sd: dict, crops: Sequence[torch.Tensor], patch: int, nH: int, dense: bool, keeps=None):
    """VisionTransformer.forward :186-231 with DINOHead heads (`head.*`, and `head_dense.*` when dense; main_esvit.py
    :304-327): dense -> (head(cls), head_dense(region), region, npatch); view -> head(cls)"""
    from .swin import dino_head
    cls, region, npatch = forward_dense(sd, crops, patch, nH, keeps)
    if dense:
        return dino_head(cls, sd, "head"), dino_head(region, sd, "head_dense"), region, npatch
    return dino_head(cls, sd, "head")
