"""Functional fp32 restatement of the reference CvT backbone (models/cvt_v4_transformer.py) over a reference state_dict.

TEST INFRASTRUCTURE.  Plain PyTorch, no modules: every function cites the reference lines it follows.  BatchNorm:
train=True uses the batch statistics of the (padded) map and updates the running statistics held in `bufs` (a dict of
the state_dict's running_mean / running_var / num_batches_tracked tensors, modified in place, as the reference's
nn.BatchNorm2d does); train=False uses them.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn.functional as F

EPS = 1e-5          # get_cls_model: norm_layer=partial(LayerNorm, eps=1e-5) (:694)
BN_EPS, BN_MOMENTUM = 1e-5, 0.1   # nn.BatchNorm2d defaults (:94)


def layout(sd: dict):
    """-> [(dim, heads, depth, k, stride, pad)] per stage, read from the state_dict (head dim 64)"""
    out, i = [], 0
    while f"stage{i}.0.proj.weight" in sd:
        w = sd[f"stage{i}.0.proj.weight"]
        depth = 1 + max(int(k.split(".")[3]) for k in sd if k.startswith(f"stage{i}.1.layers."))
        k = w.shape[-1]
        stride, pad = (4, 2) if i == 0 else (2, 1)   # s1.yaml PATCH_STRIDE / PATCH_PADDING
        out.append((w.shape[0], w.shape[0] // 64, depth, k, stride, pad))
        i += 1
    return out


def layer_norm(x, sd, pre):
    """LayerNorm :35-41 (fp32)"""
    return F.layer_norm(x, (x.shape[-1],), sd[pre + "weight"], sd[pre + "bias"], EPS)


def batch_norm(x, sd, bufs, pre, train: bool):
    """nn.BatchNorm2d :94 in train mode (batch statistics, running-statistic update, momentum 0.1, unbiased running
    variance, num_batches_tracked += 1) or eval mode (running statistics)"""
    return F.batch_norm(x, bufs[pre + "running_mean"], bufs[pre + "running_var"], sd[pre + "weight"], sd[pre + "bias"],
                        train, BN_MOMENTUM, BN_EPS)


def bn_step(bufs, pre, train: bool):
    if train:
        bufs[pre + "num_batches_tracked"] += 1


def attention(sd, bufs, pre, x, heads, window, train):
    """Attention.forward :165-220 (no rel-pos bias, no mask); x [B, C, H, W]"""
    B, C, H, W = x.shape
    w = min(window, H, W)
    pad_r, pad_b = (w - W % w) % w, (w - H % w) % w
    x = F.pad(x, (0, pad_r, 0, pad_b))
    Hp, Wp = x.shape[-2:]
    sx, sy = Hp // w, Wp // w
    t = F.conv2d(x, sd[pre + "qkv.dw.weight"], None, padding=1, groups=C)          # DepthWiseConv2d :101-105
    t = batch_norm(t, sd, bufs, pre + "qkv.bn.", train)
    bn_step(bufs, pre + "qkv.bn.", train)
    t = F.conv2d(t, sd[pre + "qkv.pw.weight"], sd.get(pre + "qkv.pw.bias"))
    q, k, v = t.chunk(3, dim=1)

    def part(u):  # 'b (h d) (s_x w_x) (s_y w_y) -> (b s_x s_y) h (w_x w_y) d'
        u = u.reshape(B, heads, 64, sx, w, sy, w).permute(0, 3, 5, 1, 4, 6, 2)
        return u.reshape(B * sx * sy, heads, w * w, 64)

    q, k, v = part(q), part(k), part(v)
    attn = (q @ k.transpose(-1, -2) * C ** -0.5).softmax(dim=-1)     # scale = dim_out ** -0.5 (:126)
    o = (attn @ v).reshape(B, sx, sy, heads, w, w, 64).permute(0, 3, 6, 1, 4, 2, 5).reshape(B, C, Hp, Wp)
    o = o[:, :, :H, :W]
    return F.conv2d(o, sd[pre + "proj_out.weight"], sd[pre + "proj_out.bias"])


def prenorm(x, sd, pre):
    """PreNorm :55-59: LN over channels of [B, C, H, W]"""
    return layer_norm(x.permute(0, 2, 3, 1), sd, pre).permute(0, 3, 1, 2)


def feed_forward(sd, pre, x):
    """FeedForward :62-72 with QuickGELU :44-46"""
    h = F.conv2d(x, sd[pre + "net.0.weight"], sd[pre + "net.0.bias"])
    return F.conv2d(h * torch.sigmoid(1.702 * h), sd[pre + "net.2.weight"], sd[pre + "net.2.bias"])


def conv_embed(sd, i, x, k, stride, pad):
    """ConvEmbed.forward :373-382"""
    pre = f"stage{i}.0."
    x = F.conv2d(x, sd[pre + "proj.weight"], sd[pre + "proj.bias"], stride=stride, padding=pad)
    return prenorm(x, sd, pre + "norm.")


def stage_blocks(sd, bufs, i, x, heads, depth, train, window=7, keeps=None):
    """Transformer.forward_with_features :338-346 -> (x, [x after each block]); keeps: per block (k1, k2) [B] or None"""
    feats = []
    for j in range(depth):
        pre = f"stage{i}.1.layers.{j}."
        k1, k2 = keeps[j] if keeps is not None else (None, None)
        a = attention(sd, bufs, pre + "0.fn.", prenorm(x, sd, pre + "0.norm."), heads, window, train)
        x = x + (a if k1 is None else a * k1[:, None, None, None])
        f = feed_forward(sd, pre + "1.fn.", prenorm(x, sd, pre + "1.norm."))
        x = x + (f if k2 is None else f * k2[:, None, None, None])
        feats.append(x)
    return x, feats


def forward_features(sd, bufs, x, train, keeps=None):
    """CvT.forward_features :549-563 -> (pooled [B, C], x_region [B, N, C]); keeps: per stage, per block (k1, k2)"""
    for i, (dim, heads, depth, k, s, p) in enumerate(layout(sd)):
        x = conv_embed(sd, i, x, k, s, p)
        x, _ = stage_blocks(sd, bufs, i, x, heads, depth, train, keeps=None if keeps is None else keeps[i])
    region = layer_norm(x.flatten(2).transpose(1, 2), sd, "norm.")
    return region.mean(dim=1), region


def forward_dense(sd, bufs, crops: Sequence[torch.Tensor], train: bool, keeps=None):
    """CvT.forward :619-647 without the heads -> (pooled [sum B, C], region [sum B*N, C], npatch); the resolution
    groups run one after the other, so the 224^2 group updates the running statistics first"""
    pooled, fea, npatch = [], [], []
    start = 0
    sides = [c.shape[-1] for c in crops]
    for end in range(1, len(crops) + 1):
        if end == len(crops) or sides[end] != sides[start]:
            p, r = forward_features(sd, bufs, torch.cat(list(crops[start:end])), train,
                                    None if keeps is None else keeps[len(npatch)])
            B, N, C = r.shape
            pooled.append(p)
            fea.append(r.reshape(B * N, C))
            npatch.append(N)
            start = end
    return torch.cat(pooled), torch.cat(fea), npatch


def n_last_blocks(sd, bufs, x, n: int, train: bool = False):
    """forward_return_n_last_blocks :567-615"""
    lay = layout(sd)
    depths = [d for _, _, d, _, _, _ in lay]
    start = sum(depths) - n
    out: List[torch.Tensor] = []
    acc = 0
    for i, (dim, heads, depth, k, s, p) in enumerate(lay):
        x = conv_embed(sd, i, x, k, s, p)
        x, feats = stage_blocks(sd, bufs, i, x, heads, depth, train)
        for j, f in enumerate(feats):
            if acc + j >= start:
                if i == len(lay) - 1:
                    f = prenorm(f, sd, "norm.")
                out.append(f.mean(dim=(2, 3)))
        acc += depth
    return torch.cat(out, dim=-1)


def multicrop_forward(sd, bufs, crops, dense: bool, train: bool = True, keeps=None):
    """CvT.forward with DINOHead heads (`head.*`, and `head_dense.*` when dense; main_esvit.py:280-301)"""
    from .swin import dino_head
    pooled, region, npatch = forward_dense(sd, bufs, crops, train, keeps)
    if dense:
        return dino_head(pooled, sd, "head"), dino_head(region, sd, "head_dense"), region, npatch
    return dino_head(pooled, sd, "head")


def buffers(sd: dict) -> dict:
    """fresh copies of the BatchNorm buffers of a state_dict"""
    return {k: v.clone() for k, v in sd.items() if "running_" in k or k.endswith("num_batches_tracked")}
