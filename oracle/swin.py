"""Functional fp32 oracle of the reference Swin backbone + DINOHead.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  All functions take the
reference ``state_dict`` (``sd``) and a key prefix, so the weights are
literally the reference's tensors.  Citations are into the reference repository.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
LN_EPS = 1e-6  # get_cls_model passes partial(nn.LayerNorm, eps=1e-6): models/swin_transformer.py:962


@dataclass
class SwinSpec:
    """MODEL.SPEC of experiments/imagenet/swin/*.yaml + TRAIN.IMAGE_SIZE."""
    img_size: int = 224
    patch_size: int = 4
    embed_dim: int = 96
    depths: Sequence[int] = (2, 2, 6, 2)
    num_heads: Sequence[int] = (3, 6, 12, 24)
    window_size: int = 7
    mlp_ratio: float = 4.0
    use_dense_prediction: bool = False

    @property
    def num_features(self) -> int:
        return int(self.embed_dim * 2 ** (len(self.depths) - 1))

    def stage_resolution(self, i: int) -> int:
        return (self.img_size // self.patch_size) // (2 ** i)

    def block_window_shift(self, stage: int, blk: int) -> Tuple[int, int]:
        """Window/shift fixed at construction from the *nominal* resolution
        (models/swin_transformer.py:203-209, 466)."""
        ws = self.window_size
        shift = 0 if blk % 2 == 0 else self.window_size // 2
        res = self.stage_resolution(stage)
        if res <= ws:
            shift = 0
            ws = res
        return ws, shift


SWIN_T_W7 = dict(embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=7)
SWIN_S_W14 = dict(embed_dim=96, depths=(2, 2, 18, 2), num_heads=(3, 6, 12, 24), window_size=14)
SWIN_B_W14 = dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32), window_size=14)


def rel_pos_index(ws: int) -> Tensor:
    """Closed form of relative_position_index (models/swin_transformer.py:99-110):
    idx(i,j) = (yi-yj+ws-1)*(2ws-1) + (xi-xj+ws-1), tokens row-major in the window."""
    t = torch.arange(ws * ws)
    y, x = t // ws, t % ws
    return (y[:, None] - y[None, :] + ws - 1) * (2 * ws - 1) + (x[:, None] - x[None, :] + ws - 1)


def shift_mask(H: int, W: int, ws: int, shift: int) -> Tensor:
    """Closed form of create_attn_mask (models/swin_transformer.py:249-272).
    Region id of a coordinate p in the rolled+padded frame of extent Hp:
    0 if p < Hp-ws, 1 if p < Hp-shift, else 2; mask = -100 where the (rid_h, rid_w)
    pair of two tokens of one window differ.  Returns [nW, ws*ws, ws*ws] fp32."""
    Hp = -(-H // ws) * ws
    Wp = -(-W // ws) * ws

    def rid(n):
        p = torch.arange(n)
        return (p >= n - ws).long() + (p >= n - shift).long()

    reg = rid(Hp)[:, None] * 3 + rid(Wp)[None, :]  # [Hp, Wp]
    reg = reg.view(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    diff = reg[:, None, :] != reg[:, :, None]
    return diff.float() * -100.0


def layer_norm(x: Tensor, sd: Dict[str, Tensor], p: str) -> Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], LN_EPS)


def linear(x: Tensor, sd: Dict[str, Tensor], p: str) -> Tensor:
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def patch_embed(x: Tensor, sd, p: str, patch: int) -> Tensor:
    """PatchEmbed.forward (models/swin_transformer.py:537-547): conv k=s=patch, flatten, LN."""
    y = F.conv2d(x, sd[p + ".proj.weight"], sd[p + ".proj.bias"], stride=patch)
    y = y.flatten(2).transpose(1, 2)
    return layer_norm(y, sd, p + ".norm")


def window_attention(xw: Tensor, sd, p: str, num_heads: int, ws: int, mask: Optional[Tensor]) -> Tensor:
    """WindowAttention.forward (models/swin_transformer.py:120-152); xw is [B_, N, C]."""
    B_, N, C = xw.shape
    hd = C // num_heads
    qkv = linear(xw, sd, p + ".qkv").reshape(B_, N, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0] * (hd ** -0.5), qkv[1], qkv[2]
    attn = q @ k.transpose(-2, -1)
    table = sd[p + ".relative_position_bias_table"]  # [(2ws-1)^2, nH]
    bias = table[rel_pos_index(ws).to(table.device).view(-1)].view(N, N, num_heads).permute(2, 0, 1)
    attn = attn + bias.unsqueeze(0)
    if mask is not None:
        nW = mask.shape[0]
        attn = attn.view(B_ // nW, nW, num_heads, N, N) + mask[None, :, None]
        attn = attn.view(-1, num_heads, N, N)
    attn = attn.softmax(dim=-1)
    out = (attn @ v).transpose(1, 2).reshape(B_, N, C)
    return linear(out, sd, p + ".proj")


def swin_block(x: Tensor, sd, p: str, num_heads: int, ws: int, shift: int,
               keep1: Optional[Tensor] = None, keep2: Optional[Tensor] = None) -> Tensor:
    """SwinTransformerBlock.forward (models/swin_transformer.py:275-333).
    keep1/keep2: optional DropPath scale vectors [B] (0 or 1/keep_prob) for the two
    residual branches; None = identity (parity runs use DROP_PATH_RATE 0)."""
    B, L, C = x.shape
    H = W = int(math.sqrt(L))
    shortcut = x
    y = layer_norm(x, sd, p + ".norm1").view(B, H, W, C)
    pad_r = (ws - W % ws) % ws
    pad_b = (ws - H % ws) % ws
    y = F.pad(y, (0, 0, 0, pad_r, 0, pad_b))  # zeros AFTER norm1 (:287-290)
    Hp, Wp = H + pad_b, W + pad_r
    mask = None
    if shift > 0:
        y = torch.roll(y, shifts=(-shift, -shift), dims=(1, 2))
        mask = shift_mask(H, W, ws, shift).to(y.device)
    yw = y.view(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)
    aw = window_attention(yw, sd, p + ".attn", num_heads, ws, mask)
    y = aw.view(B, Hp // ws, Wp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, C)
    if shift > 0:
        y = torch.roll(y, shifts=(shift, shift), dims=(1, 2))
    y = y[:, :H, :W, :].reshape(B, H * W, C)
    if keep1 is not None:
        y = y * keep1.view(B, 1, 1)
    x = shortcut + y
    z = linear(F.gelu(linear(layer_norm(x, sd, p + ".norm2"), sd, p + ".mlp.fc1")), sd, p + ".mlp.fc2")
    if keep2 is not None:
        z = z * keep2.view(B, 1, 1)
    return x + z


def patch_merging(x: Tensor, sd, p: str) -> Tensor:
    """PatchMerging.forward (models/swin_transformer.py:393-420)."""
    B, L, C = x.shape
    H = W = int(math.sqrt(L))
    x = x.view(B, H, W, C)
    if H % 2 == 1:
        x = F.pad(x, (0, 0, 0, W % 2, 0, H % 2))
    x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
    x = x.view(B, -1, 4 * C)
    x = layer_norm(x, sd, p + ".norm")
    return F.linear(x, sd[p + ".reduction.weight"])


def forward_features(x: Tensor, sd, spec: SwinSpec, prefix: str = "",
                     keep: Optional[Dict[str, Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """SwinTransformer.forward_features (models/swin_transformer.py:678-694).
    Returns (pooled [B,D], region [B,N,D])."""
    x = patch_embed(x, sd, prefix + "patch_embed", spec.patch_size)
    for i, depth in enumerate(spec.depths):
        for j in range(depth):
            ws, shift = spec.block_window_shift(i, j)
            p = f"{prefix}layers.{i}.blocks.{j}"
            k1 = keep.get(p + ".1") if keep else None
            k2 = keep.get(p + ".2") if keep else None
            x = swin_block(x, sd, p, spec.num_heads[i], ws, shift, k1, k2)
        if i < len(spec.depths) - 1:
            x = patch_merging(x, sd, f"{prefix}layers.{i}.downsample")
    region = layer_norm(x, sd, prefix + "norm")
    pooled = region.mean(dim=1)  # AdaptiveAvgPool1d(1) over tokens (:688-689)
    return pooled, region


def dino_head(x: Tensor, sd, p: str) -> Tensor:
    """DINOHead.forward, nlayers=3, no BN (models/vision_transformer.py:384-418);
    weight_norm: w = g * v / ||v||_row (dim=0 default of nn.utils.weight_norm)."""
    x = F.gelu(linear(x, sd, p + ".mlp.0"))
    x = F.gelu(linear(x, sd, p + ".mlp.2"))
    x = linear(x, sd, p + ".mlp.4")
    x = F.normalize(x, dim=-1, p=2)
    v, g = sd[p + ".last_layer.weight_v"], sd[p + ".last_layer.weight_g"]
    w = v * (g / v.norm(2, dim=1, keepdim=True))
    return F.linear(x, w)


def group_crops(crops: List[Tensor]) -> List[Tuple[int, int]]:
    """Consecutive same-resolution groups (unique_consecutive/cumsum at
    models/swin_transformer.py:729-732)."""
    groups, start = [], 0
    for i in range(1, len(crops) + 1):
        if i == len(crops) or crops[i].shape[-1] != crops[start].shape[-1]:
            groups.append((start, i))
            start = i
    return groups


def multicrop_forward(crops, sd, spec: SwinSpec, keep=None):
    """SwinTransformer.forward (models/swin_transformer.py:713-763).  Dense mode
    returns (head(cls), head_dense(fea), fea, npatch); view mode returns head(cls)."""
    if not isinstance(crops, list):
        crops = [crops]
    cls_l, fea_l, npatch = [], [], []
    for (s, e) in group_crops(crops):
        pooled, region = forward_features(torch.cat(crops[s:e]), sd, spec, keep=keep)
        B, N, C = region.shape
        cls_l.append(pooled)
        fea_l.append(region.reshape(B * N, C))
        npatch.append(N)
    out_cls = torch.cat(cls_l)
    if spec.use_dense_prediction:
        out_fea = torch.cat(fea_l)
        return dino_head(out_cls, sd, "head"), dino_head(out_fea, sd, "head_dense"), out_fea, npatch
    return dino_head(out_cls, sd, "head")
