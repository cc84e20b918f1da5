"""Functional fp32 oracle of the attention-map entry points.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into the reference repository.

  * ``block_attention``: the ``attn_out`` probabilities of one SwinTransformerBlock (models/swin_transformer.py:283-308
    pad after norm1, roll, window_partition; WindowAttention.forward :120-147), [B*nW, nH, ws*ws, ws*ws];
  * ``selfattention``: SwinTransformer.forward_selfattention (:766-796) over BasicLayer.forward_with_attention
    (:492-499); the residual stream is ``oracle.swin``'s, unchanged.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from . import eval as E
from . import golden as GD
from . import swin as S

Tensor = torch.Tensor


def block_attention(x: Tensor, sd, p: str, num_heads: int, ws: int, shift: int) -> Tensor:
    """Softmax probabilities of block ``p`` on its input x [B, L, C] (the same arithmetic as oracle.swin.swin_block)."""
    B, L, C = x.shape
    H = W = int(math.sqrt(L))
    y = S.layer_norm(x, sd, p + ".norm1").view(B, H, W, C)
    y = F.pad(y, (0, 0, 0, (ws - W % ws) % ws, 0, (ws - H % ws) % ws))  # zeros AFTER norm1 (:287-290)
    Hp, Wp = y.shape[1], y.shape[2]
    if shift > 0:
        y = torch.roll(y, shifts=(-shift, -shift), dims=(1, 2))
    N, hd = ws * ws, C // num_heads
    yw = y.view(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, N, C)
    qkv = S.linear(yw, sd, p + ".attn.qkv").reshape(-1, N, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    attn = (qkv[0] * (hd ** -0.5)) @ qkv[1].transpose(-2, -1)
    table = sd[p + ".attn.relative_position_bias_table"]
    attn = attn + table[S.rel_pos_index(ws).view(-1)].view(N, N, num_heads).permute(2, 0, 1).unsqueeze(0)
    if shift > 0:
        mask = S.shift_mask(H, W, ws, shift)
        nW = mask.shape[0]
        attn = (attn.view(-1, nW, num_heads, N, N) + mask[None, :, None]).view(-1, num_heads, N, N)
    return attn.softmax(dim=-1)


def selfattention(x: Tensor, sd, spec: S.SwinSpec, n: int = 1, prefix: str = ""):
    """forward_selfattention (:766-778): the last block's probabilities if n == 1 (:780-787), else the list of every
    block's in execution order (:789-796)."""
    x = S.patch_embed(x, sd, prefix + "patch_embed", spec.patch_size)
    maps = []
    for i, depth in enumerate(spec.depths):
        for j in range(depth):
            ws, shift = spec.block_window_shift(i, j)
            p = f"{prefix}layers.{i}.blocks.{j}"
            maps.append(block_attention(x, sd, p, spec.num_heads[i], ws, shift))
            x = S.swin_block(x, sd, p, spec.num_heads[i], ws, shift)
        if i < len(spec.depths) - 1:
            x = S.patch_merging(x, sd, f"{prefix}layers.{i}.downsample")
    return maps[-1] if n == 1 else maps


def load_golden_attn(path: str) -> dict:
    """tests/golden/esvit_attn.pt with every case's seeded weights and images rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    for C in G["cases"].values():
        C["state_dict"] = GD.seeded_state_dict(C["state_recipe"], C["weight_seed"])
        C["images"] = E.probe_images(C["batch"], C["side"], C["image_seed"])
    return G
