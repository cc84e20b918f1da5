"""Functional fp32 restatement of the reference Vision Longformer backbone (models/vision_longformer.py MsViT with
layers/longformer2d.py Long2DSCSelfAttention) over a reference state_dict.

TEST INFRASTRUCTURE.  Plain PyTorch, no modules: every function cites the reference lines it follows.  The served
configuration only: rpe (`a0`), one global token in the sliding-chunk stages, sharew, exact 0, w = 7, LN eps 1e-6, no
DropPath.  The sliding-chunk attention is the dense masked restatement of oracle/vil_attn.py.  `modes` is an iterator of
the sliding-chunk modes drawn in train mode with mode > 0 (longformer2d.py:149-151), consumed in the reference's order.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn.functional as F

from . import vil_attn as VA
from .swin import dino_head

EPS = 1e-6   # MsViT norm_layer=partial(nn.LayerNorm, eps=1e-6) (:413); LN_EPS is read but not used (:419-424)
W = VA.W


def sc_index(w: int = W) -> torch.Tensor:
    """longformer2d.py:69-102: [w*w, 9*w*w] table index of (query token of the centre chunk, key r of chunk j)"""
    idx = torch.empty(w * w, 9 * w * w, dtype=torch.long)
    for qx in range(w):
        for qy in range(w):
            for j in range(9):
                cx, cy = j // 3 - 1, j % 3 - 1
                for kx in range(w):
                    for ky in range(w):
                        dx = qx - (cx * w + kx) + 2 * w - 1
                        dy = qy - (cy * w + ky) + 2 * w - 1
                        idx[qx * w + qy, j * w * w + kx * w + ky] = dx * (4 * w - 1) + dy
    return idx


def dense_index(wx: int, wy: int) -> torch.Tensor:
    """vision_longformer.py:73-84: [wx*wy, wx*wy] table index"""
    idx = torch.empty(wx * wy, wx * wy, dtype=torch.long)
    for a in range(wx * wy):
        for b in range(wx * wy):
            idx[a, b] = (a // wy - b // wy + wx - 1) * (2 * wy - 1) + (a % wy - b % wy + wy - 1)
    return idx


def layout(sd: dict):
    """-> [(dim, heads, blocks, patch, nglo, sliding)] per stage (layer1..layer4), read from the state_dict"""
    out, i = [], 1
    while f"layer{i}.0.proj.weight" in sd:
        w = sd[f"layer{i}.0.proj.weight"]
        blocks = max(int(k.split(".")[1]) for k in sd if k.startswith(f"layer{i}.")) // 2
        out.append((w.shape[0], w.shape[0] // 32, blocks, w.shape[-1], 1 if f"layer{i}.0.cls_token" in sd else 0,
                    f"layer{i}.1.attn.query.weight" in sd))
        i += 1
    return out


def ln(x, sd, pre):
    return F.layer_norm(x, (x.shape[-1],), sd[pre + "weight"], sd[pre + "bias"], EPS)


def lin(x, sd, pre):
    return F.linear(x, sd[pre + "weight"], sd.get(pre + "bias"))


def patch_embed(sd, i, x, nglo):
    """PatchEmbed.forward :227-259 (ape False): conv, LN over the patch rows, cat(cls_token, x)"""
    pre = f"layer{i}.0."
    p = sd[pre + "proj.weight"].shape[-1]
    x = F.conv2d(x, sd[pre + "proj.weight"], sd[pre + "proj.bias"], stride=p)
    nx, ny = x.shape[-2:]
    x = ln(x.flatten(2).transpose(1, 2), sd, pre + "norm_embed.")
    if nglo:
        x = torch.cat([sd[pre + "cls_token"].expand(x.shape[0], -1, -1), x], 1)
    return x, nx, ny


def sc_attention(sd, pre, x, nx, ny, heads, mode):
    """Long2DSCSelfAttention.forward :139-330 (rpe, one global token, sharew, exact 0) as one masked attention"""
    B, N, C = x.shape
    q = lin(x, sd, pre + "query.").reshape(B * N, C)
    kv = lin(x, sd, pre + "kv.").reshape(B * N, 2 * C)
    table = sd[pre + "local_relative_position_bias_table"]
    g2l, g2g = sd[pre + "g2l_relative_position_bias"], sd[pre + "g2g_relative_position_bias"]
    lb = table[sd[pre + "relative_position_index"].reshape(-1)].view(W * W, 9 * W * W, heads).permute(2, 0, 1)
    bias = torch.cat([g2l[1][:, :, None].expand(heads, W * W, 1), lb], -1)
    bias_g = torch.cat([g2g[:, 0, :], g2l[0].expand(heads, N - 1)], -1)
    ctx = VA.dense_attention(q, kv, bias, bias_g, VA.dense_index(nx, ny, mode), B, N, heads, 32 ** -0.5)
    return lin(ctx.view(B, N, C), sd, pre + "proj.")


def full_attention(sd, pre, x, heads, nglo):
    """Attention.forward :86-131 with rpe: the [nH, N, N] bias from g2g / g2l and the table, the local block bicubic-
    resized (interpolate_pos_encoding :134-151) when the map is not the table's"""
    B, N, C = x.shape
    qkv = lin(x, sd, pre + "qkv.").reshape(B, N, 3, heads, 32).permute(2, 0, 3, 1, 4)
    idx = sd[pre + "relative_position_index"]
    L0 = idx.shape[0]
    loc = sd[pre + "local_relative_position_bias_table"][idx.reshape(-1)].view(L0, L0, heads)
    npatch = N - nglo
    if npatch != L0:
        loc = F.interpolate(loc.reshape(1, L0, L0, heads).permute(0, 3, 1, 2), scale_factor=npatch / L0,
                            mode='bicubic').permute(0, 2, 3, 1)[0]
    bias = loc.permute(2, 0, 1)
    if nglo:
        g2l, g2g = sd[pre + "g2l_relative_position_bias"], sd[pre + "g2g_relative_position_bias"]
        top = torch.cat([g2g, g2l[0].unsqueeze(-1).expand(-1, -1, npatch)], -1)
        bias = torch.cat([top, torch.cat([g2l[1].unsqueeze(1).expand(-1, npatch, -1), bias], -1)], 1)
    s = qkv[0] @ qkv[1].transpose(-2, -1) * 32 ** -0.5 + bias[None]
    o = (s.softmax(-1) @ qkv[2]).transpose(1, 2).reshape(B, N, C)
    return lin(o, sd, pre + "proj.")


def stage(sd, i, x, lay, modes, train, feats=None):
    """layer{i}: PatchEmbed, then AttnBlock / MlpBlock pairs (:372-403); feats collects every MlpBlock output"""
    dim, heads, blocks, p, nglo, sliding = lay
    x, nx, ny = patch_embed(sd, i, x, nglo)
    for j in range(blocks):
        pre = f"layer{i}.{1 + 2 * j}."
        y = ln(x, sd, pre + "norm.")
        if sliding:
            mode = next(modes) if train else 0   # MODE 1: a draw in train mode, all chunks in eval
            x = x + sc_attention(sd, pre + "attn.", y, nx, ny, heads, mode)
        else:
            x = x + full_attention(sd, pre + "attn.", y, heads, nglo)
        pre = f"layer{i}.{2 + 2 * j}."
        x = x + lin(F.gelu(lin(ln(x, sd, pre + "norm."), sd, pre + "mlp.fc1.")), sd, pre + "mlp.fc2.")
        if feats is not None:
            feats.append(x)
    return x, nx, ny


def _to_map(x, nglo, nx, ny):
    """forward_features :584: drop the global rows, tokens -> [B, C, nx, ny]"""
    return x[:, nglo:].transpose(-2, -1).reshape(x.shape[0], -1, nx, ny)


def forward_features(sd, x, modes, train: bool):
    """MsViT.forward_features :581-605 -> (x_cls [B, C], x_region [B, N, C]); the last stage has no global token"""
    lays = layout(sd)
    for i, lay in enumerate(lays, 1):
        x, nx, ny = stage(sd, i, x, lay, modes, train)
        if i < len(lays):
            x = _to_map(x, lay[4], nx, ny)
    x = ln(x, sd, "norm.")
    if lays[-1][4]:
        return x[:, 0], x[:, 1:]
    return x.mean(1), x


def forward_dense(sd, crops: Sequence[torch.Tensor], modes, train: bool):
    """MsViT.forward :719-756 without the heads -> (x_cls [sum B, C], region [sum B*N, C], npatch)"""
    cls, fea, npatch, start = [], [], [], 0
    sides = [c.shape[-1] for c in crops]
    for end in range(1, len(crops) + 1):
        if end == len(crops) or sides[end] != sides[start]:
            c, r = forward_features(sd, torch.cat(list(crops[start:end])), modes, train)
            B, N, C = r.shape
            cls.append(c)
            fea.append(r.reshape(B * N, C))
            npatch.append(N)
            start = end
    return torch.cat(cls), torch.cat(fea), npatch


def n_last_blocks(sd, x, n: int, modes=iter(()), train: bool = False):
    """forward_return_n_last_blocks :636-676: every MlpBlock output; the global row where the stage has one, else the
    token mean; the last stage's through the final norm"""
    lays = layout(sd)
    start = sum(l[2] for l in lays) - n
    out: List[torch.Tensor] = []
    acc = 0
    for i, lay in enumerate(lays, 1):
        feats = []
        x, nx, ny = stage(sd, i, x, lay, modes, train, feats)
        for j, f in enumerate(feats):
            if acc + j >= start:
                if i == len(lays):
                    f = ln(f, sd, "norm.")
                out.append(f[:, 0] if lay[4] else f.mean(1))
        acc += lay[2]
        if i < len(lays):
            x = _to_map(x, lay[4], nx, ny)
    return torch.cat(out, dim=-1)


def multicrop_forward(sd, crops, dense: bool, modes, train: bool = True):
    """MsViT.forward with DINOHead heads (`head.*`, and `head_dense.*` when dense; main_esvit.py:257-276)"""
    cls, region, npatch = forward_dense(sd, crops, modes, train)
    if dense:
        return dino_head(cls, sd, "head"), dino_head(region, sd, "head_dense"), region, npatch
    return dino_head(cls, sd, "head")


def seeded(rec, seed: int) -> dict:
    """golden.seeded_state_dict for the float tensors, the closed-form index buffers for the integer ones; the aliased
    `*_global.*` entries (sharew: the same modules as query / kv / proj) get the values of the entries they alias"""
    from . import golden as GD
    sd = GD.seeded_state_dict([r for r in rec if r[2]], seed)
    for name, shape, is_float in rec:
        if not is_float:
            idx = sc_index() if shape[1] == 9 * shape[0] else dense_index(*(int(round(shape[0] ** 0.5)),) * 2)
            assert tuple(idx.shape) == tuple(shape), (name, shape)
            sd[name] = idx
    for name in sd:
        if "_global." in name:
            sd[name] = sd[name.replace("_global.", ".")]
    return {name: sd[name] for name, _, _ in rec}
