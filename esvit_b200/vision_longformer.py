"""Vision Longformer backbone (models/vision_longformer.py MsViT, layers/longformer2d.py Long2DSCSelfAttention) behind
the reference's signatures, attribute names and state_dict keys (incl. the aliased ``attn.{query,kv,proj}_global.*``
entries and the ``relative_position_index`` buffers), so a reference state_dict loads with strict=True.

Served configuration: the `vil_2262` family of experiments/imagenet/vil (4 stages, head dim 32, `a0` = relative position
bias and no absolute position embedding, sliding chunks of w = 7 with one global token and shared global weights,
sw_exact 0, NORM_EMBED True, AVG_POOL False); anything else raises NotImplementedError naming the key.

Execution follows the Swin / CvT ports: one fp32 token-major residual stream [T, C] holding every image of every
resolution group back to back (N = Nglo + H*W rows per image, the global row first), bf16 branches, the residual add +
DropPath deferred into the next fused add + LN, every per-token op run once over all groups.  The sliding-chunk attention
(ops.SlidingChunkAttnGroupsFn), the dense biased attention (ops.DenseBiasAttnGroupsFn), the stream patch embedding
(ops.VilStreamEmbedFn) and the global-token assembly (ops.ClsCatGroupsFn) launch per group on pointer offsets.  The
relative-position biases of every group come from one sparse gather per module and step (ops.RelBiasFn, bias_plan).

Mode draws (longformer2d.py:146-156): every sliding-chunk call in train mode with mode > 0 draws its neighbour chunk;
here the draws are one torch.randint on the device per forward (int32 [sliding-chunk modules, groups]), so a captured
CUDA graph draws fresh modes on every replay; eval uses 0, mode <= 0 its fixed value.
"""
from __future__ import annotations

import math
from functools import partial
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import backbone, linear, ops
from .backbone import MultiCropBackbone, _CastCache

Tensor = torch.Tensor
BF16 = torch.bfloat16
W = ops.VIL_W


def _trunc_normal_(t: Tensor, std: float = .02) -> Tensor:
    return nn.init.trunc_normal_(t, std=std)


def sc_relative_position_index(w: int = W) -> Tensor:
    """[w*w, 9*w*w] index into the (4w-1)^2 local table (longformer2d.py:69-102): query token of the centre chunk vs.
    key token r of neighbour chunk j = 3 (dx + 1) + (dy + 1)"""
    c = torch.arange(-w, 2 * w)
    coords = torch.stack(torch.meshgrid([c, c], indexing="ij"))                       # 2, 3w, 3w
    unfold = coords.view(2, 3, w, 3, w).permute(0, 1, 3, 2, 4).reshape(2, 3, 3, w * w)  # c m n (x y)
    q = unfold[:, 1, 1, :]
    rel = torch.cat([q[:, :, None] - unfold[:, m, n, :][:, None, :] for m in range(3) for n in range(3)], -1)
    rel = rel.permute(1, 2, 0).contiguous()
    rel[:, :, 0] += 2 * w - 1
    rel[:, :, 1] += 2 * w - 1
    rel[:, :, 0] *= 4 * w - 1
    return rel.sum(-1)


def dense_relative_position_index(wx: int, wy: int) -> Tensor:
    """[wx*wy, wx*wy] index into the (2wx-1)(2wy-1) table (vision_longformer.py:73-84)"""
    coords = torch.stack(torch.meshgrid([torch.arange(wx), torch.arange(wy)], indexing="ij")).flatten(1)
    rel = (coords[:, :, None] - coords[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += wx - 1
    rel[:, :, 1] += wy - 1
    rel[:, :, 0] *= 2 * wy - 1
    return rel.sum(-1)


def bicubic_matrix(n_in: int, scale_factor: float) -> np.ndarray:
    """fp64 [floor(n_in * scale_factor), n_in] weights of F.interpolate(mode='bicubic', align_corners=False,
    scale_factor=scale_factor) on fp32 input along one axis: source x = (dst + 0.5) / scale_factor - 0.5 (computed in
    fp32 as PyTorch does, so the taps' fractions agree), cubic convolution with a = -0.75, taps clamped to the border"""
    n_out = int(math.floor(n_in * scale_factor))
    a = -0.75

    def c1(t):
        return ((a + 2) * t - (a + 3)) * t * t + 1

    def c2(t):
        return ((a * t - 5 * a) * t + 8 * a) * t - 4 * a

    A = np.zeros((n_out, n_in))
    sc = np.float32(1.0 / scale_factor)
    for o in range(n_out):
        x = np.float32(sc * np.float32(o + 0.5)) - np.float32(0.5)
        i0 = math.floor(x)
        t = float(np.float32(x - np.float32(i0)))
        for k, wgt in enumerate((c2(t + 1), c1(t), c1(1 - t), c2(2 - t))):
            A[o, min(max(i0 - 1 + k, 0), n_in - 1)] += wgt
    return A


# ---- relative-position bias plans ------------------------------------------------------------------------------------
_plans = {}  # never freed: a captured CUDA graph reads the CSR arrays


def _al4(n: int) -> int:
    return (n + 3) & ~3  # 16-byte aligned slots


def _csr(rows, cols, vals, nrows, ncols, device):
    import scipy.sparse as sp
    m = sp.coo_matrix((np.asarray(vals, np.float64), (np.asarray(rows, np.int64), np.asarray(cols, np.int64))),
                      shape=(nrows, ncols)).tocsr()
    m.sum_duplicates()
    m.sort_indices()

    def dev(c):
        return (torch.from_numpy(c.indptr.astype(np.int32)).to(device),
                torch.from_numpy(c.indices.astype(np.int32)).to(device),
                torch.from_numpy(c.data.astype(np.float32)).to(device))
    mt = m.T.tocsr()
    mt.sort_indices()
    return dev(m), dev(mt)


def bias_plan(attn: nn.Module, Ns: Sequence[int], device):
    """(plan for ops.RelBiasFn, per-group offsets) of the biases `attn` uses for groups of N tokens per image.
    Sliding chunks: offsets (bias_off, bias_g_off) of [nH, 49, 442] and [nH, N]; dense: bias_off of [nH, N, N]."""
    sc = isinstance(attn, Long2DSCSelfAttention)
    nH = attn.num_heads
    nglo = attn.nglo
    T = attn.local_relative_position_bias_table.shape[0]
    key = (sc, nH, nglo, tuple(Ns), T, getattr(attn, "wx", 0), getattr(attn, "wy", 0), str(device))
    ent = _plans.get(key)
    if ent is not None:
        return ent
    n0, n1 = T * nH, 2 * nH * nglo
    h = np.arange(nH)
    rows, cols, vals, offs, o = [], [], [], [], 0

    def add(r, c, v=None):
        rows.append(np.asarray(r).ravel())
        cols.append(np.asarray(c).ravel())
        vals.append(np.ones(rows[-1].size) if v is None else np.asarray(v, np.float64).ravel())

    if sc:
        rel = attn.relative_position_index.cpu().numpy()  # [49, 441]
        nb = 1 + rel.shape[1]
        l = np.arange(rel.shape[0])
        for N in Ns:
            bo = o
            base = bo + (h[:, None] * rel.shape[0] + l[None, :]) * nb                            # [nH, 49]
            add(base, n0 + nH + h[:, None] + 0 * l[None, :])                                     # g2l[1]
            add(base[:, :, None] + 1 + np.arange(rel.shape[1])[None, None, :], rel[None] * nH + h[:, None, None])
            bgo = _al4(bo + nH * rel.shape[0] * nb)
            add(bgo + h * N, n0 + n1 + h)                                                          # g2g
            add(bgo + h[:, None] * N + np.arange(1, N)[None, :], n0 + h[:, None] + 0 * np.arange(1, N)[None, :])
            offs.append((bo, bgo))
            o = _al4(bgo + nH * N)
    else:
        wx, wy = attn.wx, attn.wy
        rel = attn.relative_position_index.cpu().numpy()  # [wx*wy, wx*wy]
        for N in Ns:
            bo = o
            npatch = N - nglo
            L = N
            if npatch == wx * wy:
                loc_rows, loc_cols, loc_w = None, rel, None
            else:  # interpolate_pos_encoding :134-151: B_s = A B A^T per head
                A = bicubic_matrix(wx * wy, npatch / (wx * wy))
                if A.shape[0] != npatch:
                    raise ValueError(f"bicubic resize of {wx * wy} gives {A.shape[0]} rows, not {npatch}")
                p_nz = [np.nonzero(A[p])[0] for p in range(npatch)]
                pr, qr, cc, ww = [], [], [], []
                for p in range(npatch):
                    for q in range(npatch):
                        ai, bj = p_nz[p], p_nz[q]
                        pr.append(np.full(ai.size * bj.size, p))
                        qr.append(np.full(ai.size * bj.size, q))
                        cc.append(rel[ai[:, None], bj[None, :]].ravel())
                        ww.append((A[p, ai][:, None] * A[q, bj][None, :]).ravel())
                loc_rows = (np.concatenate(pr), np.concatenate(qr))
                loc_cols, loc_w = np.concatenate(cc), np.concatenate(ww)
            if loc_rows is None:
                ii, jj = np.meshgrid(np.arange(npatch), np.arange(npatch), indexing="ij")
                r = bo + (h[:, None, None] * L + nglo + ii[None]) * L + nglo + jj[None]
                add(r, loc_cols[None] * nH + h[:, None, None])
            else:
                pi, qi = loc_rows
                r = bo + (h[:, None] * L + nglo + pi[None]) * L + nglo + qi[None]
                add(r, loc_cols[None] * nH + h[:, None], np.broadcast_to(loc_w[None], r.shape))
            if nglo:
                add(bo + h * L * L, n0 + n1 + h)                                                   # g2g
                j = np.arange(1, L)
                add(bo + h[:, None] * L * L + j[None], n0 + h[:, None] + 0 * j[None])              # g2l[0]: row 0
                add(bo + (h[:, None] * L + j[None]) * L, n0 + nH + h[:, None] + 0 * j[None])       # g2l[1]: column 0
            offs.append(bo)
            o = _al4(bo + nH * L * L)
    fwd, bwd = _csr(np.concatenate(rows), np.concatenate(cols), np.concatenate(vals), o, n0 + n1 + (nH if nglo else 0),
                    device)
    ent = _plans[key] = ((fwd, bwd, o), tuple(offs))
    return ent


# ---- modules ----------------------------------------------------------------------------------------------------------
class Mlp(nn.Module):
    """:18-35 (GELU, drop 0)"""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.GELU, drop=0.):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.act = act_layer()
        self.fc2 = nn.Linear(hidden_features, out_features)
        self.drop = nn.Dropout(drop)

    def fused(self, y: Tensor, cc: _CastCache) -> Tensor:
        """y bf16 [T, C] -> fc2(GELU(fc1(y))) bf16; fc2.bias gets its gradient from the residual-add consumer"""
        return linear.MlpFn.apply(y, self.fc1.weight, cc.nograd(self.fc1.weight), self.fc1.bias, self.fc2.weight,
                                  cc.nograd(self.fc2.weight), self.fc2.bias)


def _lin(y: Tensor, lin: nn.Linear, cc: _CastCache) -> Tensor:
    return linear.LinearFn.apply(y, lin.weight, cc.nograd(lin.weight), lin.bias)


class Attention(nn.Module):
    """:38-151 with rpe: dense multi-head attention plus the [nH, N, N] relative-position bias (global row / column from
    g2g / g2l, the local block from the table, bicubic-resized when the map is not wx x wy)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0., rpe=False, wx=14,
                 wy=14, nglo=1):
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = qk_scale or head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)
        self.rpe = rpe
        if not rpe:
            raise NotImplementedError("ViL Attention without rpe (ape, `a1`) is not implemented")
        self.wx, self.wy, self.nglo = wx, wy, nglo
        self.local_relative_position_bias_table = nn.Parameter(torch.zeros((2 * wx - 1) * (2 * wy - 1), num_heads))
        _trunc_normal_(self.local_relative_position_bias_table)
        if nglo >= 1:
            self.g2l_relative_position_bias = nn.Parameter(torch.zeros(2, num_heads, nglo))
            self.g2g_relative_position_bias = nn.Parameter(torch.zeros(num_heads, nglo, nglo))
            _trunc_normal_(self.g2l_relative_position_bias)
            _trunc_normal_(self.g2g_relative_position_bias)
        self.register_buffer("relative_position_index", dense_relative_position_index(wx, wy))

    def fused(self, y: Tensor, groups, Ns, cc: _CastCache) -> Tensor:
        """y bf16 [T, C] (groups ((B, row0), ...) of Ns tokens per image) -> proj(attention) bf16 [T, C]"""
        (plan, offs) = bias_plan(self, Ns, y.device)
        bias = ops.RelBiasFn.apply(self.local_relative_position_bias_table,
                                   getattr(self, "g2l_relative_position_bias", None),
                                   getattr(self, "g2g_relative_position_bias", None), plan)
        qkv = _lin(y, self.qkv, cc)
        dg = tuple((B, N, r0, bo) for (B, r0), N, bo in zip(groups, Ns, offs))
        a = ops.DenseBiasAttnGroupsFn.apply(qkv, self.qkv.bias, bias, dg, self.num_heads, float(self.scale))
        return _lin(a, self.proj, cc)


class Long2DSCSelfAttention(nn.Module):
    """layers/longformer2d.py:11-137 for the served case (rpe, sharew, one global token, exact 0, w 7): the modules and
    buffers of the reference; the attention runs on the sliding-chunk kernels (vil_attn.cu)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_scale=None, attn_drop=0., proj_drop=0., w=7, d=1,
                 autoregressive=False, sharew=False, nglo=1, only_glo=False, exact=0, autograd=False, rpe=False,
                 add_pooled=False, pool_size=1, mode=0, pool_method=None, wx=14, wy=14):
        super().__init__()
        for bad, key in ((only_glo, "only_glo"), (not sharew, "sharew False"), (add_pooled, "add_pooled"),
                         (exact != 0, "sw_exact != 0"), (not rpe, "ape (`a1`)"), (w != W, f"w != {W} (`f`)"),
                         (nglo != 1, "Nglo != 1 (`g`)"), (d != 1, "dilation")):
            if bad:
                raise NotImplementedError(f"ViL sliding-chunk attention: {key} is not implemented")
        self.num_heads = num_heads
        self.head_dim = dim // num_heads
        self.scale = qk_scale or self.head_dim ** -0.5
        self.Nglo = self.nglo = nglo
        self.only_glo = only_glo
        self.query = nn.Linear(dim, dim, bias=qkv_bias)
        self.kv = nn.Linear(dim, dim * 2, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.query_global = self.query
        self.kv_global = self.kv
        self.proj_global = self.proj
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj_drop = nn.Dropout(proj_drop)
        self.attention_window = w
        self.attention_dilation = d
        self.autoregressive = autoregressive
        self.exact = exact
        self.rpe = rpe
        self.local_relative_position_bias_table = nn.Parameter(torch.zeros((4 * w - 1) * (4 * w - 1), num_heads))
        _trunc_normal_(self.local_relative_position_bias_table)
        self.g2l_relative_position_bias = nn.Parameter(torch.zeros(2, num_heads, nglo))
        self.g2g_relative_position_bias = nn.Parameter(torch.zeros(num_heads, nglo, nglo))
        _trunc_normal_(self.g2l_relative_position_bias)
        _trunc_normal_(self.g2g_relative_position_bias)
        self.register_buffer("relative_position_index", sc_relative_position_index(w))
        self.add_pooled = False
        self.pool_method = pool_method
        self.mode = mode

    def fused(self, y: Tensor, groups, geo, modes: Tensor, cc: _CastCache) -> Tensor:
        """y bf16 [T, C] (groups ((B, row0), ...), geo ((nx, ny), ...)) -> proj(attention) bf16 [T, C]; modes int32
        [G] on the device"""
        Ns = [1 + nx * ny for nx, ny in geo]
        (plan, offs) = bias_plan(self, Ns, y.device)
        bias = ops.RelBiasFn.apply(self.local_relative_position_bias_table, self.g2l_relative_position_bias,
                                   self.g2g_relative_position_bias, plan)
        q = _lin(y, self.query, cc)
        kv = _lin(y, self.kv, cc)
        sg = tuple((B, nx, ny, r0, bo, bgo) for (B, r0), (nx, ny), (bo, bgo) in zip(groups, geo, offs))
        a = ops.SlidingChunkAttnGroupsFn.apply(q, kv, self.query.bias, self.kv.bias, bias, modes, sg, self.num_heads,
                                               float(self.scale))
        return _lin(a, self.proj, cc)


class PatchEmbed(nn.Module):
    """:191-259 with ape False: conv -> norm_embed (LN over the patch rows) -> cat(cls_token, x)"""

    def __init__(self, patch_size, nx, ny, in_chans=3, embed_dim=768, nglo=1, norm_layer=nn.LayerNorm, norm_embed=True,
                 drop_rate=0.0, ape=True):
        super().__init__()
        if ape:
            raise NotImplementedError("ViL PatchEmbed: ape (`a1`) is not implemented")
        if not norm_embed:
            raise NotImplementedError("ViL PatchEmbed: NORM_EMBED False is not implemented")
        self.patch_size = (patch_size, patch_size)
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm_embed = norm_layer(embed_dim)
        self.nx, self.ny = nx, ny
        self.Nglo = nglo
        if nglo >= 1:
            self.cls_token = nn.Parameter(torch.zeros(1, nglo, embed_dim))
            _trunc_normal_(self.cls_token)
        else:
            self.cls_token = None
        self.ape = ape
        self.pos_drop = nn.Dropout(p=drop_rate)

    def w16(self, cc: _CastCache) -> Tensor:
        """bf16 [Cout, Kp] GEMM operand: the weight in (c, ky, kx) order, K padded to a multiple of 8"""
        k = ("vil_embed", id(self.proj.weight))
        t = cc.d.get(k)
        if t is None:
            w = self.proj.weight.detach().reshape(self.proj.weight.shape[0], -1)
            t = cc.d[k] = nn.functional.pad(w, (0, -w.shape[1] % 8)).to(BF16)
        return t

    def fused(self, src, prev, cc: _CastCache) -> Tensor:
        """crops (list of fp32 NCHW, one per group) or the previous stage's stream fp32 [T, Cin] with prev = ((B, N,
        off, H, W, row0), ...) -> the new residual stream fp32 [T', C]"""
        p = self.patch_size[0]
        if prev is None:
            pe = ops.ConvEmbedFn.apply(None, self.proj.weight, self.w16(cc), self.proj.bias, src, None, p, p, 0)
            hw = [(im.shape[0], (im.shape[2] // p) * (im.shape[3] // p)) for im in src]
        else:
            pe = ops.VilStreamEmbedFn.apply(src, self.proj.weight, self.w16(cc), self.proj.bias, prev, p)
            hw = [(B, (H // p) * (Wd // p)) for B, N, off, H, Wd, r0 in prev]
        _, y = ops.add_layer_norm(None, pe, None, self.norm_embed.weight, self.norm_embed.bias, self.norm_embed.eps,
                                  y_bf16=False, delta_bias=self.proj.bias)
        if self.cls_token is None:
            return y
        return ops.ClsCatGroupsFn.apply(y, self.cls_token, tuple(hw))


class AttnBlock(nn.Module):
    """:295-379 (attn_type 'full' or 'longformerhand'); drop_path is parameter-free, the keeps are drawn by MsViT"""

    def __init__(self, dim, num_heads, qkv_bias=False, qk_scale=None, drop=0., attn_drop=0., drop_path=0.,
                 norm_layer=nn.LayerNorm, attn_type='full', w=7, d=1, sharew=False, nglo=1, only_glo=False,
                 seq_len=None, num_feats=256, share_kv=False, sw_exact=0, rratio=2, rpe=False, wx=14, wy=14,
                 add_pooled=False, pool_size=1, mode=0, pool_method=None, with_se=False, se_mlp_ratio=0.625):
        super().__init__()
        if with_se:
            raise NotImplementedError("ViL: with_se is not implemented")
        if drop or attn_drop:
            raise NotImplementedError("ViL: DROP / attn_drop > 0 is not implemented")
        if dim != 32 * num_heads:
            raise NotImplementedError(f"ViL: head dim 32 only (dim {dim}, {num_heads} heads)")
        self.norm = norm_layer(dim)
        if attn_type == 'full':
            if nglo > 1:
                raise NotImplementedError("ViL: Nglo > 1 (`g`) is not implemented")
            self.attn = Attention(dim, num_heads=num_heads, qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop,
                                  proj_drop=drop, rpe=rpe, wx=wx, wy=wy, nglo=nglo)
        elif attn_type == 'longformerhand':
            self.attn = Long2DSCSelfAttention(dim, exact=sw_exact, num_heads=num_heads, qkv_bias=qkv_bias,
                                              qk_scale=qk_scale, attn_drop=attn_drop, proj_drop=drop, w=w, d=d,
                                              sharew=sharew, nglo=nglo, only_glo=only_glo, autograd=False, rpe=rpe,
                                              add_pooled=add_pooled, pool_size=pool_size, mode=mode,
                                              pool_method=pool_method, wx=wx, wy=wy)
        else:
            raise NotImplementedError(f"ViL: attention type {attn_type!r} is not implemented (longformerhand / full)")
        self.drop_prob = float(drop_path)
        self.drop_path = nn.Identity()
        self.se = None


class MlpBlock(nn.Module):
    """:382-403"""

    def __init__(self, dim, out_dim=None, mlp_ratio=4., drop=0., drop_path=0., act_layer=nn.GELU,
                 norm_layer=nn.LayerNorm, balanced_mlp_ratio=0.0):
        super().__init__()
        if act_layer is not nn.GELU or drop or balanced_mlp_ratio or (out_dim is not None and out_dim != dim):
            raise NotImplementedError("ViL MlpBlock: GELU, drop 0, no SE balance and out_dim == dim only")
        self.drop_prob = float(drop_path)
        self.drop_path = nn.Identity()
        self.norm = norm_layer(dim)
        self.mlp = Mlp(in_features=dim, hidden_features=int(dim * mlp_ratio), out_features=out_dim, act_layer=act_layer,
                       drop=drop)
        self.shortcut = nn.Identity()


class MsViT(MultiCropBackbone):
    """:406-769"""

    def __init__(self, arch, img_size=512, in_chans=3, num_classes=1000, qkv_bias=True, qk_scale=None, drop_rate=0.,
                 attn_drop_rate=0., drop_path_rate=0., norm_layer=partial(nn.LayerNorm, eps=1e-6), norm_embed=False, w=7,
                 d=1, sharew=False, only_glo=False, share_kv=False, attn_type='longformerhand', sw_exact=0, mode=0,
                 pool_method=None, use_dense_prediction=False, with_se=False, se_mlp_ratio=0.625,
                 se_mlp_balance=False, **args):
        super().__init__()
        self.num_classes = num_classes
        # the reference reads ln_eps into self.norm_layer but builds every layer with norm_layer (:419-424)
        self.norm_layer = partial(nn.LayerNorm, eps=args['ln_eps']) if 'ln_eps' in args else norm_layer
        self.drop_path_rate = drop_path_rate
        self.attn_type = attn_type
        if attn_type not in ('longformerhand', 'full'):
            raise NotImplementedError(f"ViL: ATTN_TYPE {attn_type!r} is not implemented (longformerhand / full)")
        if args.get('avg_pool', False):
            raise NotImplementedError("ViL: AVG_POOL True is not implemented")
        self.attn_args = dict(attn_type=attn_type, qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop_rate,
                              attn_drop=attn_drop_rate, w=w, d=d, sharew=sharew, only_glo=only_glo, share_kv=share_kv,
                              sw_exact=sw_exact, norm_layer=norm_layer, mode=mode, pool_method=pool_method,
                              with_se=with_se, se_mlp_ratio=se_mlp_ratio)
        self.patch_embed_args = dict(norm_layer=norm_layer, norm_embed=norm_embed, drop_rate=drop_rate)
        self.mlp_args = dict(mlp_ratio=4.0, norm_layer=norm_layer, act_layer=nn.GELU, drop=drop_rate,
                             balanced_mlp_ratio=se_mlp_ratio if (se_mlp_balance and with_se) else 0.0)
        self.Nx = self.Ny = img_size

        def parse_arch(arch):
            layer_cfgs = []
            for layer in arch.split('_'):
                cfg = {'l': 1, 'h': 3, 'd': 192, 'n': 1, 's': 1, 'g': 1, 'p': 2, 'f': 7, 'a': 1, 'r': 0}
                for attr in layer.split(','):
                    cfg[attr[0]] = int(attr[1:])
                layer_cfgs.append(cfg)
            return layer_cfgs

        self.layer_cfgs = parse_arch(arch)
        self.num_layers = len(self.layer_cfgs)
        if self.num_layers != 4:
            raise NotImplementedError(f"ViL: {self.num_layers}-stage archs are not implemented (4 stages only)")
        for i, cfg in enumerate(self.layer_cfgs):
            for bad, key in ((cfg['a'] != 0, 'a (ape)'), (cfg['f'] != 7, 'f'), (cfg['g'] > 1, 'g'),
                             (cfg['r'] != 0, 'r (add_pooled)'), (cfg['d'] != 32 * cfg['h'], 'h (head dim 32 only)')):
                if bad:
                    raise NotImplementedError(f"ViL: layer {i + 1} key {key} = {cfg} is not implemented")
        if self.layer_cfgs[-1]['g'] != 0:
            raise NotImplementedError("ViL: a global token in the last stage (`g1` in layer 4) is not implemented")
        self.depth = sum(cfg['n'] for cfg in self.layer_cfgs)
        self.out_planes = self.layer_cfgs[-1]['d']
        self.num_features = self.out_planes
        self.Nglos = [cfg['g'] for cfg in self.layer_cfgs]
        self.avg_pool = args.get('avg_pool', False)
        dprs = torch.linspace(0, drop_path_rate, self.depth).split([cfg['n'] for cfg in self.layer_cfgs])
        self.layer1 = self._make_layer(in_chans, self.layer_cfgs[0], dprs=dprs[0], layerid=1)
        self.layer2 = self._make_layer(self.layer_cfgs[0]['d'], self.layer_cfgs[1], dprs=dprs[1], layerid=2)
        self.layer3 = self._make_layer(self.layer_cfgs[1]['d'], self.layer_cfgs[2], dprs=dprs[2], layerid=3)
        self.layer4 = self._make_layer(self.layer_cfgs[2]['d'], self.layer_cfgs[3], dprs=dprs[3], layerid=4)
        self.norm = norm_layer(self.out_planes)
        self.head = nn.Linear(self.out_planes, num_classes) if num_classes > 0 else nn.Identity()
        self.use_dense_prediction = use_dense_prediction
        if self.use_dense_prediction:
            self.head_dense = None
        self.apply(self._init_weights)
        self._forced_modes = None

    def _make_layer(self, in_dim, layer_cfg, dprs, layerid=0):
        c = layer_cfg
        if layerid != c['l']:
            raise ValueError(f"layer id {c['l']} in the arch string, expected {layerid}")
        self.Nx = nx = self.Nx // c['p']
        self.Ny = ny = self.Ny // c['p']
        self.attn_args['nglo'] = c['g']
        self.patch_embed_args['nglo'] = c['g']
        self.attn_args['num_feats'] = c['f']
        self.attn_args['rratio'] = c['f']
        self.attn_args['w'] = c['f']
        if c['s'] == 0:
            self.attn_args['attn_type'] = 'full'  # as in the reference, this sticks for the later stages
        if self.attn_args['attn_type'] == 'longformerhand' and c['g'] != 1:
            raise NotImplementedError("ViL: sliding-chunk attention needs exactly one global token (`g1`)")
        layers = [PatchEmbed(c['p'], nx, ny, in_chans=in_dim, embed_dim=c['d'], ape=c['a'], **self.patch_embed_args)]
        for dpr in dprs:
            layers.append(AttnBlock(c['d'], c['h'], drop_path=float(dpr), seq_len=nx * ny + c['g'], rpe=not c['a'],
                                    wx=nx, wy=ny, add_pooled=c['r'], pool_size=self.attn_args['w'], **self.attn_args))
            layers.append(MlpBlock(c['d'], drop_path=float(dpr), **self.mlp_args))
        return nn.Sequential(*layers)

    def _init_weights(self, m):
        if isinstance(m, nn.Linear):
            _trunc_normal_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'pos_embed', 'cls_token', 'norm.weight', 'norm.bias', 'norm_embed', 'head.bias', 'relative_position'}

    def get_classifier(self):
        return self.head

    def reset_vil_mode(self, mode):
        """:700-709: the mode of every sliding-chunk attention"""
        for m in self.modules():
            if isinstance(m, Long2DSCSelfAttention):
                m.mode = mode

    def force_modes(self, modes) -> None:
        """Test hook: the sliding-chunk modes of the following forwards.  A list of ints is consumed in the reference's
        draw order (group-major, then block order; only the calls that draw, i.e. train mode with mode > 0); an int32
        device tensor [sliding-chunk modules, groups] is used as it is by every forward; None restores the draws."""
        self._forced_modes = list(modes) if isinstance(modes, (list, tuple)) else modes

    # ---- the fused path -----------------------------------------------------------------------------------------
    def _layer(self, i: int):
        return getattr(self, f'layer{i + 1}')

    def _sc_modules(self):
        return [blk.attn for i in range(self.num_layers) for blk in self._layer(i)
                if isinstance(blk, AttnBlock) and isinstance(blk.attn, Long2DSCSelfAttention)]

    def _modes(self, G: int, device) -> Optional[Tensor]:
        """int32 [sliding-chunk modules, G] for this forward: longformer2d.py:146-156 per (module, group)"""
        mods = self._sc_modules()
        if not mods:
            return None
        fixed = [None if (m.mode > 0 and self.training) else (0 if m.mode > 0 else int(m.mode)) for m in mods]
        f = self._forced_modes
        if isinstance(f, Tensor):
            if tuple(f.shape) != (len(mods), G) or f.dtype != torch.int32:
                raise ValueError(f"forced modes must be int32 [{len(mods)}, {G}]")
            return f
        if isinstance(f, list):
            n = sum(v is None for v in fixed) * G
            if len(f) < n:
                raise ValueError(f"{len(f)} forced modes left, this forward draws {n}")
            seq, self._forced_modes = f[:n], f[n:]
            it = iter(seq)
            vals = [[None] * G for _ in mods]
            for g in range(G):
                for k, v in enumerate(fixed):
                    vals[k][g] = next(it) if v is None else v
            return torch.tensor(vals, dtype=torch.int32).to(device)
        cache = self.__dict__.setdefault("_mode_cache", {})
        key = (tuple(fixed), G, device)
        const = cache.get(key)
        if const is None:  # built eagerly before a CUDA-graph capture replays the step: no copy inside the step
            const = cache[key] = torch.tensor([[0 if v is None else v] * G for v in fixed], dtype=torch.int32).to(device)
        if all(v is not None for v in fixed):
            return const
        r = torch.randint(1, 9, (len(mods), G), dtype=torch.int32, device=device)
        if any(v is not None for v in fixed):
            draw = cache.get(("draw",) + key)
            if draw is None:
                draw = cache[("draw",) + key] = torch.tensor([[v is None] * G for v in fixed]).to(device)
            r = torch.where(draw, r, const)
        return r

    def _geometry(self, imgs: Sequence[Tensor]):
        """per stage: ((B, H, W, N, row0), ...) with N = Nglo + H*W rows per image"""
        backbone.check_crops(imgs)
        sizes = [(im.shape[0], im.shape[2], im.shape[3]) for im in imgs]
        geo = []
        for i, cfg in enumerate(self.layer_cfgs):
            p = cfg['p']
            sizes = [(B, H // p, Wd // p) for B, H, Wd in sizes]
            st, r0 = [], 0
            for B, H, Wd in sizes:
                if H < 1 or Wd < 1:
                    raise ValueError(f"crops of {tuple(imgs[0].shape)} leave no tokens at stage {i + 1}")
                N = cfg['g'] + H * Wd
                st.append((B, H, Wd, N, r0))
                r0 += B * N
            geo.append(tuple(st))
        return geo

    def _depths(self) -> List[int]:
        return [cfg['n'] for cfg in self.layer_cfgs]

    def _run(self, imgs: List[Tensor], taps=None):
        """-> (stream fp32 [T, C] after the last stage, pending delta, last-stage geometry); taps: see backbone.tap,
        called after each MlpBlock with the stage's geometry."""
        cc = _CastCache()
        geo = self._geometry(imgs)
        modes = self._last_modes = self._modes(len(imgs), imgs[0].device)
        k_sc = 0
        x, pend, prev, b = None, None, None, 0
        for i in range(self.num_layers):
            layer = self._layer(i)
            st = geo[i]
            emb = layer[0]
            if i == 0:
                x = emb.fused(list(imgs), None, cc)
            else:
                x = emb.fused(ops.residual_add(x, *pend) if pend is not None else x, prev, cc)
            pend = None
            # the DropPath scales of the AttnBlock and MlpBlock of every block, per image (the global row included)
            scales = backbone.drop_path_scales(self, [blk.drop_prob for blk in layer[1:]],
                                               sum(B for B, _, _, _, _ in st), x.device)
            keeps = backbone.drop_path_rows(self, scales, [(B, N) for B, _, _, N, _ in st], x.device)
            groups = tuple((B, r0) for B, _, _, _, r0 in st)
            Ns = [N for _, _, _, N, _ in st]
            for j in range((len(layer) - 1) // 2):
                ab, mb = layer[1 + 2 * j], layer[2 + 2 * j]
                k1 = keeps[2 * j] if keeps is not None and ab.drop_prob > 0. else None
                k2 = keeps[2 * j + 1] if keeps is not None and mb.drop_prob > 0. else None
                if isinstance(ab.attn, Long2DSCSelfAttention):
                    sc_modes = modes[k_sc]
                    k_sc += 1
                    attend = partial(ab.attn.fused, groups=groups, geo=[(H, Wd) for _, H, Wd, _, _ in st],
                                     modes=sc_modes, cc=cc)
                else:
                    attend = partial(ab.attn.fused, groups=groups, Ns=Ns, cc=cc)
                x, pend = backbone.pre_norm_block(x, pend, ab.norm, attend, mb.norm, ab.attn.proj.bias,
                                                  partial(mb.mlp.fused, cc=cc), mb.mlp.fc2.bias, k1, k2)
                x, pend = backbone.tap(taps, b, x, pend, st)
                b += 1
            prev = tuple((B, N, self.Nglos[i], H, Wd, r0) for B, H, Wd, N, r0 in st)
        return x, pend, geo[-1]

    def _tap_feature(self, i: int, x: Tensor, st) -> Tensor:
        """:636-676: the global row of a block's output where the stage has one (:665-666), else its token mean"""
        if self.Nglos[i] > 0:
            return ops.VitSplitGroupsFn.apply(x, tuple((B, H * Wd) for B, H, Wd, _, _ in st))[0]
        return ops.TokenMeanGroupsFn.apply(x, tuple((B, H, Wd, r0) for B, H, Wd, _, r0 in st))

    def _features(self, imgs: List[Tensor], taps=None):
        """-> (x_cls fp32 [sum B, C] = token mean of the final norm's tokens, x_region fp32 [sum B*N, C], tokens per
        image)"""
        x, pend, st = self._run(imgs, taps)
        region = self._final_norm(x, pend)
        pooled = ops.TokenMeanGroupsFn.apply(region, tuple((B, H, Wd, r0) for B, H, Wd, _, r0 in st))
        return pooled, region, [N for _, _, _, N, _ in st]


def get_cls_model(config, is_teacher=False, use_dense_prediction=False, **kwargs):
    """:772-804 (yacs config in, nn.Module out)"""
    s = config.MODEL.SPEC
    m = s.MSVIT
    args = dict(img_size=config.TRAIN.IMAGE_SIZE[0], drop_rate=s.DROP, drop_path_rate=0.0 if is_teacher else s.DROP_PATH,
                norm_embed=s.NORM_EMBED, avg_pool=s.AVG_POOL, arch=m.ARCH, sharew=m.SHARE_W, attn_type=m.ATTN_TYPE,
                share_kv=m.SHARE_KV, only_glo=m.ONLY_GLOBAL, sw_exact=m.SW_EXACT, ln_eps=m.LN_EPS, mode=m.MODE,
                pool_method=m.POOL_METHOD, use_dense_prediction=use_dense_prediction, with_se=m.WITH_SE,
                se_mlp_ratio=m.SE_MLP_RATIO, se_mlp_balance=m.SE_MLP_BALANCE)
    return MsViT(num_classes=config.MODEL.NUM_CLASSES, **args)


# the README's vil_2262 command line over experiments/imagenet/vil/vil_small/base.yaml
VIL_2262 = dict(arch='l1,h3,d96,n2,s1,g1,p4,f7,a0_l2,h6,d192,n2,s1,g1,p2,f7,a0_l3,h12,d384,n6,s0,g1,p2,f7,a0_'
                     'l4,h24,d768,n2,s0,g0,p2,f7,a0',
                img_size=224, drop_rate=0.0, drop_path_rate=0.1, norm_embed=True, avg_pool=False, sharew=True,
                attn_type='longformerhand', share_kv=True, only_glo=False, sw_exact=0, ln_eps=1e-6, mode=1,
                pool_method=None, with_se=False)


def msvit(spec: Optional[dict] = None, num_classes: int = 0, use_dense_prediction: bool = False,
          drop_path_rate: Optional[float] = None) -> MsViT:
    """MsViT with get_cls_model's arguments from a dict (default: vil_2262)"""
    spec = dict(VIL_2262 if spec is None else spec)
    if drop_path_rate is not None:
        spec['drop_path_rate'] = drop_path_rate
    return MsViT(num_classes=num_classes, use_dense_prediction=use_dense_prediction, **spec)
