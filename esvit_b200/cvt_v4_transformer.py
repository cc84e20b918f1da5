"""CvT backbone (models/cvt_v4_transformer.py, specs experiments/imagenet/cvt_v4/s1.yaml, s3.yaml, win_size/s1.yaml and
win_size/s3.yaml) behind the reference's signatures and state_dict keys.

CvT / get_cls_model take the reference's MODEL.SPEC keys and hold the reference's parameters AND buffers
(``stage{i}.0.{proj,norm}.*``, ``stage{i}.1.layers.{j}.0.{norm,fn.qkv.dw,fn.qkv.bn,fn.qkv.pw,fn.proj_out}.*``,
``stage{i}.1.layers.{j}.1.{norm,fn.net.0,fn.net.2}.*``, ``norm.*``), so a reference state_dict loads with strict=True.
The 1x1 convs keep their Conv2d weights [N, K, 1, 1]; the GEMMs read them as [N, K].  The BatchNorm2d modules stay real
nn.BatchNorm2d instances (parameter / buffer containers), so utils.has_batchnorms and
nn.SyncBatchNorm.convert_sync_batchnorm behave as with the reference.

Execution follows the Swin / ViT ports: an fp32 residual stream token-major [T, C] holding every crop of every resolution
group back to back, bf16 branches, the residual add + DropPath deferred into the next fused add + LN, every per-token op
(LN, GEMMs) run once over all groups; the conv embedding gather, depthwise conv + BN statistics and window attention
launch per group on pointer offsets (ops.ConvEmbedFn / DwBnFn / MhsaWinGroupsFn).  BatchNorm follows main_esvit.py: the
module's mode decides (train: batch statistics per resolution group over the zero-padded map, running statistics updated;
eval: running statistics).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist
import torch.nn as nn

from . import backbone, linear, ops
from .backbone import MultiCropBackbone, _CastCache

Tensor = torch.Tensor
BF16 = torch.bfloat16


class LayerNorm(nn.LayerNorm):
    """:35-41 (LayerNorm computed in fp32)."""

    def forward(self, x: Tensor) -> Tensor:
        return super().forward(x.float()).type(x.dtype)


class QuickGELU(nn.Module):
    """:44-46; the fused path applies it in the fc1 GEMM epilogue."""

    def forward(self, x: Tensor) -> Tensor:
        return x * torch.sigmoid(1.702 * x)


class PreNorm(nn.Module):
    def __init__(self, norm, dim, fn):
        super().__init__()
        self.norm = norm(dim)
        self.fn = fn


class FeedForward(nn.Module):
    def __init__(self, dim, act_layer, mult=4):
        super().__init__()
        self.net = nn.Sequential(nn.Conv2d(dim, int(dim * mult), 1), act_layer(), nn.Conv2d(int(dim * mult), dim, 1))

    def fused(self, y: Tensor, cc: _CastCache) -> Tensor:
        """y bf16 [T, C] -> fc2(QuickGELU(fc1(y))) bf16; fc2's bias gets its gradient from the residual-add consumer."""
        f1, f2 = self.net[0], self.net[2]
        return linear.MlpFn.apply(y, f1.weight, _w2d(cc, f1.weight), f1.bias, f2.weight, _w2d(cc, f2.weight), f2.bias, 2)


class DepthWiseConv2d(nn.Module):
    def __init__(self, dim_in, dim_out, kernel_size, padding, stride, bias=True):
        super().__init__()
        self.dw = nn.Conv2d(dim_in, dim_in, kernel_size=kernel_size, padding=padding, groups=dim_in, stride=stride,
                            bias=False)
        self.bn = nn.BatchNorm2d(dim_in)
        self.pw = nn.Conv2d(dim_in, dim_out, kernel_size=1, bias=bias)


def _w2d(cc: _CastCache, w: Tensor) -> Tensor:
    """bf16 [N, K] GEMM operand of a 1x1 conv weight [N, K, 1, 1]"""
    return cc.nograd(w).view(w.shape[0], -1)


def _sync_group(bn: nn.Module):
    """the process group whose statistics a SyncBatchNorm combines, or None (plain BN, or a world of one)"""
    if not isinstance(bn, nn.SyncBatchNorm) or not (dist.is_available() and dist.is_initialized()):
        return None
    pg = bn.process_group if bn.process_group is not None else dist.group.WORLD
    return pg if dist.get_world_size(pg) > 1 else None


class Attention(nn.Module):
    """:108-220 with head dim 64 (s1) or 32 (s3), no rel-pos bias and no shift."""

    def __init__(self, dim_in, dim_out, num_heads, qkv_bias, kernel_size, padding, window_size, shift_size,
                 rel_pos_embed, **kwargs):
        super().__init__()
        self.heads = num_heads
        self.window_size = window_size
        self.shift_size = shift_size
        self.scale = dim_out ** -0.5
        self.qkv = DepthWiseConv2d(dim_in, dim_out * 3, kernel_size, padding=padding, stride=1, bias=qkv_bias)
        self.proj_out = nn.Conv2d(dim_out, dim_in, 1)

    def fused(self, y: Tensor, wgroups, cc: _CastCache) -> Tensor:
        """y = PreNorm output bf16 [T, C] -> proj_out(attention) bf16 [T, C]; proj_out.bias gets its gradient from the
        residual-add consumer."""
        q = self.qkv
        bn = q.bn
        train = bn.training or not bn.track_running_stats
        if train and bn.track_running_stats and bn.momentum is None:
            raise NotImplementedError("BatchNorm2d(momentum=None) (cumulative running average) is not implemented")
        u = ops.DwBnFn.apply(y, q.dw.weight, bn.weight, bn.bias, bn, wgroups, train, _sync_group(bn))
        qkv = linear.LinearFn.apply(u, q.pw.weight, _w2d(cc, q.pw.weight), q.pw.bias)
        a = ops.MhsaWinGroupsFn.apply(qkv, q.pw.bias, wgroups, self.heads, float(self.scale))
        return linear.LinearFn.apply(a, self.proj_out.weight, _w2d(cc, self.proj_out.weight), self.proj_out.bias)


class Transformer(nn.Module):
    """:242-346; layers[j] = [PreNorm(Attention), PreNorm(FeedForward), DropPath]."""

    def __init__(self, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4., qkv_bias=False, drop_path_rate=None,
                 act_layer=nn.GELU, norm_layer=nn.LayerNorm, kernel_qkv=3, padding_qkv=1, window_size=-1, shift=False,
                 rel_pos_embed=False, **kwargs):
        super().__init__()
        self.layers = nn.ModuleList([])
        self.drop_probs = [float(p) for p in drop_path_rate] if isinstance(drop_path_rate, list) else [0.] * depth
        for i in range(depth):
            self.layers.append(nn.ModuleList([
                PreNorm(norm_layer, embed_dim,
                        Attention(dim_in=embed_dim, dim_out=embed_dim, num_heads=num_heads, qkv_bias=qkv_bias,
                                  kernel_size=kernel_qkv, padding=padding_qkv, window_size=window_size, shift_size=0,
                                  rel_pos_embed=rel_pos_embed)),
                PreNorm(norm_layer, embed_dim, FeedForward(embed_dim, act_layer, mlp_ratio)),
                nn.Identity(),  # DropPath: parameter-free; the per-row scales are drawn by CvT._run
            ]))
        self.window_size = window_size
        self.shift = shift

    def block(self, j: int, x: Tensor, pend, wgroups, cc: _CastCache, k1: Optional[Tensor], k2: Optional[Tensor]):
        """backbone.pre_norm_block of layer j (:333-335)"""
        attn, ff, _ = self.layers[j]
        return backbone.pre_norm_block(x, pend, attn.norm, lambda y: attn.fn.fused(y, wgroups, cc), ff.norm,
                                       attn.fn.proj_out.bias, lambda y: ff.fn.fused(y, cc), ff.fn.net[2].bias, k1, k2)


class ConvEmbed(nn.Module):
    """:349-382"""

    def __init__(self, patch_size=7, in_chans=3, embed_dim=64, stride=4, padding=2, norm_layer=None):
        super().__init__()
        self.patch_size = patch_size
        self.stride, self.padding = stride, padding
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=stride, padding=padding)
        if norm_layer is None:
            raise NotImplementedError("ConvEmbed without a norm layer is not used by CvT")
        self.norm = norm_layer(embed_dim)

    def w16(self, cc: _CastCache) -> Tensor:
        """bf16 [Cout, Kp] GEMM operand: the weight in (c, ky, kx) order, K padded to a multiple of 8 (16-byte TMA rows)"""
        k = ("cvt_embed", id(self.proj.weight))
        t = cc.d.get(k)
        if t is None:
            w = self.proj.weight.detach().reshape(self.proj.weight.shape[0], -1)
            K = w.shape[1]
            t = cc.d[k] = nn.functional.pad(w, (0, -K % 8)).to(BF16)
        return t

    def fused(self, src, groups, cc: _CastCache) -> Tensor:
        """crops (list of fp32 NCHW tensors) or the previous stage's stream fp32 [T, Cin] with groups ((B, H, W, row0),
        ...) -> LN(conv) fp32 [T', C], the new residual stream."""
        imgs = src if isinstance(src, (list, tuple)) else None
        pe = ops.ConvEmbedFn.apply(None if imgs is not None else src, self.proj.weight, self.w16(cc), self.proj.bias,
                                   imgs, groups, self.patch_size, self.stride, self.padding)
        _, x = ops.add_layer_norm(None, pe, None, self.norm.weight, self.norm.bias, self.norm.eps, y_bf16=False,
                                  delta_bias=self.proj.bias)
        return x


def _spec(spec, key, default=None):
    if isinstance(spec, dict):
        return spec.get(key, default)
    return getattr(spec, key, default)


class CvT(MultiCropBackbone):
    """:434-661"""

    def __init__(self, *, num_classes, act_layer=nn.GELU, norm_layer=nn.LayerNorm, init='trunc_norm',
                 use_dense_prediction=False, spec=None):
        super().__init__()
        self.num_stages = spec['NUM_STAGES']
        if spec['REL_POS_EMBED']:
            raise NotImplementedError("CvT: REL_POS_EMBED is not implemented")
        if any(spec['SHIFT'][:self.num_stages]):
            raise NotImplementedError("CvT: shifted windows are not implemented")
        if _spec(spec, 'RES_STEM', False):
            raise NotImplementedError("CvT: RES_STEM is not implemented")
        if act_layer is not QuickGELU:
            raise NotImplementedError("CvT: the FeedForward activation is QuickGELU (get_cls_model)")
        # the window attention kernels run head dim 64 (s1) or 32 (s3); one head dim serves every stage of a model
        head_dims = [spec['DIM_EMBED'][i] / spec['NUM_HEADS'][i] for i in range(self.num_stages)]
        if len(set(head_dims)) != 1 or head_dims[0] not in (32, 64):
            raise NotImplementedError("CvT: one head dim per model, 32 or 64 (per stage DIM_EMBED / NUM_HEADS: %s)"
                                      % ", ".join(f"{d:g}" for d in head_dims))
        for i in range(self.num_stages):
            if spec['KERNEL_QKV'][i] != 3 or spec['PADDING_QKV'][i] != 1:
                raise NotImplementedError("CvT: KERNEL_QKV 3 with PADDING_QKV 1 only")
            if spec['WINDOW_SIZE'][i] < 1:
                raise ValueError(f"CvT: WINDOW_SIZE must be >= 1 (stage {i}: {spec['WINDOW_SIZE'][i]})")
        total_depth = sum(spec['DEPTH'])
        dpr = [x.item() for x in torch.linspace(0, spec['DROP_PATH_RATE'], total_depth)]
        in_chans, depth_accum = 3, 0
        for i in range(self.num_stages):
            conv = ConvEmbed(patch_size=spec['PATCH_SIZE'][i], in_chans=in_chans, embed_dim=spec['DIM_EMBED'][i],
                             stride=spec['PATCH_STRIDE'][i], padding=spec['PATCH_PADDING'][i], norm_layer=norm_layer)
            stage = nn.Sequential(conv, Transformer(
                embed_dim=spec['DIM_EMBED'][i], depth=spec['DEPTH'][i], num_heads=spec['NUM_HEADS'][i],
                mlp_ratio=spec['MLP_RATIO'][i], qkv_bias=spec['QKV_BIAS'][i],
                drop_path_rate=dpr[depth_accum: depth_accum + spec['DEPTH'][i]], act_layer=act_layer,
                norm_layer=norm_layer, kernel_qkv=spec['KERNEL_QKV'][i], padding_qkv=spec['PADDING_QKV'][i],
                window_size=spec['WINDOW_SIZE'][i], shift=spec['SHIFT'][i], rel_pos_embed=spec['REL_POS_EMBED']))
            setattr(self, f'stage{i}', stage)
            in_chans = spec['DIM_EMBED'][i]
            depth_accum += spec['DEPTH'][i]
        self.num_features = self.embed_dim = in_chans
        self.norm = norm_layer(in_chans)
        self.head = nn.Linear(in_chans, num_classes) if num_classes > 0 else nn.Identity()
        self.use_dense_prediction = use_dense_prediction
        if self.use_dense_prediction:
            self.head_dense = None
        self.apply(self._init_weights_trunc_normal if init != 'xavier' else self._init_weights_xavier)

    def _init_weights_trunc_normal(self, m):
        if isinstance(m, (nn.Linear, nn.Conv2d)):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, (nn.LayerNorm, nn.BatchNorm2d)):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    def _init_weights_xavier(self, m):
        if isinstance(m, nn.Linear):
            nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, (nn.LayerNorm, nn.BatchNorm2d)):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)

    # ---- the fused path ---------------------------------------------------------------------------------------
    def _stage(self, i: int):
        return getattr(self, f'stage{i}')

    def _geometry(self, imgs: Sequence[Tensor]):
        """per stage: (token groups ((B, H, W, row0), ...), window groups ((B, H, W, w, row0, prow0), ...))"""
        backbone.check_crops(imgs)
        sizes = [(im.shape[0], im.shape[2], im.shape[3]) for im in imgs]
        geo = []
        for i in range(self.num_stages):
            emb, tr = self._stage(i)
            sizes = [(B, ops.conv_out_size(H, emb.patch_size, emb.stride, emb.padding),
                      ops.conv_out_size(W, emb.patch_size, emb.stride, emb.padding)) for B, H, W in sizes]
            tg, wg, r0, p0 = [], [], 0, 0
            for B, H, W in sizes:
                if H < 1 or W < 1:
                    raise ValueError(f"crops of {tuple(imgs[0].shape)} leave no tokens at stage {i}")
                w = min(tr.window_size, H, W)
                Hp, Wp = ops.win_padded(H, W, w)
                tg.append((B, H, W, r0))
                wg.append((B, H, W, w, r0, p0))
                r0 += B * H * W
                p0 += B * Hp * Wp
            geo.append((tuple(tg), tuple(wg)))
        return geo

    def _depths(self) -> List[int]:
        return [len(self._stage(i)[1].layers) for i in range(self.num_stages)]

    def _run(self, imgs: List[Tensor], taps=None):
        """-> (stream fp32 [T, C] after the last stage, pending delta, last-stage token groups); taps: see backbone.tap,
        called with the stage's token groups."""
        cc = _CastCache()
        geo = self._geometry(imgs)
        x, pend, prev, b = None, None, None, 0
        for i in range(self.num_stages):
            emb, tr = self._stage(i)
            tg, wg = geo[i]
            if i == 0:
                x = emb.fused(list(imgs), None, cc)
            else:
                x = emb.fused(ops.residual_add(x, *pend) if pend is not None else x, prev, cc)
            pend = None
            probs = [p for p in tr.drop_probs for _ in range(2)]
            scales = backbone.drop_path_scales(self, probs, sum(B for B, _, _, _ in tg), x.device)
            keeps = backbone.drop_path_rows(self, scales, [(B, H * W) for B, H, W, _ in tg], x.device)
            for j in range(len(tr.layers)):
                k1 = k2 = None
                if keeps is not None and tr.drop_probs[j] > 0.:
                    k1, k2 = keeps[2 * j], keeps[2 * j + 1]
                x, pend = tr.block(j, x, pend, wg, cc, k1, k2)
                x, pend = backbone.tap(taps, b, x, pend, tg)
                b += 1
            prev = tg
        return x, pend, geo[-1][0]

    def _tap_feature(self, i: int, x: Tensor, tg) -> Tensor:
        """:567-615: the token mean of a block's output"""
        return ops.TokenMeanGroupsFn.apply(x, tg)

    def _features(self, imgs: List[Tensor], taps=None):
        """-> (pooled fp32 [sum B, C], region fp32 [sum B*N, C] = the final norm's tokens, tokens per image)"""
        x, pend, tg = self._run(imgs, taps)
        region = self._final_norm(x, pend)
        return ops.TokenMeanGroupsFn.apply(region, tg), region, [H * W for _, H, W, _ in tg]


def get_cls_model(config, is_teacher=False, use_dense_prediction=False, **kwargs):
    """:685-707 (yacs config in, nn.Module out); the teacher gets DROP_PATH_RATE 0 without the spec being modified."""
    spec = dict(config.MODEL.SPEC)
    if is_teacher:
        spec['DROP_PATH_RATE'] = 0.0
    return CvT(num_classes=config.MODEL.NUM_CLASSES, act_layer=QuickGELU, norm_layer=_layer_norm_1e5,
               init='trunc_norm', use_dense_prediction=use_dense_prediction, spec=spec)


def _layer_norm_1e5(dim):
    return LayerNorm(dim, eps=1e-5)


# experiments/imagenet/cvt_v4/s1.yaml MODEL.SPEC
S1_SPEC = dict(INIT='trunc_norm', NUM_STAGES=4, REL_POS_EMBED=False, SHIFT=[False] * 4, DROP_PATH_RATE=0.1,
               PATCH_SIZE=[7, 3, 3, 3], PATCH_STRIDE=[4, 2, 2, 2], PATCH_PADDING=[2, 1, 1, 1], WINDOW_SIZE=[7] * 4,
               DIM_EMBED=[64, 192, 384, 768], NUM_HEADS=[1, 3, 6, 12], DEPTH=[2, 2, 6, 2], MLP_RATIO=[4.0] * 4,
               QKV_BIAS=[True] * 4, KERNEL_QKV=[3] * 4, PADDING_QKV=[1] * 4)
# experiments/imagenet/cvt_v4/win_size/s1.yaml MODEL.SPEC: s1 with 14 x 14 windows in stages 0-2
S1_W14_SPEC = dict(S1_SPEC, WINDOW_SIZE=[14, 14, 14, 7])
# experiments/imagenet/cvt_v4/s3.yaml MODEL.SPEC (head dim 32 in every stage)
S3_SPEC = dict(INIT='trunc_norm', NUM_STAGES=4, REL_POS_EMBED=False, SHIFT=[False] * 4, DROP_PATH_RATE=0.2,
               PATCH_SIZE=[7, 3, 3, 3], PATCH_STRIDE=[4, 2, 2, 2], PATCH_PADDING=[2, 1, 1, 1], WINDOW_SIZE=[7] * 4,
               DIM_EMBED=[64, 128, 256, 512], NUM_HEADS=[2, 4, 8, 16], DEPTH=[2, 2, 10, 4], MLP_RATIO=[4.0] * 4,
               QKV_BIAS=[True] * 4, KERNEL_QKV=[3] * 4, PADDING_QKV=[1] * 4)
# experiments/imagenet/cvt_v4/win_size/s3.yaml MODEL.SPEC: s3 with 14 x 14 windows in stages 0-2
S3_W14_SPEC = dict(S3_SPEC, WINDOW_SIZE=[14, 14, 14, 7])


def cvt(spec: Optional[dict] = None, num_classes: int = 0, use_dense_prediction: bool = False,
        drop_path_rate: Optional[float] = None) -> CvT:
    """CvT with get_cls_model's layers from a MODEL.SPEC dict (default: s1)"""
    spec = dict(S1_SPEC if spec is None else spec)
    if drop_path_rate is not None:
        spec['DROP_PATH_RATE'] = drop_path_rate
    return CvT(num_classes=num_classes, act_layer=QuickGELU, norm_layer=_layer_norm_1e5, init='trunc_norm',
               use_dense_prediction=use_dense_prediction, spec=spec)
