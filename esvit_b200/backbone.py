"""What the four backbones (Swin, ViT / DeiT, CvT, ViL) share on the host: the multi-crop entry points over resolution
groups, the DropPath scales, the pre-norm block step on the residual stream, the probe taps and the bf16 weight cache of
a forward call.

A backbone derives from MultiCropBackbone and provides what differs between them:
  * ``_run(imgs, taps)``: one pass over the crops (fp32, one tensor per resolution group) -> (stream fp32 [T, C],
    pending (delta bf16, keep, delta_bias) or None, the last stage's geometry).  taps is None or one entry per block in
    execution order, each None or a callable (x, geometry) handed to ``tap``;
  * ``_features(imgs, taps)`` -> (pooled fp32 [sum B, C], region fp32 [T, C], tokens per image of each group), through
    ``_final_norm``;
  * ``_tap_feature(stage, x, geometry)``: the probe feature of a block output (the final norm already applied on the
    last stage);
  * ``_depths()``: the blocks per stage.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn as nn

from . import ops, shadow

Tensor = torch.Tensor


class _CastCache:
    """bf16 copies of weights shared by the resolution groups of one forward call (one cast per step)."""

    def __init__(self):
        self.d: Dict[int, Tensor] = {}

    def expanded_bias(self, table: Tensor, num_heads: int, ws: int) -> Optional[Tensor]:
        """the rel-pos bias table expanded once per forward call (ops.expand_rel_pos_bias), shared by the crop groups."""
        k = ("B", id(table))
        if k not in self.d:
            self.d[k] = ops.expand_rel_pos_bias(table, num_heads, ws)
        return self.d[k]

    def nograd(self, p: Tensor) -> Tensor:
        k = ("ng", id(p))
        t = self.d.get(k)
        if t is None:
            t = self.d[k] = shadow.as_bf16(p)  # optimiser-maintained bf16 shadow when registered, else a cast
        return t


# ---- DropPath ---------------------------------------------------------------------------------------------------------
def _cached(owner: nn.Module, key, make) -> Tensor:
    """owner's device tensor for key, built by make() once: eagerly, before a CUDA-graph capture replays the step, so
    the step makes no host-to-device copy"""
    cache = owner.__dict__.setdefault("_drop_path_cache", {})
    t = cache.get(key)
    if t is None:
        if len(cache) >= 32:  # a handful of crop geometries per run; keep the cache from growing with odd batches
            cache.clear()
        t = cache[key] = make()
    return t


def drop_path_scales(owner: nn.Module, probs: Sequence[float], samples: int, device) -> Optional[Tensor]:
    """timm 0.3.2 DropPath scales floor(keep + U) / keep, keep = 1 - p: fp32 [len(probs), samples], one per (DropPath
    call, sample), from one torch.rand.  None when owner is in eval mode or no probability is positive."""
    if not owner.training or not any(p > 0. for p in probs):
        return None
    kp = _cached(owner, ("keep", tuple(probs), device),
                 lambda: torch.tensor([[1.0 - p] for p in probs], dtype=torch.float32).to(device))
    r = torch.rand(kp.shape[0], samples, dtype=torch.float32, device=device)
    return r.add_(kp).floor_().div_(kp)


def row_samples(owner: nn.Module, counts, device) -> Tensor:
    """int64 [T]: the sample index of every row of a stream holding counts = ((B, rows per sample), ...) back to back."""
    counts = tuple(counts)

    def make():
        rows = torch.tensor([L for B, L in counts for _ in range(B)])
        return torch.arange(rows.numel()).repeat_interleave(rows).to(device)
    return _cached(owner, ("rows", counts, device), make)


def drop_path_rows(owner: nn.Module, scales: Optional[Tensor], counts, device) -> Optional[Tensor]:
    """per-sample scales [n, sum B] (drop_path_scales) -> per-row scales fp32 [n, T] of the stream described by counts
    (row_samples); None stays None."""
    return None if scales is None else scales.index_select(1, row_samples(owner, counts, device))


def block_keeps(block: nn.Module, B: int, L: int, device) -> List[Optional[Tensor]]:
    """[k1, k2]: the two DropPath scales (block.drop_prob) of a block called on B samples of L tokens outside its
    backbone, two per-sample draws spread per row (fp32 [B*L]); None = identity."""
    ks = [drop_path_scales(block, [block.drop_prob], B, device) for _ in range(2)]
    return [None if k is None else drop_path_rows(block, k, ((B, L),), device)[0] for k in ks]


# ---- the residual stream ----------------------------------------------------------------------------------------------
def pre_norm_block(x: Optional[Tensor], pend, norm1: nn.Module, attend, norm2: nn.Module, attn_bias: Optional[Tensor],
                   mlp, mlp_bias: Optional[Tensor], k1: Optional[Tensor], k2: Optional[Tensor]):
    """One pre-norm block on the residual stream: (x fp32 [T, C], pend = (delta bf16, keep, delta_bias) or None) ->
    (x, (mlp delta, k2, mlp_bias)).  x + pend is fused with norm1, x + k1 * attend(y) with norm2; the MLP branch's add
    is deferred into the next fused add + LN.  x None: the stream starts as fp32(delta).  attend / mlp: bf16 [T, C] ->
    bf16 [T, C] with their output bias (attn_bias / mlp_bias) already added; its gradient comes from the add + LN
    kernel.  k1 / k2: per-row DropPath scales fp32 [T] or None."""
    delta, keep, dbias = pend if pend is not None else (None, None, None)
    x, y = ops.add_layer_norm(x, delta, keep, norm1.weight, norm1.bias, norm1.eps, delta_bias=dbias)
    x, y = ops.add_layer_norm(x, attend(y), k1, norm2.weight, norm2.bias, norm2.eps, delta_bias=attn_bias)
    return x, (mlp(y), k2, mlp_bias)


def tap(taps, b: int, x: Tensor, pend, geometry):
    """After block b: if taps[b] is set, the block's output is materialised (pending residual added), handed to it with
    the geometry, and the stream continues from it -> (x, pend)."""
    if taps is None or taps[b] is None:
        return x, pend
    x = ops.residual_add(x, *pend)
    taps[b](x, geometry)
    return x, None


def check_crops(imgs: Sequence[Tensor]) -> None:
    for im in imgs:
        if im.dim() != 4 or im.shape[1] != 3:
            raise ValueError(f"expected crops [B, 3, H, W], got {tuple(im.shape)}")


class MultiCropBackbone(nn.Module):
    """The entry points every backbone shares, written on its _run / _features / _tap_feature / _depths."""

    def _final_norm(self, x: Tensor, pend) -> Tensor:
        """the final norm of the stream with its pending residual added: fp32 [T, C]"""
        delta, keep, dbias = pend if pend is not None else (None, None, None)
        _, y = ops.add_layer_norm(x, delta, keep, self.norm.weight, self.norm.bias, self.norm.eps, y_bf16=False,
                                  delta_bias=dbias)
        return y

    def forward(self, x):
        """Multi-crop forward: consecutive same-resolution crops form one group; the outputs are concatenated
        group-major exactly as the reference's per-group loop concatenates them.  -> head(pooled), or in dense mode
        (head(pooled), head_dense(region), region, tokens per image of each group)."""
        if not isinstance(x, list):
            x = [x]
        groups, start = [], 0
        for i in range(1, len(x) + 1):
            if i == len(x) or x[i].shape[-1] != x[start].shape[-1]:
                groups.append((start, i))
                start = i
        pooled, region, ntok = self._features([ops.cat_adjacent(x[s:e]).float() for s, e in groups])
        if self.use_dense_prediction:
            return self.head(pooled), self.head_dense(region), region, ntok
        return self.head(pooled)

    def forward_features(self, x: Tensor):
        """-> pooled fp32 [B, C] (and the region tokens fp32 [B, N, C] in dense mode)."""
        pooled, region, _ = self._features([x.float()])
        if self.use_dense_prediction:
            return pooled, region.view(x.shape[0], -1, region.shape[-1])
        return pooled

    def forward_return_n_last_blocks(self, x: Tensor, n: int = 1, return_patch_avgpool: bool = False, depth=[]):
        """eval_linear.py's probe features: the features of the last n blocks in execution order, concatenated.
        `depth` must list the model's blocks per stage; return_patch_avgpool is ignored, as in the reference."""
        return torch.cat(self._last_blocks(x, n, depth)[0], dim=-1)

    def _last_blocks(self, x: Tensor, n: int, depth):
        """-> ([_tap_feature of each of the last n blocks], the final norm's region tokens fp32 [T, C]).  Only a tapped
        block's output is materialised and the stream continues from it; the last block's feature is the pooled
        output of _features itself."""
        depths = self._depths()
        if [int(d) for d in depth] != depths:
            raise ValueError(f"depth {list(depth)} does not match the model's depths {depths}")
        total = sum(depths)
        if not 1 <= int(n) <= total:
            raise ValueError(f"n must be in [1, {total}], got {n}")
        out, taps = [], []
        for i, d in enumerate(depths):
            def feature(xs: Tensor, geometry, i=i):
                if i == len(depths) - 1:  # the final norm on the last stage's blocks
                    xs = ops.LayerNormFn.apply(xs, self.norm.weight, self.norm.bias, self.norm.eps, False)
                out.append(self._tap_feature(i, xs, geometry))
            b0 = len(taps)
            taps += [feature if total - int(n) <= b0 + j < total - 1 else None for j in range(d)]
        pooled, region, _ = self._features([x.float()], taps)
        return out + [pooled], region
