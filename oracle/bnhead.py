"""CPU fp32 restatement of DINOHead(use_bn=True) and of the multi-step training sequence with such heads.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  DINOHead (models/vision_transformer.py:384-418) with use_bn:
mlp = Linear, BatchNorm1d, GELU, [Linear, BatchNorm1d, GELU]*(nlayers-2), Linear.  BatchNorm1d in train mode normalises
with the biased batch variance and updates running_mean / running_var (unbiased variance) with momentum 0.1 and
num_batches_tracked += 1; in eval mode it normalises with the running statistics (eps 1e-5).  Each head is called once
per network forward on the rows of every crop, so one batch of statistics spans all resolution groups.

``OracleBnStep`` is oracle/step.py's OracleStep with these heads and the running buffers kept apart from the parameters
(the teacher EMA covers parameters only).  Backbones: the Swin (oracle/swin.py) and ViT (oracle/vit.py) oracles.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from . import golden as GD
from . import losses as L
from . import swin as S
from . import vit as V

Tensor = torch.Tensor

BN_EPS, BN_MOMENTUM = 1e-5, 0.1
BUFFERS = (".running_mean", ".running_var", ".num_batches_tracked")


def is_buffer(name: str) -> bool:
    return name.endswith(BUFFERS) or name.endswith("relative_position_index")


def bn_prefixes(names) -> set:
    return {k[:-len(".running_mean")] for k in names if k.endswith(".running_mean")}


def seeded_state_dict(rec, seed: int) -> Dict[str, Tensor]:
    """oracle/golden.py's seeded weights for a layout with BatchNorm entries: every other entry as GD.seeded_state_dict;
    the BatchNorm ones from seed + 1: weight 1 + N(0, 0.1), bias N(0, 0.05), running_mean N(0, 0.1), running_var
    1 + U(0, 1), num_batches_tracked 0."""
    pre = bn_prefixes(k for k, _, _ in rec)
    in_bn = lambda k: k.rsplit(".", 1)[0] in pre  # noqa: E731
    sd = GD.seeded_state_dict([r for r in rec if not in_bn(r[0])], seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k, shape, _ in rec:
        if not in_bn(k):
            continue
        if k.endswith(".num_batches_tracked"):
            sd[k] = torch.zeros(shape, dtype=torch.long)
        elif k.endswith(".weight"):
            sd[k] = 1 + torch.randn(shape, generator=g) * 0.1
        elif k.endswith(".bias"):
            sd[k] = torch.randn(shape, generator=g) * 0.05
        elif k.endswith(".running_mean"):
            sd[k] = torch.randn(shape, generator=g) * 0.1
        else:
            sd[k] = 1 + torch.rand(shape, generator=g)
    return {k: sd[k] for k, _, _ in rec}


def batch_norm(x: Tensor, sd: Dict[str, Tensor], p: str, train: bool) -> Tensor:
    """BatchNorm1d.forward over rows x [R, C]; train mode updates sd's running buffers in place."""
    rm, rv = sd[p + ".running_mean"], sd[p + ".running_var"]
    if train:
        n = x.shape[0]
        if n <= 1:
            raise ValueError("Expected more than 1 value per channel when training")
        mean = x.mean(0)
        var = ((x - mean) ** 2).mean(0)
        with torch.no_grad():
            rm.mul_(1 - BN_MOMENTUM).add_(BN_MOMENTUM * mean.detach())
            rv.mul_(1 - BN_MOMENTUM).add_(BN_MOMENTUM * var.detach() * n / (n - 1))
            sd[p + ".num_batches_tracked"].add_(1)
    else:
        mean, var = rm, rv
    return (x - mean) / torch.sqrt(var + BN_EPS) * sd[p + ".weight"] + sd[p + ".bias"]


def dino_head_bn(x: Tensor, sd: Dict[str, Tensor], p: str, train: bool) -> Tensor:
    """DINOHead(use_bn=True).forward (models/vision_transformer.py:384-418) for any nlayers."""
    i = 0
    while p + f".mlp.{i + 1}.running_mean" in sd:
        x = F.gelu(batch_norm(S.linear(x, sd, f"{p}.mlp.{i}"), sd, f"{p}.mlp.{i + 1}", train))
        i += 3
    x = F.normalize(S.linear(x, sd, f"{p}.mlp.{i}"), dim=-1, p=2)
    v, g = sd[p + ".last_layer.weight_v"], sd[p + ".last_layer.weight_g"]
    return F.linear(x, v * (g / v.norm(2, dim=1, keepdim=True)))


def backbone(arch: dict, sd, crops: Sequence[Tensor]):
    """(cls [sum B, D], region [sum B*N, D], npatch) of arch = {"kind": "swin", "spec": SwinSpec} or
    {"kind": "vit", "patch": p, "num_heads": h}"""
    if arch["kind"] == "vit":
        return V.forward_dense(sd, list(crops), arch["patch"], arch["num_heads"])
    cls_l, fea_l, npatch = [], [], []
    for s, e in S.group_crops(list(crops)):
        pooled, region = S.forward_features(torch.cat(list(crops[s:e])), sd, arch["spec"])
        B, N, C = region.shape
        cls_l.append(pooled)
        fea_l.append(region.reshape(B * N, C))
        npatch.append(N)
    return torch.cat(cls_l), torch.cat(fea_l), npatch


def multicrop_forward(arch: dict, sd, crops: Sequence[Tensor], dense: bool, train: bool = True):
    """the network's forward with use_bn heads: dense -> (head(cls), head_dense(region), region, npatch); view ->
    head(cls)"""
    cls, region, npatch = backbone(arch, sd, crops)
    if dense:
        return dino_head_bn(cls, sd, "head", train), dino_head_bn(region, sd, "head_dense", train), region, npatch
    return dino_head_bn(cls, sd, "head", train)


def running_stats(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    return {k: v.detach().clone() for k, v in sd.items() if k.endswith(BUFFERS)}


class OracleBnStep:
    """main_esvit.py:507-590 for one process with BN heads: lr / wd set, teacher forward (train mode, no grad), student
    forward, DINO / DDINO loss + center update, backward, per-tensor clip, cancel last-layer gradients, AdamW with
    utils.get_params_groups' groups, teacher EMA over the parameters."""

    def __init__(self, state_dict: Dict[str, Tensor], arch: dict, dense: bool, ncrops: int, out_dim: int,
                 teacher_temp: float = 0.04, student_temp: float = 0.1, center_momentum: float = 0.9,
                 lr: float = 5e-4, weight_decay: float = 0.04, clip_grad: float = 3.0, freeze_last_layer: int = 1,
                 momentum_teacher: float = 0.996, norm_last_layer: bool = True):
        self.arch, self.dense, self.ncrops = arch, dense, ncrops
        self.teacher_temp, self.student_temp, self.center_momentum = teacher_temp, student_temp, center_momentum
        self.clip_grad, self.freeze_last_layer, self.m = clip_grad, freeze_last_layer, momentum_teacher
        self.lr, self.wd = lr, weight_decay
        self.names = [k for k in state_dict if not is_buffer(k)]
        self.student = {k: v.detach().clone() for k, v in state_dict.items()}
        self.teacher = {k: v.detach().clone() for k, v in state_dict.items()}
        for k in self.names:
            self.student[k].requires_grad_(not (norm_last_layer and k.endswith("last_layer.weight_g")))
        reg = [self.student[k] for k in self.names if self.student[k].requires_grad
               and not (k.endswith(".bias") or self.student[k].dim() == 1)]
        noreg = [self.student[k] for k in self.names if self.student[k].requires_grad
                 and (k.endswith(".bias") or self.student[k].dim() == 1)]
        self.opt = torch.optim.AdamW([{"params": reg}, {"params": noreg, "weight_decay": 0.0}])
        self.center = torch.zeros(1, out_dim)
        self.center_grid = torch.zeros(1, out_dim)

    def step(self, crops: List[Tensor], epoch: int = 0):
        """-> (loss, student output, teacher output, raw student gradients)"""
        for i, g in enumerate(self.opt.param_groups):
            g["lr"] = self.lr
            if i == 0:
                g["weight_decay"] = self.wd
        with torch.no_grad():
            t_out = multicrop_forward(self.arch, self.teacher, crops[:2], self.dense)
        s_out = multicrop_forward(self.arch, self.student, crops, self.dense)
        if self.dense:
            loss = L.ddino_loss(s_out, t_out, self.center, self.center_grid, self.ncrops, self.teacher_temp,
                                self.student_temp)
            with torch.no_grad():
                self.center = L.center_update(self.center, t_out[0], self.center_momentum)
                self.center_grid = L.center_update(self.center_grid, t_out[1], self.center_momentum)
        else:
            loss = L.dino_loss(s_out, t_out, self.center, self.ncrops, self.teacher_temp, self.student_temp)
            with torch.no_grad():
                self.center = L.center_update(self.center, t_out, self.center_momentum)
        self.opt.zero_grad(set_to_none=True)
        loss.backward()
        grads = {k: self.student[k].grad.detach().clone() for k in self.names if self.student[k].grad is not None}
        params = [self.student[k] for k in self.names]
        if self.clip_grad:
            L.clip_gradients([p.grad for p in params], self.clip_grad)
        if epoch < self.freeze_last_layer:
            for k in self.names:
                if "last_layer" in k:
                    self.student[k].grad = None
        self.opt.step()
        L.ema_update([self.teacher[k] for k in self.names], params, self.m)
        return float(loss.detach()), s_out, t_out, grads
