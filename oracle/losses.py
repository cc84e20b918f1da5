"""Functional fp32 oracle of DINOLoss / DDINOLoss and the optimiser-side helpers.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into
the reference's main_esvit.py and utils.py.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def teacher_temp_schedule(warmup_teacher_temp: float, teacher_temp: float,
                          warmup_teacher_temp_epochs: int, nepochs: int) -> np.ndarray:
    """main_esvit.py:614-618 / 677-681."""
    return np.concatenate((np.linspace(warmup_teacher_temp, teacher_temp, warmup_teacher_temp_epochs),
                           np.ones(nepochs - warmup_teacher_temp_epochs) * teacher_temp))


def dino_loss(student_output: Tensor, teacher_output: Tensor, center: Tensor, ncrops: int,
              temp: float, student_temp: float = 0.1) -> Tensor:
    """DINOLoss.forward without the center update (main_esvit.py:620-648, targets_mixup=None)."""
    s = (student_output / student_temp).chunk(ncrops)
    q = F.softmax((teacher_output - center) / temp, dim=-1).detach().chunk(2)
    total, n = 0.0, 0
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            total = total + torch.sum(-q[iq] * F.log_softmax(s[v], dim=-1), dim=-1).mean()
            n += 1
    return total / n


def region_match(s_fea: Tensor, t_fea: Tensor) -> Tensor:
    """Cosine arg-max of main_esvit.py:735-736: s_fea [B,Ts,P], t_fea [B,Tt,P] -> int64 [B,Ts];
    torch.max returns the FIRST maximal index."""
    sim = torch.matmul(F.normalize(s_fea, p=2, dim=-1), F.normalize(t_fea, p=2, dim=-1).permute(0, 2, 1))
    return sim.max(dim=2)[1]


def ddino_loss(student_output, teacher_output, center: Tensor, center_grid: Tensor, ncrops: int,
               temp: float, student_temp: float = 0.1, return_indices: bool = False):
    """DDINOLoss.forward without the center update (main_esvit.py:683-746)."""
    s_cls_out, s_region_out, s_fea, s_npatch = student_output
    t_cls_out, t_region_out, t_fea, t_npatch = teacher_output
    t_cls = F.softmax((t_cls_out - center) / temp, dim=-1).detach().chunk(2)
    t_region = F.softmax((t_region_out - center_grid) / temp, dim=-1).detach().chunk(2)
    t_fea = t_fea.chunk(2)
    N = t_npatch[0]
    B = t_region[0].shape[0] // N
    s_cls = (s_cls_out / student_temp).chunk(ncrops)
    split = [s_npatch[0]] * 2 + [s_npatch[1]] * (ncrops - 2) if ncrops > 2 else [s_npatch[0]] * 2
    split_bs = [i * B for i in split]
    s_region = torch.split(s_region_out / student_temp, split_bs, dim=0)
    s_feas = torch.split(s_fea, split_bs, dim=0)
    total, n = 0.0, 0
    indices = {}
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            loss = 0.5 * torch.sum(-t_cls[iq] * F.log_softmax(s_cls[v], dim=-1), dim=-1)
            s_r = s_region[v].view(B, split[v], -1)
            t_r = t_region[iq].view(B, N, -1)
            idx = region_match(s_feas[v].view(B, split[v], -1), t_fea[iq].view(B, N, -1))
            indices[(iq, v)] = idx
            t_idx = torch.gather(t_r, 1, idx.unsqueeze(2).expand(-1, -1, t_r.size(2)))
            loss_grid = torch.sum(-t_idx * F.log_softmax(s_r, dim=-1), dim=-1).mean(-1)
            loss = loss + 0.5 * loss_grid
            total = total + loss.mean()
            n += 1
    total = total / n
    return (total, indices) if return_indices else total


def center_update(center: Tensor, teacher_output: Tensor, momentum: float = 0.9, world_size: int = 1,
                  all_reduce: Optional[Callable[[Tensor], None]] = None) -> Tensor:
    """update_center (main_esvit.py:650-660, 752-770): column sum, SUM all-reduce,
    / (rows * world), EMA."""
    bc = torch.sum(teacher_output, dim=0, keepdim=True)
    if all_reduce is not None:
        all_reduce(bc)
    bc = bc / (len(teacher_output) * world_size)
    return center * momentum + bc * (1 - momentum)


def clip_gradients(grads: Sequence[Optional[Tensor]], clip: float) -> List[float]:
    """utils.clip_gradients (utils.py:106-115): PER-TENSOR L2 clip, in place."""
    norms = []
    for g in grads:
        if g is None:
            continue
        n = g.norm(2)
        norms.append(n.item())
        coef = clip / (n + 1e-6)
        if coef < 1:
            g.mul_(coef)
    return norms


def ema_update(teacher_params: Sequence[Tensor], student_params: Sequence[Tensor], m: float) -> None:
    """main_esvit.py:587-590: k = fl(fl(k*m) + fl((1-m)*q)), parameters only, in place."""
    with torch.no_grad():
        for k, q in zip(teacher_params, student_params):
            k.mul_(m).add_((1 - m) * q.detach())


def cosine_scheduler(base_value, final_value, epochs, niter_per_ep, warmup_epochs=0, start_warmup_value=0):
    """utils.cosine_scheduler (utils.py:161-173)."""
    warmup = np.array([])
    wi = warmup_epochs * niter_per_ep
    if warmup_epochs > 0:
        warmup = np.linspace(start_warmup_value, base_value, wi)
    it = np.arange(epochs * niter_per_ep - wi)
    sched = final_value + 0.5 * (base_value - final_value) * (1 + np.cos(np.pi * it / len(it)))
    return np.concatenate((warmup, sched))
