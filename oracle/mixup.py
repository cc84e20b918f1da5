"""Functional fp32 oracle of DINOLoss with mixup targets (``--use_mixup``) and timm's mixup targets.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into
the reference's main_esvit.py.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


def dino_loss_mixup(student_output: Tensor, teacher_output: Tensor, center: Tensor, ncrops: int, temp: float,
                    targets_mixup: Sequence[Tensor], student_temp: float = 0.1) -> Tensor:
    """DINOLoss.forward with mixup targets, without the center update (main_esvit.py:638-641), restated in the folded
    form the kernels compute: per view v and student sample b, the mixed teacher row q~ = sum_{iq != v} T_v[:, b]^T q^iq
    and its mass C = sum_{iq != v} sum_j T_v[j, b]; term (iq, v) summed over iq = mean_b (C * LSE(s_vb) - <q~, s_vb>)."""
    s = (student_output / student_temp).chunk(ncrops)
    q = F.softmax((teacher_output - center) / temp, dim=-1).detach().chunk(2)
    B = q[0].shape[0]
    total = 0.0
    for v in range(ncrops):
        T = targets_mixup[v].to(s[v].dtype)
        iqs = [iq for iq in range(2) if iq != v]
        q_mix = sum(T.t() @ q[iq] for iq in iqs)
        mass = T.sum(0) * len(iqs)
        total = total + (mass * torch.logsumexp(s[v], dim=-1) - (q_mix * s[v]).sum(-1)).sum() / B
    return total / (2 * ncrops - 2)


def timm_mixup_target(B: int, lam, smoothing: float = 0.0) -> Tensor:
    """The targets timm 0.3.2's Mixup(num_classes=B) gives for labels arange(B) (timm/data/mixup.py, mixup_target):
    lam * onehot(j) + (1 - lam) * onehot(B - 1 - j) with on / off values 1 - eps + eps / B and eps / B.  lam is a float
    ("batch" mode) or a [B] tensor ("pair" / "elem" mode, one value per row)."""
    off = smoothing / B
    on = 1.0 - smoothing + off
    target = torch.arange(B)
    y1 = torch.full((B, B), off).scatter_(1, target.view(-1, 1), on)
    y2 = torch.full((B, B), off).scatter_(1, target.flip(0).view(-1, 1), on)
    lam = torch.as_tensor(lam, dtype=torch.float32)
    if lam.dim() == 1:
        lam = lam.unsqueeze(1)
    return y1 * lam + y2 * (1.0 - lam)
