"""DINOLoss / DDINOLoss behind the reference's constructor + call signatures (main_esvit.py:603-770).

``loss(student_output, teacher_output, epoch, targets_mixup) -> 0-dim tensor``: DINOLoss weights its terms by the
mixup targets when they are given (``--use_mixup``), DDINOLoss ignores them like the reference's; buffers ``center`` (and
``center_grid``) [1, out_dim] live in ``state_dict()`` like the reference's.

Fused formulation (DESIGN.md): one streaming pass per student row over its <= 2 paired teacher rows
(ops.DinoCEFn), the DDINO region pairing comes from the cosine arg-max kernel (ops.region_match), and the two
center column sums are reduced with ONE packed all-reduce.  Nothing of shape [B, T, out_dim] is materialised.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from . import ops

BF16 = torch.bfloat16


def _teacher_temp_schedule(warmup_teacher_temp, teacher_temp, warmup_teacher_temp_epochs, nepochs):
    return np.concatenate((np.linspace(warmup_teacher_temp, teacher_temp, warmup_teacher_temp_epochs),
                           np.ones(nepochs - warmup_teacher_temp_epochs) * teacher_temp))


def _world() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


class _CenteredLoss(nn.Module):
    def __init__(self, out_dim, ncrops, warmup_teacher_temp, teacher_temp, warmup_teacher_temp_epochs, nepochs,
                 student_temp=0.1, center_momentum=0.9):
        super().__init__()
        self.student_temp = student_temp
        self.center_momentum = center_momentum
        self.ncrops = ncrops
        self.out_dim = out_dim
        self.register_buffer("center", torch.zeros(1, out_dim))
        self.teacher_temp_schedule = _teacher_temp_schedule(warmup_teacher_temp, teacher_temp,
                                                            warmup_teacher_temp_epochs, nepochs)
        self._tables: Dict[Tuple, Tuple[torch.Tensor, torch.Tensor]] = {}

    def _cls_tables(self, B: int, weight: float, device):
        """trow int32 [ncrops*B, 2]: teacher cls row of view iq for student row (v, b), -1 where v == iq."""
        key = ("cls", B, weight, str(device))
        if key not in self._tables:
            v = torch.arange(self.ncrops).repeat_interleave(B)
            b = torch.arange(B).repeat(self.ncrops)
            trow = torch.stack([torch.where(v == iq, torch.full_like(b, -1), iq * B + b) for iq in range(2)], 1)
            w = torch.full((self.ncrops * B,), weight, dtype=torch.float32)
            self._tables[key] = (trow.to(torch.int32).contiguous().to(device), w.to(device))
        return self._tables[key]

    def _order(self, B: int, groups, device) -> torch.Tensor:
        """int32 permutation of the student rows, IMAGE-major: rows are stored (crop, image, token); CTA i of the CE kernels
        works on row order[i], so the CTAs resident together share one image's teacher rows (L2 instead of DRAM re-reads).
        groups = [(number of crops, tokens per crop)] in storage order."""
        key = ("order", B, tuple(groups), str(device))
        if key not in self._tables:
            parts, base = [], 0
            for ncr, T in groups:
                idx = base + torch.arange(ncr * B * T).view(ncr, B, T)   # [crop, image, token] -> row
                parts.append(idx.permute(1, 0, 2).reshape(B, ncr * T))    # per image: its rows of this group
                base += ncr * B * T
            self._tables[key] = (torch.cat(parts, 1).reshape(-1).to(torch.int32).contiguous().to(device), None)
        return self._tables[key][0]

    @staticmethod
    def _as_bf16(t: torch.Tensor) -> torch.Tensor:
        return t if t.dtype == BF16 else t.to(BF16)

    @torch.no_grad()
    def _reduce_and_update(self, sums: torch.Tensor, rows, names):
        """sums fp32 [n, K] local column sums -> one SUM all-reduce -> EMA of each center (main_esvit.py:650-660).
        The buffers are updated IN PLACE (stable addresses: CUDA-graph replays must see the running centers); the
        loss forward therefore hands autograd a private snapshot of the pre-update center (_snapshot)."""
        world = _world()
        if world > 1:
            dist.all_reduce(sums)
        for i, (name, r) in enumerate(zip(names, rows)):
            c = getattr(self, name).view(-1)
            ops.center_ema(c, sums[i], r * world, self.center_momentum, out=c)

    @staticmethod
    def _snapshot(center: torch.Tensor) -> torch.Tensor:
        """256 KiB copy of a center: what this step's forward AND its (later) backward read, while update_center
        overwrites the live buffer in between (the reference rebinds self.center to a new tensor instead)."""
        return center.detach().view(-1).clone()


def mixup_targets(targets_mixup, ncrops: int, B: int, device) -> torch.Tensor:
    """The per-view soft targets of main_esvit.py:515-544 (timm's ``mixup_fn`` targets, or ``torch.eye(B)`` for views
    past ``num_mixup_views``) as one fp32 [ncrops, B, B] tensor.  Raises ValueError unless they are a list of ``ncrops``
    floating [B, B] tensors on ``device`` with finite, non-negative values.  The value check reads one flag on the host;
    it is skipped while a CUDA graph is being captured (engine.SelfDistillStep checks the values it copies in)."""
    if not isinstance(targets_mixup, (list, tuple)) or len(targets_mixup) != ncrops:
        raise ValueError(f"targets_mixup must be a list of {ncrops} [B, B] tensors (one per view)")
    for v, t in enumerate(targets_mixup):
        if not isinstance(t, torch.Tensor) or not t.is_floating_point() or tuple(t.shape) != (B, B):
            raise ValueError(f"targets_mixup[{v}] must be a floating [{B}, {B}] tensor, got "
                             f"{tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__}")
        if t.device != torch.device(device):
            raise ValueError(f"targets_mixup[{v}] is on {t.device}, the logits on {device}")
    T = torch.stack([t.detach().float() for t in targets_mixup])
    if not torch.cuda.is_current_stream_capturing():
        check_mixup_values(T)
    return T


def check_mixup_values(T: torch.Tensor) -> None:
    """ValueError unless every target is finite and non-negative (one host read when they are)."""
    if not bool((torch.isfinite(T) & (T >= 0)).all()):
        bad = "non-finite" if not bool(torch.isfinite(T).all()) else "negative"
        raise ValueError(f"targets_mixup has {bad} entries; mixup targets are finite, non-negative weights")


class DINOLoss(_CenteredLoss):
    def forward(self, student_output, teacher_output, epoch, targets_mixup=None):
        s, t = self._as_bf16(student_output), self._as_bf16(teacher_output).detach()
        B = t.shape[0] // 2
        temp = float(self.teacher_temp_schedule[epoch])
        n_terms = 2 * self.ncrops - 2
        if isinstance(targets_mixup, torch.Tensor) or targets_mixup:  # (a tensor is rejected by mixup_targets)
            loss = self._mixup_loss(s, t, targets_mixup, B, temp, n_terms)
            self.update_center(t)
            return loss
        trow, w = self._cls_tables(B, 1.0 / (n_terms * B), s.device)
        center = self._snapshot(self.center)
        lse_t = None if ops.ce_q_enabled(t.shape[-1]) else ops.row_lse(t, center, 1.0 / temp)
        loss = ops.DinoCEFn.apply(s, t, center, lse_t, trow, w, 1.0 / temp, 1.0 / self.student_temp,
                                  self._order(B, [(self.ncrops, 1)], s.device))
        self.update_center(t)
        return loss

    def _mixup_loss(self, s, t, targets_mixup, B, temp, n_terms):
        """main_esvit.py:638-641: every (iq, v != iq) term is -mean_j sum_b T_v[j, b] <q^iq_j, log_softmax(s_{v,b})>.
        Both global views fold into one mixed teacher row per student row (ops.mixup_q), paired with that row alone."""
        K = t.shape[-1]
        if not ops.ce_q_enabled(K):
            raise NotImplementedError("mixup targets run on the stored teacher probabilities only "
                                      f"(ESVIT_CE_Q=0, or out_dim {K} > esvit_row_softmax_q_max_k)")
        T = mixup_targets(targets_mixup, self.ncrops, B, s.device)
        _, q = ops.row_softmax_q(t, self.center.view(-1), 1.0 / temp)
        q_hat, w = ops.mixup_q(q, T, 1.0 / (n_terms * B))
        key = ("self", s.shape[0], str(s.device))
        if key not in self._tables:
            r = torch.arange(s.shape[0], dtype=torch.int32)
            self._tables[key] = (torch.stack([r, torch.full_like(r, -1)], 1).contiguous().to(s.device), None)
        return ops.DinoCEQFn.apply(s, q_hat, self._tables[key][0], w, 1.0 / self.student_temp)

    @torch.no_grad()
    def update_center(self, teacher_output):
        sums = ops.colsum(self._as_bf16(teacher_output)).view(1, -1)
        self._reduce_and_update(sums, [teacher_output.shape[0]], ["center"])


class DDINOLoss(_CenteredLoss):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.register_buffer("center_grid", torch.zeros(1, self.out_dim))
        self.last_indices = None  # int64 [2, ncrops, B, Tg] arg-max indices of the last call (parity hook)

    def _region_weights(self, B, Tg, Tl, n_terms, device):
        key = ("reg", B, Tg, Tl, n_terms, str(device))
        if key not in self._tables:
            w = torch.cat([torch.full((2 * B * Tg,), 0.5 / (n_terms * B * Tg)),
                           torch.full(((self.ncrops - 2) * B * Tl,), 0.5 / (n_terms * B * max(Tl, 1)))])
            self._tables[key] = (None, w.float().to(device))
        return self._tables[key][1]

    def forward(self, student_output, teacher_output, epoch, targets_mixup=None):
        """targets_mixup is accepted and ignored, as the reference's DDINOLoss does (main_esvit.py:683-750)."""
        s_cls_out, s_region_out, s_fea, s_npatch = student_output
        t_cls_out, t_region_out, t_fea, t_npatch = teacher_output
        s_cls, s_reg = self._as_bf16(s_cls_out), self._as_bf16(s_region_out)
        t_cls, t_reg = self._as_bf16(t_cls_out).detach(), self._as_bf16(t_region_out).detach()
        Tg = int(t_npatch[0])
        Tl = int(s_npatch[1]) if len(s_npatch) > 1 else 0
        B = t_reg.shape[0] // (2 * Tg)
        temp = float(self.teacher_temp_schedule[epoch])
        n_terms = 2 * self.ncrops - 2
        inv_t, inv_s = 1.0 / temp, 1.0 / self.student_temp
        center, center_grid = self._snapshot(self.center), self._snapshot(self.center_grid)

        # view-level term (0.5 * DINO)
        trow_c, w_c = self._cls_tables(B, 0.5 / (n_terms * B), s_cls.device)
        use_q = ops.ce_q_enabled(t_cls.shape[-1])  # teacher probabilities stored once per row (ops.DinoCEFn)
        lse_tc = None if use_q else ops.row_lse(t_cls, center, inv_t)
        loss_c = ops.DinoCEFn.apply(s_cls, t_cls, center, lse_tc, trow_c, w_c, inv_t, inv_s,
                                    self._order(B, [(self.ncrops, 1)], s_cls.device))

        # region-level term: cosine arg-max pairing then the same fused CE
        with torch.no_grad():
            idx, trow_r = ops.region_match(s_fea.detach().float(), t_fea.detach().float(), B, self.ncrops, Tg, Tl)
            self.last_indices = idx
        w_r = self._region_weights(B, Tg, Tl, n_terms, s_reg.device)
        lse_tr = None if use_q else ops.row_lse(t_reg, center_grid, inv_t)
        groups = [(2, Tg)] + ([(self.ncrops - 2, Tl)] if self.ncrops > 2 and Tl > 0 else [])
        loss_r = ops.DinoCEFn.apply(s_reg, t_reg, center_grid, lse_tr, trow_r, w_r, inv_t, inv_s,
                                    self._order(B, groups, s_reg.device))

        self.update_center(t_cls, t_reg)
        return loss_c + loss_r

    @torch.no_grad()
    def update_center(self, teacher_output, teacher_grid_output):
        K = self.out_dim
        sums = torch.empty(2, K, dtype=torch.float32, device=teacher_output.device)
        ops.colsum(self._as_bf16(teacher_output), out=sums[0])
        ops.colsum(self._as_bf16(teacher_grid_output), out=sums[1])
        self._reduce_and_update(sums, [teacher_output.shape[0], teacher_grid_output.shape[0]],
                                ["center", "center_grid"])
