"""Generate tests/golden/esvit_mixup.pt by RUNNING THE UNMODIFIED REFERENCE DINOLoss with mixup targets.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout):

    python -m oracle.make_golden_mixup

DINOLoss is AST-extracted from main_esvit.py (oracle/reference_import.py), so timm is not needed; the targets are
timm 0.3.2's ``mixup_target`` restated in oracle/mixup.py (``batch`` mode: one lambda, ``elem`` mode: one per row, label
smoothing 0 / 0.1, ``torch.eye(B)`` past ``num_mixup_views`` as main_esvit.py:526-532 does) plus an arbitrary
non-negative matrix with a zero column.  Every case runs two epochs of a warm-up teacher-temperature schedule on one
loss module (the center carries over) and stores the loss, a sample of the student-logit gradient and the updated
center.  The logits are regenerated from their seed (``case_inputs``); the oracle is asserted against every stored value
while the file is written.
"""
from __future__ import annotations

import os
import sys

import torch

from . import golden as GD
from . import losses as L
from . import mixup as M
from . import reference_import as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_mixup.pt")

# warmup_teacher_temp, teacher_temp, warmup_teacher_temp_epochs, nepochs, student_temp, center_momentum
SCHEDULE = (0.04, 0.07, 3, 10, 0.1, 0.9)
EPOCHS = (0, 1)

# name -> (B, K, ncrops, targets kind, num_mixup_views, label smoothing, seed)
CASES = {
    "small_batch": (2, 64, 4, "batch", 4, 0.0, 1),
    "batch_eps": (8, 384, 6, "batch", 4, 0.1, 2),
    "elem": (8, 384, 6, "elem", 3, 0.0, 3),
    "elem_eps": (8, 384, 6, "elem", 5, 0.1, 4),
    "arbitrary_zero_column": (6, 256, 4, "arbitrary", 4, 0.0, 5),
}


def case_targets(B: int, ncrops: int, kind: str, n_mix: int, eps: float, seed: int):
    """Per-view targets: timm-shaped for the first n_mix views, eye(B) after (main_esvit.py:526-532)."""
    g = torch.Generator().manual_seed(1000 + seed)
    out = []
    for v in range(ncrops):
        if v >= n_mix:
            out.append(torch.eye(B))
        elif kind == "batch":
            out.append(M.timm_mixup_target(B, float(torch.rand((), generator=g)), eps))
        elif kind == "elem":
            out.append(M.timm_mixup_target(B, torch.rand(B, generator=g), eps))
        else:
            T = torch.rand(B, B, generator=g) * 2
            T[:, (v + 1) % B] = 0  # a student sample no teacher row is paired with: C = 0
            out.append(T)
    return out


def case_inputs(B: int, K: int, ncrops: int, seed: int, epoch: int):
    """bf16-representable fp32 logits (student [ncrops*B, K], teacher [2B, K]) of one case and epoch."""
    g = torch.Generator().manual_seed(seed * 100 + epoch)
    s = (torch.randn(ncrops * B, K, generator=g) * 2.0).to(torch.bfloat16).float()
    t = (torch.randn(2 * B, K, generator=g) * 1.5).to(torch.bfloat16).float()
    return s, t


def make_case(ns, B, K, ncrops, kind, n_mix, eps, seed):
    wt, tt, wte, ne, st, cm = SCHEDULE
    mod = ns.DINOLoss(K, ncrops, wt, tt, wte, ne, st, cm)
    sched = L.teacher_temp_schedule(wt, tt, wte, ne)
    targets = case_targets(B, ncrops, kind, n_mix, eps, seed)
    center = torch.zeros(1, K)
    rec = []
    for epoch in EPOCHS:
        s, t = case_inputs(B, K, ncrops, seed, epoch)
        s_ref = s.clone().requires_grad_(True)
        loss = mod(s_ref, t, epoch, targets)
        loss.backward()
        # the oracle must reproduce it
        s_o = s.clone().requires_grad_(True)
        lo = M.dino_loss_mixup(s_o, t, center, ncrops, float(sched[epoch]), targets, st)
        lo.backward()
        loss, lo = float(loss.detach()), float(lo.detach())
        assert abs(lo - loss) <= 2e-5 * max(1.0, abs(loss)), (lo, loss)
        assert torch.allclose(s_o.grad, s_ref.grad, rtol=1e-4, atol=1e-6 * float(s_ref.grad.abs().max())), kind
        center = L.center_update(center, t, cm)
        assert torch.allclose(center, mod.center, atol=1e-7), kind
        rec.append(dict(epoch=epoch, loss=loss, grad=GD.sample(s_ref.grad, seed=seed), center=mod.center.clone()))
    return dict(B=B, K=K, ncrops=ncrops, kind=kind, num_mixup_views=n_mix, smoothing=eps, seed=seed,
                targets=torch.stack(targets), steps=rec)


def make():
    R.ensure_process_group()
    ns = R.load()
    cases = {name: make_case(ns, *c) for name, c in CASES.items()}
    return dict(meta=dict(schedule=SCHEDULE, epochs=EPOCHS,
                          generator="oracle/make_golden_mixup.py (reference DINOLoss on CPU fp32, torch %s)"
                          % torch.__version__), cases=cases)


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    G = make()
    torch.save(G, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB;",
          {k: [r["loss"] for r in c["steps"]] for k, c in G["cases"].items()})
