"""Generate tests/golden/esvit_optim.pt by RUNNING THE REFERENCE'S OWN ``--optimizer sgd`` / ``--optimizer lars`` step.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, default oracle/_ref/):

    python -m oracle.make_golden_optim

utils.LARS, utils.get_params_groups, utils.clip_gradients and utils.cancel_gradients_last_layer are AST-extracted from
the reference's utils.py and exec'd verbatim (as oracle/reference_import.py does for clip_gradients), so nothing else of
the reference is imported.  The optimisers are built as main_esvit.py:410-415 builds them over get_params_groups, and
driven through the tail of train_one_epoch (main_esvit.py:507-510, 579-590) on the toy module below for STEPS: changing
lr / wd / EMA momentum, the last layer cancelled on the first step, gradients large enough on steps 0 and 2 that the
per-tensor clip fires.  The toy covers the LARS corner cases: a zero-valued 2-D weight (||p|| = 0: q = 1), a 2-D `.bias`
(group 1, wd 0, trust ratio by dimension) whose gradient is zero (||d|| = 0: q = 1), a 3-D token table, 1-D LayerNorm
and bias parameters, and a frozen weight-norm gain that only the EMA touches.  Stored per optimiser and step: the
student and teacher parameters and the momentum buffers.  Initial weights and gradients are regenerated from their
seeds (toy / step_grads); oracle/optim.py is asserted against every stored value while the file is written.
"""
from __future__ import annotations

import ast
import math
import os
import sys

import torch
import torch.nn as nn

from . import optim as O
from . import reference_import as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_optim.pt")

# lr, wd (group 0), EMA momentum, last layer cancelled, gradient scale
STEPS = ((0.1, 0.04, 0.996, True, 20.0), (0.2, 0.05, 0.997, False, 0.05), (0.05, 0.1, 0.99, False, 20.0))
CLIP = 3.0
KINDS = ("sgd", "lars")


class Toy(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(12, 20)
        self.norm = nn.LayerNorm(20)
        self.pos = nn.Parameter(torch.randn(1, 4, 20) * 0.02)
        self.z = nn.Linear(20, 6, bias=False)
        self.tok = nn.Module()
        self.tok.bias = nn.Parameter(torch.randn(3, 5))
        self.last_layer = nn.Linear(20, 24, bias=False)
        self.g = nn.Parameter(torch.ones(24, 1), requires_grad=False)


def toy(seed: int = 0) -> Toy:
    torch.manual_seed(seed)
    m = Toy()
    with torch.no_grad():
        m.z.weight.zero_()
        m.norm.weight.add_(torch.randn(20) * 0.1)
    return m


def step_grads(module: nn.Module, it: int) -> dict:
    """raw gradients of step `it` for every trainable parameter; tok.bias gets zeros"""
    g = torch.Generator().manual_seed(100 + it)
    scale = STEPS[it][4]
    out = {}
    for n, p in module.named_parameters():
        if p.requires_grad:
            out[n] = torch.zeros(p.shape) if n == "tok.bias" else torch.randn(p.shape, generator=g) * scale
    return out


def _reference():
    src = open(os.path.join(R.REF_ROOT, "utils.py")).read()
    env = {"torch": torch, "nn": nn, "math": math}
    for node in ast.parse(src).body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in (
                "LARS", "get_params_groups", "clip_gradients", "cancel_gradients_last_layer"):
            exec(compile(ast.Module([node], []), "utils.py", "exec"), env)
    return env


def _reference_run(U: dict, kind: str):
    student, teacher = toy(), toy()
    for p in teacher.parameters():
        p.requires_grad = False
    groups = U["get_params_groups"](student)
    opt = torch.optim.SGD(groups, lr=0, momentum=0.9) if kind == "sgd" else U["LARS"](groups)
    rec = []
    for it, (lr, wd, m, cancel, _) in enumerate(STEPS):
        for i, pg in enumerate(opt.param_groups):  # main_esvit.py:507-510
            pg["lr"] = lr
            if i == 0:
                pg["weight_decay"] = wd
        grads = step_grads(student, it)
        for n, p in student.named_parameters():
            p.grad = grads[n].clone() if n in grads else None
        U["clip_gradients"](student, CLIP)
        U["cancel_gradients_last_layer"](0 if cancel else 1, student, 1)
        opt.step()
        with torch.no_grad():  # main_esvit.py:587-590
            for param_q, param_k in zip(student.parameters(), teacher.parameters()):
                param_k.data.mul_(m).add_((1 - m) * param_q.detach().data)
        rec.append(dict(student={n: p.detach().clone() for n, p in student.named_parameters()},
                        teacher={n: p.detach().clone() for n, p in teacher.named_parameters()},
                        buffers={n: b.clone() for n, b in O.buffers(opt, student).items()}))
    return rec


def oracle_run(kind: str):
    """the same three steps through oracle/optim.py"""
    student, teacher = toy(), toy()
    for p in teacher.parameters():
        p.requires_grad = False
    opt = O.make_optimizer(kind, student)
    rec = []
    for it, (lr, wd, m, cancel, _) in enumerate(STEPS):
        O.train_step_tail(student, teacher, opt, step_grads(student, it), lr, wd, m, cancel, CLIP)
        rec.append(dict(student={n: p.detach().clone() for n, p in student.named_parameters()},
                        teacher={n: p.detach().clone() for n, p in teacher.named_parameters()},
                        buffers={n: b.clone() for n, b in O.buffers(opt, student).items()}))
    return rec


def make():
    U = _reference()
    runs = {}
    for kind in KINDS:
        ref = _reference_run(U, kind)
        orc = oracle_run(kind)
        for r, o in zip(ref, orc):
            assert r["buffers"].keys() == o["buffers"].keys(), kind
            for part in ("student", "teacher", "buffers"):
                for n, v in r[part].items():
                    assert torch.allclose(o[part][n], v, rtol=1e-6, atol=1e-7), (kind, part, n)
        runs[kind] = ref
    return dict(meta=dict(steps=STEPS, clip=CLIP,
                          generator="oracle/make_golden_optim.py (reference utils.LARS / torch.optim.SGD on CPU fp32, "
                                    "torch %s)" % torch.__version__), runs=runs)


if __name__ == "__main__":
    if not os.path.isfile(os.path.join(R.REF_ROOT, "utils.py")):
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    G = make()
    torch.save(G, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
