"""Functional fp32 oracle of the reference's ``--optimizer sgd`` / ``--optimizer lars`` training-step tail.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into the reference's main_esvit.py and utils.py.

Per step (train_one_epoch, main_esvit.py:507-590): lr to both param groups and the scheduled wd to group 0, then
utils.clip_gradients (per tensor), cancel_gradients_last_layer (grads -> None), optimizer.step(), the teacher EMA over
zip(student.parameters(), teacher.parameters()).  SGD is torch.optim.SGD(params_groups, lr=0, momentum=0.9) itself;
LARS is restated below.
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from . import losses as L


class LARS(torch.optim.Optimizer):
    """utils.LARS (utils.py:519-557) with its defaults, restated.  A parameter with a gradient steps as

        d = g + wd p,  d *= eta ||p|| / ||d||      only when p.ndim != 1 (1 when either norm is 0)
        mu = momentum mu + d                       (mu starts at zeros)
        p -= lr mu

    The trust ratio goes by dimension, not by param group; 1-D parameters get neither decay nor trust ratio.  The
    filters are accepted for the state_dict layout and, as in the reference, not used."""

    def __init__(self, params, lr=0, weight_decay=0, momentum=0.9, eta=0.001, weight_decay_filter=None,
                 lars_adaptation_filter=None):
        super().__init__(params, dict(lr=lr, weight_decay=weight_decay, momentum=momentum, eta=eta,
                                      weight_decay_filter=weight_decay_filter,
                                      lars_adaptation_filter=lars_adaptation_filter))

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                d = p.grad
                if p.ndim != 1:
                    d = d.add(p, alpha=group["weight_decay"])
                    pn, dn = torch.norm(p), torch.norm(d)
                    if pn > 0 and dn > 0:  # the trust ratio; 1 (d unchanged) otherwise
                        d = d.mul(group["eta"] * pn / dn)
                st = self.state[p]
                if "mu" not in st:
                    st["mu"] = torch.zeros_like(p)
                st["mu"].mul_(group["momentum"]).add_(d)
                p.add_(st["mu"], alpha=-group["lr"])


def params_groups(module: nn.Module) -> List[dict]:
    """utils.get_params_groups (utils.py:672-683): group 0 = trainable, not `.bias`, not 1-D; group 1 = the rest of the
    trainable parameters, weight_decay 0."""
    reg, noreg = [], []
    for name, p in module.named_parameters():
        if not p.requires_grad:
            continue
        (noreg if name.endswith(".bias") or p.dim() == 1 else reg).append(p)
    return [{"params": reg}, {"params": noreg, "weight_decay": 0.0}]


def make_optimizer(kind: str, module: nn.Module) -> torch.optim.Optimizer:
    """main_esvit.py:412-415 for kind = sgd | lars"""
    if kind == "sgd":
        return torch.optim.SGD(params_groups(module), lr=0, momentum=0.9)
    if kind == "lars":
        return LARS(params_groups(module))
    raise ValueError(kind)


def train_step_tail(student: nn.Module, teacher: nn.Module, opt: torch.optim.Optimizer, grads: dict, lr: float,
                    wd: float, m: float, cancel_last_layer: bool, clip: float = 3.0) -> List[float]:
    """Everything after backward (main_esvit.py:507-510, 579-590): `grads` maps trainable parameter names to their raw
    gradients (copied in).  Returns the pre-clip norms."""
    for i, g in enumerate(opt.param_groups):
        g["lr"] = lr
        if i == 0:
            g["weight_decay"] = wd
    for n, p in student.named_parameters():
        p.grad = grads[n].clone().to(p.device) if n in grads else None
    norms = L.clip_gradients([p.grad for p in student.parameters()], clip)
    if cancel_last_layer:
        for n, p in student.named_parameters():
            if "last_layer" in n:
                p.grad = None
    opt.step()
    L.ema_update(list(teacher.parameters()), list(student.parameters()), m)
    return norms


def buffers(opt: torch.optim.Optimizer, module: nn.Module) -> dict:
    """name -> momentum buffer (SGD's momentum_buffer / LARS's mu) of every parameter that has one"""
    out = {}
    for n, p in module.named_parameters():
        st = opt.state.get(p, {})
        b = st.get("momentum_buffer", st.get("mu"))
        if b is not None:
            out[n] = b
    return out
