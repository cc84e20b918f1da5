"""Functional fp32 oracle of the linear probe (eval_linear.py).

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into the reference repository.

  * ``init_classifier``: LinearClassifier (eval_linear.py:307-320) under a seed: nn.Linear's own init, then
    normal_(0, 0.01) on the weight and a zero bias, consuming the global RNG as the reference does;
  * ``train_step``: one iteration of train() (:244-275): logits, mean cross-entropy, its weight / bias gradients and
    torch.optim.SGD(momentum, dampening 0, no weight decay, no Nesterov);
  * ``hits`` / ``validate``: utils.accuracy (utils.py:468-475) with the top-k order made explicit - the target's rank is
    the number of logits ahead of it by (value desc, index asc) - and validate_network's averaging (:278-304);
  * ``cosine_lrs``: CosineAnnealingLR(optimizer, epochs, eta_min=0)'s recursive update, one value per epoch;
  * ``probe_features``: the seeded synthetic features and labels of the fixture and tests.
"""
from __future__ import annotations

import ast
import math
import os
import types

import torch
import torch.nn as nn

from . import reference_import as R

Tensor = torch.Tensor


def init_classifier(dim: int, num_labels: int, seed: int):
    """(weight fp32 [C, D], bias fp32 [C]) of LinearClassifier(dim, num_labels) built right after manual_seed(seed)"""
    torch.manual_seed(seed)
    lin = nn.Linear(dim, num_labels)
    lin.weight.data.normal_(mean=0.0, std=0.01)
    lin.bias.data.zero_()
    return lin.weight.detach().clone(), lin.bias.detach().clone()


def forward(w: Tensor, b: Tensor, x: Tensor) -> Tensor:
    return x @ w.t() + b


def cross_entropy(logits: Tensor, target: Tensor):
    """(mean loss, dlogits = (softmax - onehot) / B) in fp32"""
    B = logits.shape[0]
    lse = torch.logsumexp(logits, dim=1)
    loss = (lse - logits.gather(1, target.view(-1, 1)).view(-1)).mean()
    d = torch.softmax(logits, dim=1)
    d[torch.arange(B), target] -= 1.0
    return loss, d / B


def train_step(w, b, buf_w, buf_b, x, target, lr: float, momentum: float = 0.9):
    """one train() iteration on fp32 tensors -> (loss, w, b, buf_w, buf_b); buf_* None before the first step"""
    loss, d = cross_entropy(forward(w, b, x), target)
    gw, gb = d.t() @ x, d.sum(0)
    buf_w = gw.clone() if buf_w is None else buf_w * momentum + gw
    buf_b = gb.clone() if buf_b is None else buf_b * momentum + gb
    return float(loss), w - lr * buf_w, b - lr * buf_b, buf_w, buf_b


def ranks(logits: Tensor, target: Tensor) -> Tensor:
    """number of logits ahead of the target's by (value desc, index asc)"""
    lt = logits.gather(1, target.view(-1, 1))
    idx = torch.arange(logits.shape[1]).view(1, -1)
    ahead = (logits > lt) | ((logits == lt) & (idx < target.view(-1, 1)))
    return ahead.sum(1)


def hits(logits: Tensor, target: Tensor):
    r = ranks(logits, target)
    return int((r < 1).sum()), int((r < 5).sum())


def validate(w, b, x, target, batch: int) -> dict:
    """validate_network: loss = mean over batches of the batch mean loss; acc1 / acc5 = hits / images in percent"""
    losses, h1, h5 = [], 0, 0
    for r0 in range(0, x.shape[0], batch):
        lg = forward(w, b, x[r0:r0 + batch])
        t = target[r0:r0 + batch]
        losses.append(float(cross_entropy(lg, t)[0]))
        a, c = hits(lg, t)
        h1, h5 = h1 + a, h5 + c
    n = x.shape[0]
    return {"loss": sum(losses) / len(losses), "acc1": h1 * 100.0 / n, "acc5": h5 * 100.0 / n}


def cosine_lrs(base_lr: float, epochs: int):
    """the lr of every epoch under CosineAnnealingLR(T_max=epochs, eta_min=0) stepped once per epoch"""
    lrs, lr = [base_lr], base_lr
    for e in range(1, epochs):
        lr = (1 + math.cos(math.pi * e / epochs)) / (1 + math.cos(math.pi * (e - 1) / epochs)) * (lr - 0) + 0
        lrs.append(lr)
    return lrs


def logit_bound(w: Tensor, x: Tensor) -> Tensor:
    """[B, C] bound on |bf16-operand logit - fp32 logit| (DESIGN.md §4.20): (2u + u^2 + D 2^-23) sum_i |x_i| |w_ji|"""
    u = 2.0 ** -8
    return (2 * u + u * u + x.shape[1] * 2.0 ** -23) * (x.abs() @ w.abs().t())


def decided(logits: Tensor, target: Tensor, delta: Tensor, ks=(1, 5)) -> Tensor:
    """rows whose top-k outcomes hold for any logits within delta: at least k classes surely ahead of the target, or
    fewer than k possibly ahead"""
    lt = logits.gather(1, target.view(-1, 1))
    dt = delta.gather(1, target.view(-1, 1))
    gap = logits - lt
    sure = (gap > delta + dt).sum(1)
    maybe = (gap >= -(delta + dt)).sum(1) - 1  # the target itself has gap 0
    ok = torch.ones(logits.shape[0], dtype=torch.bool)
    for k in ks:
        ok &= (sure >= k) | (maybe < k)
    return ok


def probe_features(centre_seed: int, seed: int, n: int, dim: int, classes_used: int, noise: float = 1.0):
    """(features fp32 [n, dim], labels int64 [n] in [0, classes_used)): Gaussian samples around classes_used seeded
    Gaussian centres (centre_seed), drawn with `seed`"""
    centres = torch.randn(classes_used, dim, generator=torch.Generator().manual_seed(centre_seed))
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, classes_used, (n,), generator=g)
    return centres[y] + noise * torch.randn(n, dim, generator=g), y


def reference_probe():
    """the UNMODIFIED LinearClassifier, train, validate_network (eval_linear.py) and utils.accuracy / MetricLogger /
    SmoothedValue (utils.py), AST-extracted: the scripts import torchvision datasets and the model zoo"""
    env = {"torch": torch, "nn": nn}
    import collections
    import datetime
    import time
    import torch.distributed as dist
    env.update(defaultdict=collections.defaultdict, deque=collections.deque, datetime=datetime, time=time, dist=dist)
    for fname, names in (("utils.py", ("accuracy", "MetricLogger", "SmoothedValue", "is_dist_avail_and_initialized")),
                         ("eval_linear.py", ("LinearClassifier", "train", "validate_network"))):
        path = os.path.join(R.REF_ROOT, fname)
        tree = ast.parse(open(path).read())
        for node in tree.body:
            if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
                exec(compile(ast.Module([node], []), path, "exec"), env)
    env["utils"] = types.SimpleNamespace(**{k: env[k] for k in ("accuracy", "MetricLogger", "SmoothedValue")})
    return env
