"""Linear probe of frozen features (eval_linear.py) on the esvit_b200 kernels.

  * ``LinearClassifier``: eval_linear.LinearClassifier (:307-320) - same module, initialisation and state_dict keys -
    whose forward runs the fp32-output wgmma GEMM (esvit_gemm_f32) on bf16 operands;
  * ``ProbeSGD``: the script's ``torch.optim.SGD(params, lr, momentum=0.9, weight_decay=0)`` (:188-193) as a torch
    Optimizer that ``CosineAnnealingLR`` drives and ``restart_from_checkpoint`` loads, stepping through the fused SGD
    sweep (esvit_sgd_ema_multi: no teacher, no clip, no decay) with the scheduler's lr staged to the device;
  * ``LinearProbeStep``: the body of train() (:244-275): features (no grad) -> logits -> mean cross-entropy -> weight /
    bias gradients -> AVG all-reduce under a process group -> SGD, eager or as one CUDA graph, without host
    synchronisation;
  * ``evaluate``: validate_network() (:278-304) with one host synchronisation at the end.

Classes are padded to a multiple of 8 (the GEMMs' N): the bf16 weight shadow is the leading rows of a zero-filled
[C_pad, D] buffer the sweep keeps current, and the padded classes never enter a loss, a rank or a gradient
(csrc/probe.cu).  Rows are padded to a multiple of 8 with label -1.  Hit counts and losses accumulate on the device in a
``ProbeMeter`` that the caller reads once per epoch.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from . import _lib, ops, shadow
from .augment import MultiCropBatch
from .optim import FusedSGDEMA
from .ops import _p, _stream

Tensor = torch.Tensor
BF16, F32 = torch.bfloat16, torch.float32
MAX_CLASSES = 12288  # one logit row in shared memory (csrc/probe.cu)


def _pad8(n: int) -> int:
    return -(-int(n) // 8) * 8


def _multi() -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


def _padded_weight(weight: Tensor) -> Tensor:
    """bf16 [C_pad, D] whose first C rows are the registered shadow of `weight` (re-cast when the weight was modified
    outside the fused sweep) and whose padding rows are zero"""
    C, D = weight.shape
    s = shadow.lookup(weight)
    if s is None:
        buf = torch.zeros(_pad8(C), D, dtype=BF16, device=weight.device)
        s = shadow.register(weight, out=buf[:C])
    base = s._base
    if base is None or tuple(base.shape) != (_pad8(C), D) or s.device != weight.device:
        raise RuntimeError("the classifier weight already has an unpadded bf16 shadow on another path")
    return base


def check_labels(target, batch: int, num_labels: int) -> Tensor:
    """host int64 [batch] labels, every one in [0, num_labels): checked before the copy to the device (the reference's
    CUDA cross-entropy would assert on the device)"""
    if not isinstance(target, Tensor) or target.is_cuda or target.dtype.is_floating_point or target.dtype == torch.bool:
        raise ValueError("labels must be a host integer tensor")
    if target.numel() != batch:
        raise ValueError(f"{target.numel()} labels for a batch of {batch}")
    t = target.reshape(-1).to(torch.int64)
    if batch and (int(t.min()) < 0 or int(t.max()) >= num_labels):
        raise ValueError(f"labels must lie in [0, {num_labels})")
    return t


def _check_features(x, dim: int) -> Tensor:
    if not isinstance(x, Tensor) or not x.is_cuda or x.dtype != F32:
        raise ValueError("features must be a CUDA float32 tensor")
    x = x.reshape(x.shape[0], -1) if x.dim() > 2 else x
    if x.dim() != 2 or x.shape[0] == 0:
        raise ValueError(f"features must be a non-empty [batch, dim] matrix, got {tuple(x.shape)}")
    if x.shape[1] != dim:
        raise ValueError(f"feature dimension {x.shape[1]} differs from the classifier's {dim}")
    return x.contiguous()


class ProbeMeter:
    """Device accumulators of the probe: the sum of batch mean losses (fp64) and {batches, images, top-1 hits, top-5
    hits} (int64), written by esvit_probe_ce in a fixed order.  read() is the one host synchronisation."""

    def __init__(self, device):
        self.acc = torch.zeros(1, dtype=torch.float64, device=device)
        self.counts = torch.zeros(4, dtype=torch.int64, device=device)

    def reset(self) -> None:
        self.acc.zero_()
        self.counts.zero_()

    def read(self) -> dict:
        """{"loss": mean over batches of the batch mean loss (MetricLogger.update(loss=...) with n = 1), "acc1" /
        "acc5": hits / images in percent, "batches", "images"}, summed over the process group like
        MetricLogger.synchronize_between_processes"""
        acc, counts = self.acc, self.counts
        if _multi():
            acc, counts = acc.clone(), counts.clone()
            dist.all_reduce(acc)
            dist.all_reduce(counts)
        loss = float(acc.cpu()[0])
        nb, ni, h1, h5 = counts.tolist()
        return {"loss": loss / max(nb, 1), "acc1": h1 * 100.0 / max(ni, 1), "acc5": h5 * 100.0 / max(ni, 1),
                "batches": nb, "images": ni}


class _Workspace:
    """Buffers of one padded batch shape: bf16 features, the padded bias, fp32 logits, labels (-1 = padding row), the
    cross-entropy scratch and, for training, the bf16 logit gradient and one flat fp32 gradient [dW | db] (one
    all-reduce)."""

    def __init__(self, rows: int, C: int, D: int, device, train: bool):
        R, Cp = _pad8(rows), _pad8(C)
        self.R, self.C, self.Cp, self.D = R, C, Cp, D
        self.xb = torch.empty(R, D, dtype=BF16, device=device)
        self.norm = torch.empty(R, dtype=F32, device=device)  # esvit_knn_prep's row norms: unused here
        self.max_norm = torch.zeros(1, dtype=F32, device=device)
        self.bias = torch.zeros(Cp, dtype=F32, device=device)
        self.logits = torch.empty(R, Cp, dtype=F32, device=device)
        self.labels = torch.full((R,), -1, dtype=torch.int64, device=device)
        self.row_loss = torch.empty(R, dtype=F32, device=device)
        self.row_rank = torch.empty(R, dtype=torch.int32, device=device)
        self.loss = torch.zeros(1, dtype=F32, device=device)
        self.dlogits = self.grad = self.dw = self.db = None
        if train:
            self.dlogits = torch.empty(R, Cp, dtype=BF16, device=device)
            self.grad = torch.zeros(Cp * D + Cp, dtype=F32, device=device)
            self.dw = self.grad[:Cp * D].view(Cp, D)
            self.db = self.grad[Cp * D:]

    def set_labels(self, labels: Tensor) -> None:
        """host labels of the first rows; every other row becomes padding"""
        B = labels.numel()
        self.labels[:B].copy_(labels, non_blocking=True)
        if B < self.R:
            self.labels[B:].fill_(-1)

    def logits_of(self, linear: nn.Linear, x: Tensor) -> None:
        """logits fp32 [R, Cp] = bf16(x) . bf16(W)^T + bias for the rows of x (the rest are zero rows)"""
        B, D = x.shape
        _lib.call("esvit_knn_prep", _p(x), _p(self.xb), _p(self.norm), _p(self.max_norm), B, self.R, D, _stream())
        self.bias[:self.C].copy_(linear.bias.detach())
        w16 = _padded_weight(linear.weight)
        _lib.call("esvit_gemm_f32", _p(self.xb), _p(w16), _p(self.bias), _p(self.logits), self.R, self.Cp, D, 0,
                  _stream())

    def cross_entropy(self, meter: Optional[ProbeMeter], train: bool) -> None:
        _lib.call("esvit_probe_ce", _p(self.logits), self.Cp, _p(self.labels), self.R, self.C,
                  _p(self.dlogits) if train else None, _p(self.row_loss), _p(self.row_rank), _p(self.loss),
                  _p(meter.acc) if meter else None, _p(meter.counts) if meter else None, _stream())

    def gradients(self) -> None:
        """dW = dlogits^T . x (split-K, fixed-order fold), db = column sums of dlogits; padded rows and classes are 0"""
        ops.gemm_wgrad(self.dlogits, self.xb, out=self.dw)
        ops.colsum(self.dlogits, out=self.db)


def _linear_of(classifier: nn.Module) -> nn.Linear:
    m = classifier.module if isinstance(classifier, nn.parallel.DistributedDataParallel) else classifier
    if not isinstance(getattr(m, "linear", None), nn.Linear):
        raise ValueError("expected a LinearClassifier (a module with a `linear` nn.Linear)")
    return m.linear


class LinearClassifier(nn.Module):
    """Linear layer to train on top of frozen features (eval_linear.LinearClassifier).  forward() -> fp32 logits from
    the bf16 GEMM; it builds no autograd graph: LinearProbeStep trains it."""

    def __init__(self, dim, num_labels=1000):
        super().__init__()
        self.linear = nn.Linear(dim, num_labels)
        self.linear.weight.data.normal_(mean=0.0, std=0.01)
        self.linear.bias.data.zero_()
        self._ws = {}

    def forward(self, x):
        x = _check_features(x.view(x.size(0), -1), self.linear.in_features)
        C = self.linear.out_features
        if C > MAX_CLASSES or self.linear.in_features % 8:
            raise ValueError(f"num_labels <= {MAX_CLASSES} and dim % 8 == 0 required")
        key = (x.device, _pad8(x.shape[0]))
        ws = self._ws.get(key)
        if ws is None:
            ws = self._ws[key] = _Workspace(x.shape[0], C, x.shape[1], x.device, train=False)
        with torch.no_grad():
            ws.logits_of(self.linear, x)
            return ws.logits[:x.shape[0], :C].clone()


class ProbeSGD(torch.optim.Optimizer):
    """``torch.optim.SGD(linear_classifier.parameters(), lr, momentum=0.9, weight_decay=0)`` on the fused SGD sweep.
    One param group holding (weight, bias); its ``lr`` is what CosineAnnealingLR writes, staged to the device (the
    sweep's pinned ring) before each step without re-capturing a graph.  state_dict() / load_state_dict() use
    torch.optim.SGD's layout, so checkpoints move between the two in both directions."""

    def __init__(self, params, lr, momentum: float = 0.9, weight_decay: float = 0):
        params = list(params)
        if float(weight_decay) != 0.0:
            raise ValueError("ProbeSGD has no weight decay (eval_linear.py uses weight_decay=0)")
        if (len(params) != 2 or params[0].dim() != 2 or params[1].dim() != 1
                or params[1].shape[0] != params[0].shape[0]):
            raise ValueError("ProbeSGD takes a LinearClassifier's parameters: weight [C, D] and bias [C]")
        defaults = dict(lr=lr, momentum=momentum, dampening=0, weight_decay=0, nesterov=False, maximize=False,
                        foreach=None, differentiable=False, fused=None)
        super().__init__(params, defaults)
        weight, bias = params
        _padded_weight(weight)
        named = nn.Module()  # the sweep's parameter names: linear.weight (bf16 shadow kept by the sweep), linear.bias
        named.linear = nn.Module()
        named.linear.weight, named.linear.bias = weight, bias
        self.sweep = FusedSGDEMA(named, None, momentum=momentum, clip_grad=0.0)
        self._staged = None

    def stage(self) -> None:
        """copy the group's lr to the device when it changed (an async copy from the sweep's pinned ring)"""
        lr = float(self.param_groups[0]["lr"])
        if lr != self._staged:
            self.sweep.set_hyper(lr, 0.0, 0.0)
            self._staged = lr

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise ValueError("ProbeSGD.step takes no closure")
        if not torch.cuda.is_current_stream_capturing():
            self.stage()
        self.sweep.step()

    def state_dict(self):
        steps = self.sweep.state[:, 0].cpu()
        state = {i: {"momentum_buffer": self.sweep.momentum_buffer[i].detach().clone()}
                 for i in range(2) if float(steps[i]) > 0}
        group = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        group["params"] = [0, 1]
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, state_dict, **kwargs) -> None:
        groups = state_dict["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != 2:
            raise ValueError("expected torch.optim.SGD's single group over (weight, bias)")
        g = groups[0]
        if float(g.get("weight_decay", 0)) != 0 or g.get("nesterov", False) or float(g.get("dampening", 0)) != 0:
            raise ValueError("the checkpoint's SGD uses weight decay, dampening or Nesterov momentum")
        sw = self.sweep
        for b in sw.momentum_buffer:
            b.zero_()
        sw.state[:, 0] = 0.0
        for k, pid in enumerate(g["params"]):
            st = state_dict["state"].get(pid)
            buf = st.get("momentum_buffer") if st else None
            if buf is not None:
                sw.momentum_buffer[k].copy_(buf)
                sw.state[k, 0] = 1.0
        self.param_groups[0].update({k: v for k, v in g.items() if k != "params"})
        sw.momentum = float(self.param_groups[0]["momentum"])
        sw._hyper_host[2] = sw.momentum
        self._staged = None  # restage lr and momentum before the next step
        self.stage()


class LinearProbeStep:
    """One iteration of eval_linear.train(): features of the frozen backbone (forward_return_n_last_blocks under
    no_grad), logits, mean cross-entropy, weight and bias gradients, their AVG all-reduce when a process group of more
    than one rank is initialised (DDP's semantics), and the SGD step.  No host synchronisation.

    ``step(inp, target)``: inp is a CUDA fp32 image batch or a collated MultiCropBatch (run through ``augment``, an
    EvalAugment); target the host integer labels.  Returns the batch's mean loss as a device scalar.  Losses and hits
    accumulate in ``meter``; ``epoch_stats()`` reads and resets it once per epoch.  With use_cuda_graph=True the step
    is captured at the first batch size after three eager warm-up calls; a smaller (ragged last) batch runs in the same
    graph with its rows padded (label -1, zero images)."""

    def __init__(self, model: nn.Module, classifier: nn.Module, optimizer: ProbeSGD, n: int, avgpool: bool, depths,
                 use_cuda_graph: bool = False, augment=None):
        if not isinstance(optimizer, ProbeSGD):
            raise ValueError("LinearProbeStep steps a ProbeSGD")
        self.model, self.linear, self.opt = model, _linear_of(classifier), optimizer
        self.n, self.avgpool, self.depths = n, avgpool, list(depths)
        self.use_cuda_graph, self.augment = use_cuda_graph, augment
        C, D = self.linear.out_features, self.linear.in_features
        if C > MAX_CLASSES or D % 8:
            raise ValueError(f"num_labels <= {MAX_CLASSES} and a feature dimension divisible by 8 required, got "
                             f"{C}, {D}")
        self.meter = ProbeMeter(self.linear.weight.device)
        self.last_features = None
        self._ws = {}
        self._static = None  # graph mode: (images [cap, ...], workspace)
        self._graph = None
        self._warm = 0

    def _workspace(self, rows: int) -> _Workspace:
        key = _pad8(rows)
        ws = self._ws.get(key)
        if ws is None:
            lin = self.linear
            ws = self._ws[key] = _Workspace(rows, lin.out_features, lin.in_features, lin.weight.device, train=True)
        return ws

    def _body(self, images: Tensor, ws: _Workspace) -> None:
        with torch.no_grad():
            feats = self.model.forward_return_n_last_blocks(images, self.n, self.avgpool, self.depths)
        feats = _check_features(feats, ws.D)
        self.last_features = feats
        ws.logits_of(self.linear, feats)
        ws.cross_entropy(self.meter, train=True)
        ws.gradients()
        if _multi():
            dist.all_reduce(ws.grad, op=dist.ReduceOp.AVG)
        w, b = self.linear.weight, self.linear.bias
        w.grad, b.grad = ws.dw[:ws.C], ws.db[:ws.C]
        self.opt.step()

    def _images(self, inp, out: Optional[Tensor] = None) -> Tensor:
        if isinstance(inp, MultiCropBatch):
            if self.augment is None:
                raise ValueError("a MultiCropBatch input needs augment=EvalAugment(...)")
            return self.augment(inp, out=out)
        if not isinstance(inp, Tensor) or not inp.is_cuda or inp.dtype != F32 or inp.dim() != 4:
            raise ValueError("images must be a CUDA float32 [B, 3, H, W] tensor")
        if out is not None:
            out.copy_(inp, non_blocking=True)
            return out
        return inp

    def __call__(self, inp, target) -> Tensor:
        return self.step(inp, target)

    def step(self, inp, target) -> Tensor:
        B = int(inp.index.shape[0] if isinstance(inp, MultiCropBatch) else inp.shape[0])
        labels = check_labels(target, B, self.linear.out_features)
        self.opt.stage()
        if not self.use_cuda_graph:
            images = self._images(inp)
            ws = self._workspace(B)
            ws.set_labels(labels)
            self._body(images, ws)
            return ws.loss[0].clone()
        return self._graphed(inp, labels, B)

    def _graphed(self, inp, labels: Tensor, B: int) -> Tensor:
        """Replay path: the graph reads private static images and labels sized by the first batch"""
        if self._static is None:
            images = self._images(inp)
            self._static = (torch.empty_like(images), self._workspace(B))
        static, ws = self._static
        if B > static.shape[0]:
            raise ValueError(f"batch of {B} exceeds the captured batch of {static.shape[0]}")
        self._images(inp, out=static[:B])
        if B < static.shape[0]:
            static[B:].zero_()
        ws.set_labels(labels)
        if self._warm < 3:  # eager warm-up (allocator, workspaces, cached tables) before the capture
            self._warm += 1
            self._body(static, ws)
            return ws.loss[0].clone()
        if self._graph is None:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body(static, ws)
            self._graph = g
        self._graph.replay()
        return ws.loss[0].clone()

    def epoch_stats(self) -> dict:
        """train()'s return value for the epoch so far - {"loss": mean batch loss, "lr": the group's lr} - plus the
        training hits; resets the meter (one host synchronisation)"""
        s = self.meter.read()
        self.meter.reset()
        s["lr"] = float(self.opt.param_groups[0]["lr"])
        return s


@torch.no_grad()
def evaluate(val_loader, model: nn.Module, linear_classifier: nn.Module, n: int, avgpool: bool, depths,
             augment=None) -> dict:
    """validate_network() (eval_linear.py:278-304) -> {"loss", "acc1", "acc5"}: the mean over batches of each batch's
    mean loss, and top-1 / top-5 hits over images in percent, with one host synchronisation at the end."""
    lin = _linear_of(linear_classifier)
    C, D = lin.out_features, lin.in_features
    if C > MAX_CLASSES or D % 8:
        raise ValueError(f"num_labels <= {MAX_CLASSES} and a feature dimension divisible by 8 required, got {C}, {D}")
    meter = ProbeMeter(lin.weight.device)
    spaces = {}
    for inp, target in val_loader:
        if isinstance(inp, MultiCropBatch):
            if augment is None:
                raise ValueError("a MultiCropBatch input needs augment=EvalAugment(...)")
            images = augment(inp)
        else:
            images = inp.cuda(non_blocking=True)
        labels = check_labels(target, images.shape[0], C)
        feats = _check_features(model.forward_return_n_last_blocks(images, n, avgpool, depths), D)
        ws = spaces.get(_pad8(feats.shape[0]))
        if ws is None:
            ws = spaces[_pad8(feats.shape[0])] = _Workspace(feats.shape[0], C, D, feats.device, train=False)
        ws.set_labels(labels)
        ws.logits_of(lin, feats)
        ws.cross_entropy(meter, train=False)
    s = meter.read()
    return {"loss": s["loss"], "acc1": s["acc1"], "acc5": s["acc5"]}
