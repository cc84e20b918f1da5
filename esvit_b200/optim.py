"""Fused optimiser pass for the self-distillation step: per-tensor gradient clip (utils.clip_gradients) + the
optimiser update (the reference's two param groups, utils.get_params_groups) + teacher EMA (main_esvit.py:587-590) as
ONE multi-tensor sweep, with every step-varying scalar in device memory so that the whole training step can be captured
in a CUDA graph and replayed with fresh lr / wd / momentum.  One class per ``--optimizer`` of main_esvit.py:
FusedAdamWEMA (adamw: esvit_adamw_ema_multi) and FusedSGDEMA (sgd / lars: esvit_sgd_ema_multi).

Semantics preserved from the reference loop:
  * clipping is PER PARAMETER TENSOR (coef = clip / (norm + 1e-6), applied when < 1);
  * biases and 1-D parameters are not weight-decayed;
  * parameters whose gradient the reference sets to None (cancel_gradients_last_layer while epoch <
    freeze_last_layer) are skipped entirely by the optimiser (no decay, no moments / buffer, no step count) - flag bit 1;
  * frozen parameters (requires_grad=False, e.g. last_layer.weight_g) are never stepped but ARE part of the EMA,
    which runs over zip(student.parameters(), teacher.parameters());
  * the EMA is bit-exact with param_k.mul_(m).add_((1 - m) * param_q).
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import _lib, ops, shadow

F32 = torch.float32


def _wants_shadow(nm: str, p: torch.Tensor) -> bool:
    """bf16 shadows of everything the GEMMs consume (Linear weights and biases); written by the sweep itself"""
    if "relative_position_bias_table" in nm or "patch_embed.proj" in nm or "last_layer" in nm or "norm" in nm:
        return False
    return nm.endswith(".weight") and p.dim() == 2 or nm.endswith(".bias")


class _FusedSweep:
    """Plumbing shared by the fused sweeps: parameter names and flags, the device hyper vector and its pinned staging
    ring, the bf16 shadow registration, the pointer arrays and the per-step gradient checks.  A subclass sets the flags
    (set_flags), fills its own hyper slots and launches its kernels in step()."""

    _EMA_SLOTS = (5, 6)  # where ema_m and 1 - ema_m sit in the subclass's hyper layout

    def __init__(self, student: nn.Module, teacher: Optional[nn.Module]):
        named = list(student.named_parameters())
        self.names = [n for n, _ in named]
        self.params: List[torch.Tensor] = [p for _, p in named]
        tparams = [p for _, p in teacher.named_parameters()] if teacher is not None else None
        if tparams is not None:
            assert len(tparams) == len(self.params)
        dev = self.params[0].device
        for p in self.params:
            if not (p.is_cuda and p.dtype == F32 and p.is_contiguous()):
                raise RuntimeError(f"{type(self).__name__} needs fp32 contiguous CUDA parameters (no CPU fallback)")
        self.teacher_params = tparams
        n = len(self.params)
        self.frozen = [not p.requires_grad for p in self.params]
        self._decay = [0 if (nm.endswith(".bias") or p.dim() == 1) else 1 for nm, p in named]  # utils.py:672-683
        self._last_layer = torch.tensor([1.0 if "last_layer" in nm else 0.0 for nm in self.names])
        self.state = torch.zeros(n, 2, dtype=F32, device=dev)
        self._flags_host = torch.empty(n, dtype=F32).pin_memory()
        self.hyper = torch.zeros(8, dtype=F32, device=dev)
        # ring of pinned staging buffers: the H2D copy of step N reads its buffer at EXECUTION time, while the host may
        # already be preparing step N+k (no sync inside the step) - a single buffer would be overwritten in flight
        self._hyper_ring = [torch.zeros(8, dtype=F32).pin_memory() for _ in range(8)]
        self._hyper_events = [None] * 8
        self._hyper_slot = 0
        self._hyper_host = torch.zeros(8, dtype=F32)
        self.shadow_p = [shadow.register(p) if _wants_shadow(nm, p) else None for nm, p in named]
        self.shadow_k = None
        if tparams is not None:
            self.shadow_k = [shadow.register(k) if _wants_shadow(nm, k) else None for (nm, _), k in zip(named, tparams)]
        self._numel = ops._numel_array(self.params)
        self._ptr = {"p": ops._ptr_array(self.params)}
        self._ptr["k"] = ops._ptr_array(self.teacher_params) if tparams is not None else None
        self._ptr["sp"] = self._opt_ptr_array(self.shadow_p)
        self._ptr["sk"] = self._opt_ptr_array(self.shadow_k) if self.shadow_k is not None else None
        self._skip_last = None

    def set_flags(self, flags: List[int]) -> None:
        """per-tensor flag words of the kernel (bit0 weight-decayed group, bit1 skip; the caller ORs in bit1 for frozen
        parameters and any kernel-specific bits)"""
        self._base_flags = torch.tensor(flags, dtype=F32)
        self.state[:, 1] = self._base_flags.to(self.state.device)

    # ---- host-side knobs (tiny async H2D copies; safe between graph replays) ---------------------------------
    def set_hyper(self, lr: float, weight_decay: float, momentum: float) -> None:
        h = self._hyper_host
        h[0], h[1] = lr, weight_decay
        e0, e1 = self._EMA_SLOTS
        h[e0], h[e1] = momentum, 1.0 - momentum  # float32(m), float32(1 - m) computed in double like the reference
        i = self._hyper_slot
        self._hyper_slot = (i + 1) % len(self._hyper_ring)
        ev = self._hyper_events[i]
        if ev is not None:
            ev.synchronize()  # the copy that last used this slot has executed (8 steps ago: never waits in practice)
        self._hyper_ring[i].copy_(h)
        self.hyper.copy_(self._hyper_ring[i], non_blocking=True)
        ev = self._hyper_events[i] = ev if ev is not None else torch.cuda.Event()
        ev.record()

    def set_skip_last_layer(self, skip: bool) -> None:
        """epoch < freeze_last_layer  <=>  the reference sets last_layer grads to None (utils.py:118-123)."""
        if skip == self._skip_last:
            return
        self._skip_last = skip
        f = self._base_flags.clone()
        if skip:
            f = torch.where(self._last_layer > 0, (f.long() | 2).float(), f)
        self._flags_host.copy_(f)
        self.state[:, 1].copy_(self._flags_host, non_blocking=True)

    def zero_grad(self) -> None:
        """set_to_none: autograd then writes each gradient straight into a fresh buffer (no += pass).  Under CUDA-graph
        capture those buffers come from the graph's private pool, so their addresses are stable across replays."""
        for p in self.params:
            p.grad = None

    def _grad_ptrs(self):
        """device pointers of this step's fp32 contiguous gradients; a parameter without one gets its own pointer as a
        dummy (the kernel never reads it: frozen or skipped).  Raises when a trainable parameter lost its gradient."""
        for p in self.params:
            g = p.grad
            if g is not None and not (g.dtype == F32 and g.is_contiguous()):
                p.grad = g.float().contiguous()
        gs = [(p.grad if p.grad is not None else p) for p in self.params]  # frozen / cancelled: dummy pointer, never read
        for i, p in enumerate(self.params):
            if p.grad is None and not self.frozen[i] and not (self._skip_last and self._last_layer[i] > 0):
                raise RuntimeError(f"parameter {self.names[i]} received no gradient this step")
        return ops._ptr_array(gs)

    @staticmethod
    def _opt_ptr_array(tensors):
        arr = (ctypes.c_void_p * len(tensors))()
        for i, t in enumerate(tensors):
            arr[i] = t.data_ptr() if t is not None else None
        return arr

    def grad_norms(self) -> torch.Tensor:
        """pre-clip per-tensor gradient norms of the last step (device tensor; what clip_gradients returned)."""
        return self.sumsq.sqrt().float()

    # ---- checkpoint interchange with the reference's `optimizer` entry (a torch optimizer over utils.get_params_groups) ----
    def _torch_order(self):
        """indices of this optimiser's parameters in torch's numbering: group 0 = regularised, group 1 = biases / 1-D
        (utils.py:672-683), trainable parameters only, each in named_parameters order"""
        reg = [i for i, (nm, p) in enumerate(zip(self.names, self.params))
               if not self.frozen[i] and not (nm.endswith(".bias") or p.dim() == 1)]
        noreg = [i for i, (nm, p) in enumerate(zip(self.names, self.params))
                 if not self.frozen[i] and (nm.endswith(".bias") or p.dim() == 1)]
        return reg, noreg


class FusedAdamWEMA(_FusedSweep):
    """clip + torch.optim.AdamW + teacher EMA (esvit_adamw_ema_multi).
    hyper = {lr, wd(group 0), beta1, beta2, eps, ema_m, 1 - ema_m, clip}"""

    def __init__(self, student: nn.Module, teacher: Optional[nn.Module], betas=(0.9, 0.999), eps: float = 1e-8,
                 clip_grad: float = 3.0):
        super().__init__(student, teacher)
        self.exp_avg = [torch.zeros_like(p) for p in self.params]
        self.exp_avg_sq = [torch.zeros_like(p) for p in self.params]
        self.set_flags([d | (2 if f else 0) for d, f in zip(self._decay, self.frozen)])
        self._hyper_host[2], self._hyper_host[3], self._hyper_host[4] = betas[0], betas[1], eps
        self._hyper_host[7] = clip_grad if clip_grad else 0.0
        self.betas, self.eps, self.clip_grad = tuple(betas), eps, clip_grad
        self.sumsq = torch.zeros(len(self.params), dtype=torch.float64, device=self.state.device)
        self._ptr["m"] = ops._ptr_array(self.exp_avg)
        self._ptr["v"] = ops._ptr_array(self.exp_avg_sq)

    @torch.no_grad()
    def step(self) -> None:
        gptr = self._grad_ptrs()
        st = ops._stream()
        n = len(self.params)
        _lib.call("esvit_grad_sumsq_multi", gptr, self._numel, n, ops._p(self.sumsq), st)
        _lib.call("esvit_adamw_ema_multi", self._ptr["p"], gptr, self._ptr["m"], self._ptr["v"], self._ptr["k"],
                  self._ptr["sp"], self._ptr["sk"], self._numel, n, ops._p(self.hyper), ops._p(self.state),
                  ops._p(self.sumsq), st)

    def state_dict(self) -> Dict:
        """torch.optim.AdamW layout: state[idx] = {step, exp_avg, exp_avg_sq} (clones) + the two param_groups, so the
        reference's restart_from_checkpoint / a plain torch AdamW can load it."""
        reg, noreg = self._torch_order()
        h = self._hyper_host
        state = {}
        for k, i in enumerate(reg + noreg):
            state[k] = {"step": self.state[i, 0].detach().clone().cpu(), "exp_avg": self.exp_avg[i].detach().clone(),
                        "exp_avg_sq": self.exp_avg_sq[i].detach().clone()}
        common = dict(lr=float(h[0]), betas=self.betas, eps=self.eps, amsgrad=False, maximize=False, foreach=None,
                      capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        groups = [dict(common, weight_decay=float(h[1]), params=list(range(len(reg)))),
                  dict(common, weight_decay=0.0, params=list(range(len(reg), len(reg) + len(noreg))))]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd: Dict, **kwargs) -> None:
        """accepts the torch AdamW layout (reference checkpoints) and this class's round-1 private layout"""
        if "exp_avg" in sd:  # round-1 private format
            for a, b in zip(self.exp_avg, sd["exp_avg"]):
                a.copy_(b)
            for a, b in zip(self.exp_avg_sq, sd["exp_avg_sq"]):
                a.copy_(b)
            self.state.copy_(sd["state"])
            return
        reg, noreg = self._torch_order()
        order = reg + noreg
        for k, st in sd["state"].items():
            i = order[int(k)]
            self.exp_avg[i].copy_(st["exp_avg"])
            self.exp_avg_sq[i].copy_(st["exp_avg_sq"])
            self.state[i, 0] = float(st["step"])
        g = sd.get("param_groups")
        if g:
            self._hyper_host[0] = g[0].get("lr", float(self._hyper_host[0]))
            self._hyper_host[1] = g[0].get("weight_decay", float(self._hyper_host[1]))


class FusedSGDEMA(_FusedSweep):
    """clip + torch.optim.SGD(momentum) or utils.LARS + teacher EMA (esvit_sgd_ema_multi), the reference's
    ``--optimizer sgd`` / ``--optimizer lars`` (main_esvit.py:412-415).
    hyper = {lr, wd(group 0), momentum, eta, ema_m, 1 - ema_m, clip, unused}

    Both are coupled-L2 heavy-ball momentum (d = g + wd p; buf = momentum buf + d; p -= lr buf; dampening 0, no
    Nesterov).  LARS (lars=True) also scales d by the trust ratio eta ||p|| / ||d|| of every parameter with
    p.dim() != 1 - by dimension, not by group - and 1 where either norm is 0.  Its norms come from one extra read of g
    and p (esvit_lars_sums_multi) that also yields the clip's sum of squares."""

    _EMA_SLOTS = (4, 5)

    def __init__(self, student: nn.Module, teacher: Optional[nn.Module], momentum: float = 0.9, lars: bool = False,
                 eta: float = 0.001, clip_grad: float = 3.0):
        super().__init__(student, teacher)
        self.momentum, self.lars, self.eta, self.clip_grad = momentum, lars, eta, clip_grad
        self.momentum_buffer = [torch.zeros_like(p) for p in self.params]
        self._trust = [lars and p.dim() != 1 for p in self.params]
        self.set_flags([d | (2 if f else 0) | (4 if t else 0)
                        for d, f, t in zip(self._decay, self.frozen, self._trust)])
        self._hyper_host[2], self._hyper_host[3] = momentum, eta
        self._hyper_host[6] = clip_grad if clip_grad else 0.0
        n = len(self.params)
        self.sums = torch.zeros(3 * n if lars else n, dtype=torch.float64, device=self.state.device)
        self.sumsq = self.sums[:n]  # sum g^2 per tensor (the LARS sums are planar, this plane first)
        self._ptr["b"] = ops._ptr_array(self.momentum_buffer)

    @torch.no_grad()
    def step(self) -> None:
        gptr = self._grad_ptrs()
        st = ops._stream()
        n = len(self.params)
        if self.lars:  # ||p|| and g.p only where the trust ratio applies and the tensor steps
            pp = self._opt_ptr_array([p if t and p.grad is not None else None for p, t in zip(self.params, self._trust)])
            _lib.call("esvit_lars_sums_multi", gptr, pp, self._numel, n, ops._p(self.sums), st)
        else:
            _lib.call("esvit_grad_sumsq_multi", gptr, self._numel, n, ops._p(self.sums), st)
        _lib.call("esvit_sgd_ema_multi", self._ptr["p"], gptr, self._ptr["b"], self._ptr["k"], self._ptr["sp"],
                  self._ptr["sk"], self._numel, n, ops._p(self.hyper), ops._p(self.state), ops._p(self.sums), st)

    def state_dict(self) -> Dict:
        """the reference's layout over utils.get_params_groups, one state entry per tensor that has stepped:
        torch.optim.SGD's {momentum_buffer} or utils.LARS's {mu}, with that optimiser's param_groups keys."""
        reg, noreg = self._torch_order()
        h = self._hyper_host
        key = "mu" if self.lars else "momentum_buffer"
        steps = self.state[:, 0].cpu()
        state = {k: {key: self.momentum_buffer[i].detach().clone()}
                 for k, i in enumerate(reg + noreg) if float(steps[i]) > 0}
        if self.lars:
            common = dict(lr=float(h[0]), momentum=self.momentum, eta=self.eta, weight_decay_filter=None,
                          lars_adaptation_filter=None)
        else:
            common = dict(lr=float(h[0]), momentum=self.momentum, dampening=0, nesterov=False, maximize=False,
                          foreach=None, differentiable=False, fused=None)
        groups = [dict(common, weight_decay=float(h[1]), params=list(range(len(reg)))),
                  dict(common, weight_decay=0.0, params=list(range(len(reg), len(reg) + len(noreg))))]
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, sd: Dict, **kwargs) -> None:
        """accepts the torch.optim.SGD and the utils.LARS layouts; a tensor without an entry restarts from a zero
        buffer (what both optimisers do for a parameter they have not stepped)"""
        reg, noreg = self._torch_order()
        order = reg + noreg
        for b in self.momentum_buffer:
            b.zero_()
        self.state[:, 0] = 0.0
        for k, st in sd["state"].items():
            buf = st.get("momentum_buffer", st.get("mu"))
            if buf is None:
                continue
            i = order[int(k)]
            self.momentum_buffer[i].copy_(buf)
            self.state[i, 0] = 1.0
        g = sd.get("param_groups")
        if g:
            self._hyper_host[0] = g[0].get("lr", float(self._hyper_host[0]))
            self._hyper_host[1] = g[0].get("weight_decay", float(self._hyper_host[1]))
