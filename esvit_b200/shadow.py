"""Persistent bf16 "shadow" copies of fp32 master parameters.

The GEMMs consume bf16 weights.  Casting ~110 tensors per network per step costs ~1 ms of tiny kernels; instead the fused
optimiser sweep (esvit_adamw_ema_multi) writes the bf16 copy of every updated student / teacher parameter in the same
pass.  This registry hands those copies to the modules and keeps them honest: a shadow is re-cast whenever the master
parameter was modified by anything that bumps its autograd version counter (load_state_dict, init, a torch optimizer) -
the fused kernel itself writes master and shadow together through raw pointers and does not bump it.
"""
from __future__ import annotations

import weakref
from typing import Dict, Optional, Tuple

import torch

BF16 = torch.bfloat16
_registry: Dict[int, Tuple[weakref.ref, torch.Tensor, int]] = {}


def register(param: torch.Tensor) -> torch.Tensor:
    """Create (or return) the bf16 shadow of `param`."""
    ent = _registry.get(id(param))
    if ent is not None and ent[0]() is param:
        return ent[1]
    shadow = param.detach().to(BF16)
    _registry[id(param)] = (weakref.ref(param), shadow, param._version)
    return shadow


def lookup(param: torch.Tensor) -> Optional[torch.Tensor]:
    """The up-to-date shadow of `param`, or None when it has none."""
    ent = _registry.get(id(param))
    if ent is None or ent[0]() is not param:
        return None
    ref, shadow, ver = ent
    if param._version != ver:  # master changed behind the optimiser's back: re-cast (same storage, graph-safe)
        with torch.no_grad():
            shadow.copy_(param.detach())
        _registry[id(param)] = (ref, shadow, param._version)
    return shadow


def as_bf16(param: torch.Tensor) -> torch.Tensor:
    """bf16 copy of a parameter for a GEMM, outside autograd (the GEMM's Function routes the fp32 weight gradient to
    the master parameter): the registered shadow when there is one, a fresh cast otherwise."""
    s = lookup(param)
    return param.detach().to(BF16) if s is None else s
