"""Compact storage of the golden vectors (tests/golden/*.pt, written by oracle/make_golden.py).

What can be recomputed is not stored: the initial weights come from a seeded recipe (seeded_state_dict), the crops from
their seed (step.synthetic_crops), and tensors of more than SAMPLE elements are kept as a fixed, seeded sample of their
elements (sample / at_golden).  load() returns the fixture with `state_dict` and `crops` filled in.
"""
from __future__ import annotations

import math

import torch

from . import step as ST
from . import swin as S

SAMPLE = 2048


def recipe(sd) -> list:
    """[(name, shape, is_float)] of a state_dict: everything seeded_state_dict needs to rebuild one like it."""
    return [(k, tuple(v.shape), bool(v.dtype.is_floating_point)) for k, v in sd.items()]


def seeded_state_dict(rec, seed: int) -> dict:
    """Deterministic weights for a state_dict layout: N(0, 0.02) matrices, N(0, 0.05) biases, 1 + N(0, 0.1) LayerNorm
    scales, N(0, 0.5) relative-position bias tables (non-zero so every term is exercised), unit weight-norm gains, and
    the closed-form relative-position index buffers."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, shape, is_float in rec:
        if not is_float:
            ws = int(round(math.sqrt(shape[0])))
            idx = S.rel_pos_index(ws)
            assert tuple(idx.shape) == tuple(shape), (name, shape)
            sd[name] = idx
        elif name.endswith("weight_g"):
            sd[name] = torch.ones(shape)
        elif name.endswith(".bias"):
            sd[name] = torch.randn(shape, generator=g) * 0.05
        elif len(shape) == 1 and "norm" in name:
            sd[name] = 1 + torch.randn(shape, generator=g) * 0.1
        elif "relative_position_bias_table" in name:
            sd[name] = torch.randn(shape, generator=g) * 0.5
        else:
            sd[name] = torch.randn(shape, generator=g) * 0.02
    return sd


def _sample_index(numel: int, seed: int) -> torch.Tensor:
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:SAMPLE]


def sample(t: torch.Tensor, seed: int = 0):
    """t itself if it is small, else {"shape", "seed", "values"}: SAMPLE of its elements picked by a seeded permutation."""
    t = t.detach()
    if t.numel() <= SAMPLE:
        return t.clone()
    return {"shape": tuple(t.shape), "seed": seed, "values": t.reshape(-1)[_sample_index(t.numel(), seed)].clone()}


def at_golden(actual: torch.Tensor, ref):
    """(actual, ref) restricted to the elements the fixture stores: both full tensors, or both the sampled elements."""
    if not isinstance(ref, dict):
        return actual, ref
    assert tuple(actual.shape) == tuple(ref["shape"]), (tuple(actual.shape), ref["shape"])
    idx = _sample_index(actual.numel(), ref["seed"]).to(actual.device)
    return actual.reshape(-1)[idx], ref["values"]


def load(path: str) -> dict:
    G = torch.load(path, map_location="cpu", weights_only=False)
    D = G["dense"]
    M = D["meta"]
    D["state_dict"] = seeded_state_dict(D["state_recipe"], M["weight_seed"])
    for k, (_, nrm) in D["initial_stats"].items():  # the rebuilt weights are the ones the reference ran with
        assert abs(float(D["state_dict"][k].double().norm()) - nrm) <= 1e-6 * nrm + 1e-9, k
    D["crops"] = ST.synthetic_crops(M["batch"], M["n_local"], seed=M["crop_seed"], global_size=M["global_size"],
                                    local_size=M["local_size"])
    return G
