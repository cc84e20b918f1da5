"""Import the UNMODIFIED reference (a checkout named by ``ESVIT_REFERENCE``, else ``oracle/_ref/``).

TEST / BASELINE INFRASTRUCTURE — ``oracle/make_golden.py``, the (skipped when the
tree is absent) cross-check tests and ``baseline/reference_gpu.py`` (bench.py's GPU
reference arm) use this.  ``oracle/_ref/`` is the git-ignored verbatim copy that
``oracle/install_reference.py`` makes during ``__graft_entry__.build()``.

Shims (SURVEY.md §8c) — the reference pins timm==0.3.2 and a 2021 torch:
  * ``timm.models.layers`` -> DropPath / to_2tuple / trunc_normal_
    (call sites models/swin_transformer.py:15,117,217,628,662)
  * ``torch._six.container_abcs`` (models/cvt_v4_transformer.py:7)
  * DINOLoss / DDINOLoss are AST-extracted from main_esvit.py:603-770 and
    exec'd verbatim, so timm.data / yacs / datasets are never imported.
"""
from __future__ import annotations

import ast
import collections.abc
import os
import sys
import types
from functools import partial

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn
import torch.nn.functional as F

def _default_root() -> str:
    """the verbatim copy that oracle/install_reference.py put under the (git-ignored) oracle/_ref/"""
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


REF_ROOT = os.environ.get("ESVIT_REFERENCE") or _default_root()


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "main_esvit.py"))


def _install_shims() -> None:
    if "timm.models.layers" not in sys.modules:
        class DropPath(nn.Module):
            def __init__(self, drop_prob=None):
                super().__init__()
                self.drop_prob = drop_prob

            def forward(self, x):
                if self.drop_prob == 0. or not self.training:
                    return x
                keep = 1 - self.drop_prob
                shape = (x.shape[0],) + (1,) * (x.ndim - 1)
                r = keep + torch.rand(shape, dtype=x.dtype, device=x.device)
                r.floor_()
                return x.div(keep) * r

        timm = types.ModuleType("timm")
        models = types.ModuleType("timm.models")
        layers = types.ModuleType("timm.models.layers")
        layers.DropPath = DropPath
        layers.to_2tuple = lambda v: tuple(v) if isinstance(v, collections.abc.Iterable) else (v, v)
        layers.trunc_normal_ = torch.nn.init.trunc_normal_
        timm.models, models.layers = models, layers
        sys.modules.update({"timm": timm, "timm.models": models, "timm.models.layers": layers})
    if "torch._six" not in sys.modules:
        six = types.ModuleType("torch._six")
        six.container_abcs = collections.abc
        sys.modules["torch._six"] = six


_cache = {}


def load():
    """Returns a namespace with SwinTransformer, DINOHead, DINOLoss, DDINOLoss, utils-like helpers."""
    if "ns" in _cache:
        return _cache["ns"]
    assert available(), f"reference tree not found at {REF_ROOT}"
    _install_shims()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import swin_transformer as ref_swin  # noqa
        from models import vision_transformer as ref_vit  # noqa
    src = open(os.path.join(REF_ROOT, "main_esvit.py")).read()
    tree = ast.parse(src)
    env = {"torch": torch, "nn": nn, "F": F, "np": np, "dist": dist}
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name in ("DINOLoss", "DDINOLoss"):
            exec(compile(ast.Module([node], []), "main_esvit.py", "exec"), env)
    usrc = open(os.path.join(REF_ROOT, "utils.py")).read()
    utree = ast.parse(usrc)
    uenv = {"torch": torch, "nn": nn, "np": np, "math": __import__("math")}
    for node in utree.body:
        if isinstance(node, ast.FunctionDef) and node.name in (
                "clip_gradients", "cancel_gradients_last_layer", "get_params_groups", "cosine_scheduler"):
            exec(compile(ast.Module([node], []), "utils.py", "exec"), uenv)
    ns = types.SimpleNamespace(
        swin=ref_swin, SwinTransformer=ref_swin.SwinTransformer, DINOHead=ref_vit.DINOHead,
        DINOLoss=env["DINOLoss"], DDINOLoss=env["DDINOLoss"],
        clip_gradients=uenv["clip_gradients"], cancel_gradients_last_layer=uenv["cancel_gradients_last_layer"],
        get_params_groups=uenv["get_params_groups"], cosine_scheduler=uenv["cosine_scheduler"])
    _cache["ns"] = ns
    return ns


def ensure_process_group() -> None:
    """The reference losses call dist.all_reduce unconditionally (main_esvit.py:656)."""
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29533")
        dist.init_process_group("gloo", rank=0, world_size=1)


def build_swin(spec, out_dim: int, drop_path_rate: float = 0.0, seed: int = 0):
    """What main_esvit.py:235-254 builds for one network (student or teacher)."""
    ns = load()
    torch.manual_seed(seed)
    m = ns.SwinTransformer(
        img_size=spec.img_size, in_chans=3, num_classes=0, patch_size=spec.patch_size,
        embed_dim=spec.embed_dim, depths=list(spec.depths), num_heads=list(spec.num_heads),
        window_size=spec.window_size, mlp_ratio=spec.mlp_ratio, qkv_bias=True, drop_rate=0.0,
        attn_drop_rate=0.0, drop_path_rate=drop_path_rate, norm_layer=partial(nn.LayerNorm, eps=1e-6),
        ape=False, patch_norm=True, use_dense_prediction=spec.use_dense_prediction)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m.head = ns.DINOHead(m.num_features, out_dim)
        if spec.use_dense_prediction:
            m.head_dense = ns.DINOHead(m.num_features, out_dim)
    return m
