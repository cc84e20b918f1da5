"""The multi-crop self-distillation training step (train_one_epoch's loop body, main_esvit.py:507-590) driven
through the esvit_b200 modules.  ``main_esvit.py`` can keep its own loop (INTEGRATION.md); this class is the same
sequence packaged for bench.py / smoke / tests:

    lr/wd -> teacher fwd (no grad) -> student fwd -> DINO/DDINO loss (+ packed center all-reduce) -> backward
    (DDP gradient all-reduce when wrapped) -> per-tensor clip -> cancel last-layer grads -> AdamW / SGD / LARS
    -> teacher EMA

with NO host synchronisation inside the step (the reference syncs ~190 times per step, SURVEY.md §3.5).
"""
from __future__ import annotations

from functools import partial
from typing import List, Optional, Sequence

import torch
import torch.nn as nn

import torch.distributed as dist

from . import ops, utils
from .losses import DDINOLoss, DINOLoss, mixup_targets
from .optim import FusedAdamWEMA, FusedSGDEMA
from . import cvt_v4_transformer as cvts
from . import vision_longformer as vils
from . import vision_transformer as vits
from .swin_transformer import SwinTransformer
from .vision_transformer import DINOHead

SWIN_SPECS = {
    "swin_tiny_w7": dict(embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=7, drop_path_rate=0.1),
    "swin_tiny_w14": dict(embed_dim=96, depths=[2, 2, 6, 2], num_heads=[3, 6, 12, 24], window_size=14, drop_path_rate=0.1),
    "swin_small_w7": dict(embed_dim=96, depths=[2, 2, 18, 2], num_heads=[3, 6, 12, 24], window_size=7, drop_path_rate=0.2),
    "swin_small_w14": dict(embed_dim=96, depths=[2, 2, 18, 2], num_heads=[3, 6, 12, 24], window_size=14, drop_path_rate=0.2),
    "swin_base_w7": dict(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=7, drop_path_rate=0.2),
    "swin_base_w14": dict(embed_dim=128, depths=[2, 2, 18, 2], num_heads=[4, 8, 16, 32], window_size=14, drop_path_rate=0.2),
    "swin_large_w7": dict(embed_dim=192, depths=[2, 2, 18, 2], num_heads=[6, 12, 24, 48], window_size=7, drop_path_rate=0.2),
}
# ViT / DeiT (main_esvit.py:304-327): `vit_arch` names the factory in esvit_b200.vision_transformer
VIT_SPECS = {
    "deit_tiny_p16": dict(vit_arch="deit_tiny", patch_size=16, drop_path_rate=0.1),
    "deit_small_p16": dict(vit_arch="deit_small", patch_size=16, drop_path_rate=0.1),
    "deit_small_p8": dict(vit_arch="deit_small", patch_size=8, drop_path_rate=0.1),
    "vit_base_p16": dict(vit_arch="vit_base", patch_size=16, drop_path_rate=0.1),
}

# CvT (main_esvit.py:280-301 with experiments/imagenet/cvt_v4/s1.yaml, and win_size/s1.yaml for cvt_13_w14; s3.yaml
# and win_size/s3.yaml for cvt_s3 / cvt_s3_w14): `cvt_spec` is the MODEL.SPEC
CVT_SPECS = {
    "cvt_13": dict(cvt_spec=cvts.S1_SPEC, drop_path_rate=0.1),
    "cvt_13_w14": dict(cvt_spec=cvts.S1_W14_SPEC, drop_path_rate=0.1),
    "cvt_s3": dict(cvt_spec=cvts.S3_SPEC, drop_path_rate=0.2),
    "cvt_s3_w14": dict(cvt_spec=cvts.S3_W14_SPEC, drop_path_rate=0.2),
}

# Vision Longformer (main_esvit.py:257-276 with the README's vil_2262 arch): `vil_spec` holds MsViT's arguments
VIL_SPECS = {
    "vil_2262": dict(vil_spec=vils.VIL_2262, drop_path_rate=0.1),
}


def build_network(spec: dict, out_dim: int, use_dense_prediction: bool, is_teacher: bool = False,
                  norm_last_layer: bool = True, img_size: int = 224, head_kwargs: Optional[dict] = None) -> nn.Module:
    """What main_esvit.py:235-254 (Swin) / :304-327 (ViT, a spec with `vit_arch`) / :280-301 (CvT, a spec with
    `cvt_spec`) / :257-276 (ViL, a spec with `vil_spec`; num_features = out_planes) builds: the backbone (teacher:
    drop_path 0) + DINOHead(s) assigned to ``.head`` / ``.head_dense``."""
    spec = dict(spec)
    if is_teacher:
        spec["drop_path_rate"] = 0.0
    vit_arch = spec.pop("vit_arch", None)
    cvt_spec = spec.pop("cvt_spec", None)
    vil_spec = spec.pop("vil_spec", None)
    if vil_spec is not None:
        net = vils.msvit(vil_spec, 0, use_dense_prediction, drop_path_rate=spec["drop_path_rate"])
    elif cvt_spec is not None:
        net = cvts.cvt(cvt_spec, 0, use_dense_prediction, drop_path_rate=spec["drop_path_rate"])
    elif vit_arch is not None:
        net = vits.__dict__[vit_arch](img_size=[img_size], use_dense_prediction=use_dense_prediction, **spec)
    else:
        net = SwinTransformer(img_size=img_size, in_chans=3, num_classes=0, patch_size=4, mlp_ratio=4., qkv_bias=True,
                              norm_layer=partial(nn.LayerNorm, eps=1e-6), use_dense_prediction=use_dense_prediction,
                              **spec)
    hk = head_kwargs or {}
    net.head = DINOHead(net.num_features, out_dim, norm_last_layer=norm_last_layer, **hk)
    if use_dense_prediction:
        net.head_dense = DINOHead(net.num_features, out_dim, norm_last_layer=norm_last_layer, **hk)
    return net


class _GradReducer:
    """Bucketed gradient all-reduce overlapped with backward - what DistributedDataParallel does for the reference
    (main_esvit.py:377), in a form that is captured inside the step's CUDA graph: parameters are bucketed in REVERSE
    registration order (= the order backward completes them: the two 65536-wide last layers, 45 % of all gradient bytes,
    first), a post-accumulate-grad hook counts completed gradients per bucket and, when a bucket is full, forks a side
    stream that flattens the bucket, AVG-all-reduces it over NCCL and scatters it back while the main stream continues
    with the remaining backward kernels.  finish() launches whatever is left and joins the side stream before the
    optimiser sweep.  The result is independent of the bucketing (same AVG per element)."""

    def __init__(self, params, bucket_bytes: int = 48 << 20):
        self.params = [p for p in params if p.requires_grad]
        self.buckets, cur, size = [], [], 0
        for p in reversed(self.params):
            cur.append(p)
            size += p.numel() * 4
            if size >= bucket_bytes:
                self.buckets.append(cur)
                cur, size = [], 0
        if cur:
            self.buckets.append(cur)
        self.bucket_of = {id(p): bi for bi, b in enumerate(self.buckets) for p in b}
        self.count = [0] * len(self.buckets)
        self.launched = [False] * len(self.buckets)
        self.side = torch.cuda.Stream()
        self.enabled = True
        for p in self.params:
            p.register_post_accumulate_grad_hook(self._hook)

    def _hook(self, p) -> None:
        if not self.enabled:
            return
        bi = self.bucket_of[id(p)]
        self.count[bi] += 1
        if self.count[bi] == len(self.buckets[bi]) and not self.launched[bi]:
            self._launch(bi)

    def _launch(self, bi: int) -> None:
        self.launched[bi] = True
        grads = [p.grad for p in self.buckets[bi] if p.grad is not None]
        if not grads:
            return
        self.side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.side):
            flat = torch.cat([g.reshape(-1) for g in grads])
            dist.all_reduce(flat, op=dist.ReduceOp.AVG)
            torch._foreach_copy_(grads, [t.view_as(g) for t, g in zip(flat.split([g.numel() for g in grads]), grads)])

    def finish(self) -> None:
        for bi in range(len(self.buckets)):
            if not self.launched[bi]:
                self._launch(bi)
        torch.cuda.current_stream().wait_stream(self.side)
        self.count = [0] * len(self.buckets)
        self.launched = [False] * len(self.buckets)


class SelfDistillStep:
    """One training step.  optimizer: a torch optimizer (the reference's own sequence: clip kernel, cancel grads,
    optimizer.step(), EMA kernel) or an esvit_b200.optim.FusedAdamWEMA / FusedSGDEMA (clip + AdamW / SGD / LARS + EMA
    in one sweep).  With use_cuda_graph=True (fused optimisers only) the whole step - teacher fwd, student fwd/bwd,
    loss, center update, gradient all-reduce, optimiser sweep - is captured once per (teacher_temp, last-layer-frozen) state and replayed:
    no Python / launch overhead in the steady state.  lr / wd / momentum live in device memory and are refreshed with
    an 32-byte async copy before each replay."""

    def __init__(self, student: nn.Module, teacher: nn.Module, loss: nn.Module, optimizer, clip_grad: float = 3.0,
                 freeze_last_layer: int = 1, student_ddp: Optional[nn.Module] = None, use_cuda_graph: bool = False,
                 grad_allreduce: bool = False):
        self.student, self.teacher, self.loss, self.opt = student, teacher, loss, optimizer
        self.student_call = student_ddp if student_ddp is not None else student
        self.clip_grad, self.freeze_last_layer = clip_grad, freeze_last_layer
        self.fused = isinstance(optimizer, (FusedAdamWEMA, FusedSGDEMA))
        self.use_cuda_graph = use_cuda_graph and self.fused
        self.grad_allreduce = grad_allreduce  # own flat all-reduce of the gradients (used instead of DDP in graph mode)
        self.last_norms = None
        self._graphs = {}
        self._pool = None
        self._static_in = None
        self._static_loss = None
        self._warm = 0
        self._static_mix = None  # (teacher crops, student crops, targets) of the student_images / targets_mixup step
        self._warm_mix = 0
        for p in self.teacher.parameters():
            p.requires_grad = False
        # arena for the ACCUMULATED small gradients (LN affine, biases, rel-pos tables, patch embed): sized from the model
        small = sum(p.numel() for p in self.student.parameters() if p.dim() == 1 or p.numel() <= (1 << 16))
        self._arena_floats = 4 * small + (1 << 18)
        self._reducer = None
        if self.grad_allreduce and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            self._reducer = _GradReducer(list(self.student.parameters()))

    # ---- the step body (eager; also what gets captured) ---------------------------------------------------
    def _body(self, images: List[torch.Tensor], epoch: int, student_images: Optional[List[torch.Tensor]] = None,
              targets_mixup: Optional[List[torch.Tensor]] = None) -> torch.Tensor:
        with torch.no_grad():
            teacher_output = self.teacher(images[:2])
        student_output = self.student_call(images if student_images is None else student_images)
        loss = self.loss(student_output, teacher_output, epoch, targets_mixup)
        if self.fused:
            self.opt.zero_grad()
        else:
            self.opt.zero_grad(set_to_none=True)
        ops.begin_step(loss.device, self._arena_floats)  # one zero-filled arena for all small gradient accumulators
        try:
            loss.backward()
        finally:
            ops.end_step()
        self.reduce_gradients()
        if self.fused:
            self.opt.step()  # clip + AdamW / SGD / LARS + EMA, one sweep
        else:
            if self.clip_grad:
                self.last_norms = utils.clip_gradients(self.student, self.clip_grad)
            utils.cancel_gradients_last_layer(epoch, self.student, self.freeze_last_layer)
            self.opt.step()
        return loss.detach()

    def reduce_gradients(self) -> None:
        """DDP's gradient AVG all-reduce (main_esvit.py:377) for the graph-captured step: buckets whose gradients were
        complete during backward have already been launched on the side stream by the post-accumulate hooks
        (_GradReducer); this launches the rest and joins the side stream.  No-op at world size 1."""
        if self._reducer is not None:
            self._reducer.finish()

    def __call__(self, images: Sequence[torch.Tensor], epoch: int, lr: float, wd: float, momentum: float) -> torch.Tensor:
        return self.step(images, epoch, lr, wd, momentum)

    def step(self, images: Sequence[torch.Tensor], epoch: int, lr: float, wd: float, momentum: float,
             student_images: Optional[Sequence[torch.Tensor]] = None,
             targets_mixup: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
        """One step.  The teacher reads images[:2]; the student reads student_images when given (the mixed crops of
        ``--use_mixup``, main_esvit.py:516-543), else images; targets_mixup goes to the loss (per-view [B, B] targets)."""
        images = list(images)
        student_images = None if student_images is None else list(student_images)
        targets_mixup = list(targets_mixup) if targets_mixup else None
        if self.fused:
            self.opt.set_hyper(lr, wd, momentum)
            self.opt.set_skip_last_layer(epoch < self.freeze_last_layer)
        else:
            for i, g in enumerate(self.opt.param_groups):  # main_esvit.py:507-510
                g["lr"] = lr
                if i == 0:
                    g["weight_decay"] = wd
        if not self.use_cuda_graph:
            loss = self._body(images, epoch, student_images, targets_mixup)
            if not self.fused:
                utils.ema_update(self.student, self.teacher, momentum)
            return loss
        if student_images is None and targets_mixup is None:
            return self._graphed(images, epoch)
        return self._graphed_mixup(images, epoch, images if student_images is None else student_images, targets_mixup)

    # ---- CUDA-graph path ------------------------------------------------------------------------------------
    def _graphed(self, images: List[torch.Tensor], epoch: int) -> torch.Tensor:
        """Replay path.  The graph reads PRIVATE static input buffers (allocated on first use); every call copies the
        caller's crops into them on the current stream, so the caller may recycle its own (prefetch) buffers freely.  A
        batch of a different shape (e.g. a shorter last batch) runs the eager body instead."""
        if self._static_in is None:
            self._static_in = _static_buffers(images)
        if not _fits(self._static_in, images):
            return self._body(images, epoch)
        for s, im in zip(self._static_in, images):
            s.copy_(im, non_blocking=True)
        if self._warm < 3:  # eager warm-up (allocator, cuBLAS workspaces, cached tables) before any capture
            self._warm += 1
            return self._body(self._static_in, epoch)
        key = (float(self.loss.teacher_temp_schedule[epoch]), epoch < self.freeze_last_layer)
        ent = self._graphs.get(key)
        if ent is None:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self._pool):
                out = self._body(self._static_in, epoch)
            if self._pool is None:
                self._pool = g.pool()
            ent = self._graphs[key] = (g, out)
        ent[0].replay()
        return ent[1]

    def _graphed_mixup(self, images: List[torch.Tensor], epoch: int, student_images: List[torch.Tensor],
                       targets_mixup: Optional[List[torch.Tensor]]) -> torch.Tensor:
        """Replay path of a step with student_images / targets_mixup: its own graph per (teacher_temp, last-layer-frozen)
        state, reading private static buffers for the two teacher crops, the student crops and the targets.  The targets
        are checked (losses.mixup_targets) before they are copied in; inside the capture only their shape is."""
        if targets_mixup is not None:
            B = images[0].shape[0]
            targets = mixup_targets(targets_mixup, self.loss.ncrops, B, images[0].device)
        if self._static_mix is None:
            self._static_mix = (_static_buffers(images[:2]), _static_buffers(student_images),
                                None if targets_mixup is None else torch.empty_like(targets))
        st_t, st_s, st_y = self._static_mix
        if (not _fits(st_t, images[:2]) or not _fits(st_s, student_images) or (st_y is None) != (targets_mixup is None)
                or (st_y is not None and st_y.shape != targets.shape)):
            return self._body(images, epoch, student_images, targets_mixup)
        for s, im in zip(st_t + st_s, images[:2] + student_images):
            s.copy_(im, non_blocking=True)
        if st_y is not None:
            st_y.copy_(targets, non_blocking=True)
        args = (st_t, epoch, st_s, None if st_y is None else list(st_y.unbind(0)))
        if self._warm_mix < 3:
            self._warm_mix += 1
            return self._body(*args)
        key = (float(self.loss.teacher_temp_schedule[epoch]), epoch < self.freeze_last_layer, "mixup")
        ent = self._graphs.get(key)
        if ent is None:
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self._pool):
                out = self._body(*args)
            if self._pool is None:
                self._pool = g.pool()
            ent = self._graphs[key] = (g, out)
        ent[0].replay()
        return ent[1]


def _static_buffers(images: List[torch.Tensor]) -> List[torch.Tensor]:
    """Views of private buffers shaped like `images`.  Crops of one shape share one buffer, back to back: the multi-crop
    forward then views a resolution group as one batch instead of concatenating it (ops.cat_adjacent)."""
    out, i = [], 0
    while i < len(images):
        j = i
        while j < len(images) and images[j].shape == images[i].shape and images[j].dtype == images[i].dtype:
            j += 1
        buf = torch.empty((j - i,) + tuple(images[i].shape), dtype=images[i].dtype, device=images[i].device)
        out += [buf[k] for k in range(j - i)]
        i = j
    return out


def _fits(static: List[torch.Tensor], images: List[torch.Tensor]) -> bool:
    return len(images) == len(static) and all(s.shape == im.shape for s, im in zip(static, images))


def make_step(arch: str = "swin_tiny_w7", out_dim: int = 65536, ncrops: int = 10, dense: bool = True,
              device: str = "cuda", lr: float = 5e-4, weight_decay: float = 0.04, clip_grad: float = 3.0,
              freeze_last_layer: int = 1, drop_path: Optional[float] = None, img_size: int = 224,
              head_kwargs: Optional[dict] = None, spec: Optional[dict] = None, ddp: bool = False,
              teacher_temp: float = 0.04, seed: int = 0, optimizer: str = "fused", cuda_graph: bool = False,
              optimizer_type: str = "adamw"):
    """Build student/teacher/loss/optimizer the way train_esvit does (main_esvit.py:235-435) and return
    (step, student, teacher, loss).  optimizer_type is main_esvit.py's ``--optimizer`` (adamw | sgd | lars);
    optimizer picks the implementation: "fused" (FusedAdamWEMA / FusedSGDEMA) or "torch" (the reference's own
    torch.optim.AdamW / torch.optim.SGD objects; utils.LARS has no torch counterpart here)."""
    if optimizer_type not in ("adamw", "sgd", "lars"):
        raise ValueError(f"optimizer_type must be adamw, sgd or lars, not {optimizer_type!r}")
    if optimizer != "fused" and optimizer_type == "lars":
        raise ValueError("optimizer_type='lars' runs on the fused sweep only: use optimizer='fused'")
    if spec is None:
        spec = VIT_SPECS.get(arch) or CVT_SPECS.get(arch) or VIL_SPECS.get(arch) or SWIN_SPECS[arch]
    spec = dict(spec)
    if drop_path is not None:
        spec["drop_path_rate"] = drop_path
    torch.manual_seed(seed)
    student = build_network(spec, out_dim, dense, False, True, img_size, head_kwargs).to(device)
    teacher = build_network(spec, out_dim, dense, True, True, img_size, head_kwargs).to(device)
    teacher.load_state_dict(student.state_dict())
    Loss = DDINOLoss if dense else DINOLoss
    loss = Loss(out_dim, ncrops, teacher_temp, teacher_temp, 0, 100).to(device)
    student_ddp = None
    multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    if multi and (head_kwargs or {}).get("use_bn"):
        # main_esvit.py:366-373: BN heads -> SyncBatchNorm in both networks (their statistics span every rank's rows)
        student = nn.SyncBatchNorm.convert_sync_batchnorm(student)
        teacher = nn.SyncBatchNorm.convert_sync_batchnorm(teacher)
    if ddp and multi and optimizer != "fused":
        student_ddp = nn.parallel.DistributedDataParallel(student, device_ids=[torch.cuda.current_device()])
    if optimizer == "fused":
        for p in teacher.parameters():
            p.requires_grad = False
        if optimizer_type == "adamw":
            opt = FusedAdamWEMA(student, teacher, clip_grad=clip_grad)
        else:
            opt = FusedSGDEMA(student, teacher, lars=(optimizer_type == "lars"), clip_grad=clip_grad)
    elif optimizer_type == "sgd":  # the reference's own optimizer objects (main_esvit.py:410-415)
        opt = torch.optim.SGD(utils.get_params_groups(student), lr=0, momentum=0.9)
    else:
        opt = torch.optim.AdamW(utils.get_params_groups(student), fused=True)
    step = SelfDistillStep(student, teacher, loss, opt, clip_grad, freeze_last_layer, student_ddp,
                           use_cuda_graph=cuda_graph, grad_allreduce=(optimizer == "fused" and multi))
    return step, student, teacher, loss
