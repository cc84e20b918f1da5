"""The reference's own training step, on the GPU, from the reference's own modules - the comparator of the north-star
target ("the reference's own PyTorch/cuDNN build on the same box").

Nothing of esvit_b200 is on this path: the UNMODIFIED `models.swin_transformer.SwinTransformer`,
`models.vision_transformer.DINOHead` and the `DDINOLoss` class of main_esvit.py (imported from oracle/_ref or
the reference checkout through oracle/reference_import.py's three shims: timm.models.layers, torch._six, AST extraction of the
loss classes) are driven through the statement sequence of train_one_epoch (main_esvit.py:507-598):

    lr/wd -> autocast{teacher(images[:2]); student(images); loss} -> loss.item() finite check -> zero_grad ->
    [scaler.scale(loss)] backward -> synchronize -> [unscale_] per-parameter clip_gradients (utils.py:106-115) ->
    cancel_gradients_last_layer -> [scaler.]step -> [scaler.update] -> EMA loop over parameters -> synchronize

with DistributedDataParallel around the student at world size > 1 (main_esvit.py:377), torch.optim.AdamW over
utils.get_params_groups (main_esvit.py:410-415).  Two precisions: the reference's default fp16 autocast + GradScaler
(main_esvit.py:417-419) and bf16 autocast without a scaler (BASELINE.json configs say bf16)."""
from __future__ import annotations

import math
import os
import sys
import time
from typing import List

import torch
import torch.distributed as dist
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def available() -> bool:
    from oracle import reference_import as RI
    return RI.available()


class ReferenceGpuStep:
    def __init__(self, spec_d: dict, out_dim: int, ncrops: int, device, precision: str = "bf16", lr: float = 5e-4,
                 weight_decay: float = 0.04, clip_grad: float = 3.0, freeze_last_layer: int = 1,
                 momentum_teacher: float = 0.996, drop_path_rate: float = 0.1, seed: int = 0):
        from oracle import reference_import as RI
        from oracle import swin as S
        ns = RI.load()
        if not dist.is_initialized():  # the reference losses all-reduce unconditionally (main_esvit.py:656)
            import socket
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            if "MASTER_PORT" not in os.environ:
                with socket.socket() as sk:
                    sk.bind(("127.0.0.1", 0))
                    os.environ["MASTER_PORT"] = str(sk.getsockname()[1])
            dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device(device))
        spec = S.SwinSpec(img_size=224, embed_dim=spec_d["embed_dim"], depths=tuple(spec_d["depths"]),
                          num_heads=tuple(spec_d["num_heads"]), window_size=spec_d["window_size"],
                          use_dense_prediction=True)
        self.student = RI.build_swin(spec, out_dim, drop_path_rate=drop_path_rate, seed=seed).to(device)
        self.teacher = RI.build_swin(spec, out_dim, drop_path_rate=0.0, seed=seed).to(device)
        self.teacher.load_state_dict(self.student.state_dict())          # main_esvit.py:379
        for p in self.teacher.parameters():                              # main_esvit.py:381-382
            p.requires_grad = False
        self.student_call = self.student
        if dist.is_initialized() and dist.get_world_size() > 1 and dist.get_backend() == "nccl":
            self.student_call = nn.parallel.DistributedDataParallel(self.student, device_ids=[torch.cuda.current_device()])
        self.loss = ns.DDINOLoss(out_dim, ncrops, 0.04, 0.04, 0, 100).to(device)
        self.opt = torch.optim.AdamW(ns.get_params_groups(self.student))  # main_esvit.py:410-415
        self.ns, self.lr, self.wd = ns, lr, weight_decay
        self.clip_grad, self.freeze_last_layer, self.m = clip_grad, freeze_last_layer, momentum_teacher
        self.precision = precision
        self.scaler = torch.amp.GradScaler("cuda") if precision == "fp16" else None   # main_esvit.py:417-419
        self.dtype = {"fp16": torch.float16, "bf16": torch.bfloat16}[precision]
        self.student.train()
        self.teacher.train()

    def step(self, images: List[torch.Tensor], epoch: int = 1) -> float:
        for i, g in enumerate(self.opt.param_groups):                    # :507-510
            g["lr"] = self.lr
            if i == 0:
                g["weight_decay"] = self.wd
        with torch.autocast("cuda", dtype=self.dtype):                   # :541-544
            teacher_output = self.teacher(images[:2])
            student_output = self.student_call(images)
            loss = self.loss(student_output, teacher_output, epoch, None)
        lv = loss.item()                                                 # :546
        if not math.isfinite(lv):
            raise RuntimeError(f"reference loss is {lv}")
        self.opt.zero_grad()                                             # :565
        if self.scaler is None:                                          # :567-574
            loss.backward()
            torch.cuda.synchronize()
            if self.clip_grad:
                self.ns.clip_gradients(self.student, self.clip_grad)
            self.ns.cancel_gradients_last_layer(epoch, self.student, self.freeze_last_layer)
            self.opt.step()
        else:                                                            # :575-584
            self.scaler.scale(loss).backward()
            torch.cuda.synchronize()
            if self.clip_grad:
                self.scaler.unscale_(self.opt)
                self.ns.clip_gradients(self.student, self.clip_grad)
            self.ns.cancel_gradients_last_layer(epoch, self.student, self.freeze_last_layer)
            self.scaler.step(self.opt)
            self.scaler.update()
        with torch.no_grad():                                            # :587-590
            m = self.m
            for param_q, param_k in zip(self.student.parameters(), self.teacher.parameters()):
                param_k.data.mul_(m).add_((1 - m) * param_q.detach().data)
        torch.cuda.synchronize()                                         # :593
        return lv


def time_reference(spec_d: dict, out_dim: int, ncrops: int, crops: List[torch.Tensor], device, precision: str,
                   steps: int, warmup: int, drop_path_rate: float) -> dict:
    """ms/step of the reference step (CUDA events around `steps` steps after `warmup`), max over ranks."""
    ref = ReferenceGpuStep(spec_d, out_dim, ncrops, device, precision, drop_path_rate=drop_path_rate)
    lv = float("nan")
    for _ in range(warmup):
        lv = ref.step(crops)
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(steps):
        lv = ref.step(crops)
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / steps
    ms = e0.elapsed_time(e1) / steps
    if dist.is_initialized() and dist.get_world_size() > 1 and dist.get_backend() == "nccl":
        t = torch.tensor([ms], dtype=torch.float64, device=device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    peak = torch.cuda.max_memory_allocated(device) / 2 ** 30
    del ref
    torch.cuda.empty_cache()
    return {"ms_per_step": ms, "wall_ms_per_step": wall, "last_loss": lv, "steps": steps, "warmup": warmup,
            "precision": precision + (" autocast + GradScaler (reference default)" if precision == "fp16" else " autocast"),
            "peak_mem_gib": peak}
