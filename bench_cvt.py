"""CvT pre-training step on one GPU: CvT-13 spec s1 (--arch cvt_13, windows 7) or win_size/s1 (--arch cvt_13_w14, windows
14, 14, 14, 7), spec s3 (--arch cvt_s3, head dim 32, windows 7) or win_size/s3 (--arch cvt_s3_w14), 2 x 224^2 + 8 x
96^2 crops, DDINOLoss (dense), K = 65 536.

    python bench_cvt.py [--arch cvt_13] [--batch 64] [--steps 10] [--warmup 3] [--no-reference]

Prints one JSON line:
  * `value`: images/s of esvit_b200's captured step (engine.make_step(arch), CUDA graph, loss read back every step
    as train_one_epoch does) at the largest batch of --batch, 48, 32, 16 that fits, reported as `batch`;
  * `reference`: the UNMODIFIED reference modules (models.cvt_v4_transformer.CvT built as get_cls_model builds it from
    the arch's MODEL.SPEC, DINOHead, DDINOLoss from oracle/_ref/, installed by build()) through main_esvit.py:541-590's
    statement sequence under bf16 autocast, student and teacher in train mode, at the largest batch that fits; "not
    run" with the reason when the tree is absent or nothing fits;
  * `kernels`: CUDA-event times per step of the CvT kernels (conv-embed gather / col2im, depthwise + BN forward /
    backward, window attention forward / backward) with their algorithmic bytes (and FLOPs for attention), achieved
    TB/s, and share of the bound the data sheet gives (the larger of FLOPs / 989 TFLOP/s and bytes / 3.35 TB/s), from
    an eager step; for every arch but cvt_13 also `attention_by_L`, the window attention split by tokens per window L = w^2;
  * `gpu`: card name, power limit and maximum SM clock, read in the same run.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

K, NCROPS, LR, WD, MOM = 65536, 10, 5e-4, 0.04, 0.996
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [f.strip() for f in out.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:  # nvidia-smi missing: the name alone
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e.__class__.__name__})"}


def crops(B: int):
    g = torch.Generator(device="cuda").manual_seed(0)
    return [torch.randn(B, 3, 224, 224, device="cuda", generator=g) for _ in range(2)] + \
           [torch.randn(B, 3, 96, 96, device="cuda", generator=g) for _ in range(NCROPS - 2)]


def _timed(fn, steps: int) -> float:
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


NAMES = ("esvit_conv_im2col", "esvit_conv_col2im", "esvit_dwbn_fwd_stats", "esvit_dwbn_fwd_apply", "esvit_dwbn_bwd_stats",
         "esvit_dwbn_bwd_apply", "esvit_mhsa_win_fwd", "esvit_mhsa_win_bwd")


def _cost(r) -> tuple:
    """(algorithmic bytes, FLOPs) of one call, from its shapes"""
    n = r["name"]
    if n in ("esvit_conv_im2col", "esvit_conv_col2im"):
        Ho = (r["H"] + 2 * r["p"] - r["k"]) // r["s"] + 1
        Wo = (r["W"] + 2 * r["p"] - r["k"]) // r["s"] + 1
        return r["B"] * r["H"] * r["W"] * r["C"] * 4 + r["B"] * Ho * Wo * r["Kp"] * 2, 0.0
    if n == "esvit_dwbn_fwd_stats":    # y in, z out
        return (r["B"] * r["H"] * r["W"] + r["B"] * r["Hp"] * r["Wp"]) * r["C"] * 2, 0.0
    if n in ("esvit_dwbn_fwd_apply", "esvit_dwbn_bwd_stats"):   # two bf16 [N, C] streams
        return r["N"] * r["C"] * 4, 0.0
    if n == "esvit_dwbn_bwd_apply":    # dy, z in; dx out; filter gradient reads dy, z, y
        N, T = r["B"] * r["Hp"] * r["Wp"], r["B"] * r["H"] * r["W"]
        return (2 * N + T + 2 * N + T) * r["C"] * 2, 0.0
    # window attention: every token of the padded map once per head
    L = r["w"] * r["w"]
    Hp, Wp = -(-r["H"] // r["w"]) * r["w"], -(-r["W"] // r["w"]) * r["w"]
    Tp, T = r["B"] * Hp * Wp, r["B"] * r["H"] * r["W"]
    flops = 4.0 * Tp * L * r["C"]
    if n.endswith("fwd"):
        return Tp * 3 * r["C"] * 2 + T * r["C"] * 2 + Tp * r["nH"] * 4, flops
    return Tp * 3 * r["C"] * 2 * 2 + T * r["C"] * 2 * 2 + Tp * r["nH"] * 8, 2.5 * flops


def _rates(rows) -> dict:
    ms = sum(r["ms"] for r in rows)
    nbytes = sum(_cost(r)[0] for r in rows)
    flops = sum(_cost(r)[1] for r in rows)
    bound_ms = max(flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBS * 1e12)) * 1e3
    return {"ms_per_step": round(ms, 3), "launches": len(rows), "gb": round(nbytes / 1e9, 3),
            "tb_s": round(nbytes / ms / 1e9, 3), "tflops": round(flops / ms / 1e9, 1),
            "share_of_bound": round(bound_ms / ms, 3),
            "bound": "tensor" if flops / PEAK_TFLOPS > nbytes / PEAK_TBS else "hbm"}


def _attention_by_L(res) -> dict:
    """window attention forward / backward per window size: {"L=196": {"fwd": rates, "bwd": rates}, ...}"""
    out = {}
    for L in sorted({r["w"] * r["w"] for r in res if r["name"].startswith("esvit_mhsa_win")}, reverse=True):
        out[f"L={L}"] = {d: _rates([r for r in res if r["name"] == f"esvit_mhsa_win_{d}" and r["w"] * r["w"] == L])
                         for d in ("fwd", "bwd")}
    return out


def _kernel_rates(res) -> dict:
    out = {}
    for name in NAMES:
        rows = [r for r in res if r["name"] == name]
        if not rows:
            continue
        out[name] = _rates(rows)
    return out


def run_ours(arch: str, B: int, steps: int, warmup: int) -> dict:
    from esvit_b200 import _lib, engine
    step, student, teacher, loss = engine.make_step(arch=arch, out_dim=K, ncrops=NCROPS, dense=True, cuda_graph=True)
    imgs = crops(B)
    float(step(imgs, 1, LR, WD, MOM))                    # eager warm-up 1 (module loads, allocator)
    _lib.reset_counters()
    _lib.time_entry_point(list(NAMES))
    float(step(imgs, 1, LR, WD, MOM))                    # eager warm-up 2, timed per launch
    torch.cuda.synchronize()
    timed = _lib.timed_results()
    kernels = _kernel_rates(timed)
    _lib.time_entry_point(None)
    for _ in range(warmup):                              # warm-up 3, then capture + replays
        float(step(imgs, 1, LR, WD, MOM))
    last = [0.0]

    def one():
        last[0] = float(step(imgs, 1, LR, WD, MOM))      # loss.item() every step (main_esvit.py:546)
    ms = _timed(one, steps)
    res = {"ms_per_step": round(ms, 2), "images_per_s": round(B / ms * 1e3, 1), "last_loss": last[0],
           "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "kernels": kernels}
    if arch != "cvt_13":
        res["attention_by_L"] = _attention_by_L(timed)
    del step, student, teacher, loss
    return res


class _ReferenceStep:
    """main_esvit.py:280-301 (CvT student / teacher with DINOHeads) and :541-590 (autocast bf16 forward + loss,
    loss.item(), backward, clip_gradients, cancel_gradients_last_layer, AdamW step, EMA) on the unmodified modules."""

    def __init__(self, spec: dict, drop_path_rate: float):
        from oracle import reference_import as RI
        import torch.distributed as dist
        ns = RI.load()
        if not dist.is_initialized():  # the reference losses all-reduce unconditionally (main_esvit.py:656)
            import socket
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            with socket.socket() as sk:
                sk.bind(("127.0.0.1", 0))
                os.environ.setdefault("MASTER_PORT", str(sk.getsockname()[1]))
            dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", torch.cuda.current_device()))
        from models import cvt_v4_transformer as ref_cvt
        from functools import partial
        torch.manual_seed(0)

        def build(dpr):   # get_cls_model (:685-707) without the yacs config
            return ref_cvt.CvT(num_classes=0, act_layer=ref_cvt.QuickGELU, norm_layer=partial(ref_cvt.LayerNorm, eps=1e-5),
                               init="trunc_norm", use_dense_prediction=True, spec=dict(spec, DROP_PATH_RATE=dpr))
        self.student, self.teacher = build(drop_path_rate), build(0.0)
        for m in (self.student, self.teacher):   # main_esvit.py never calls .eval(): BatchNorm in train mode
            m.head = ns.DINOHead(spec["DIM_EMBED"][-1], K)
            m.head_dense = ns.DINOHead(spec["DIM_EMBED"][-1], K)
            m.cuda().train()
        self.teacher.load_state_dict(self.student.state_dict())
        for p in self.teacher.parameters():
            p.requires_grad = False
        self.loss = ns.DDINOLoss(K, NCROPS, 0.04, 0.04, 0, 100).cuda()
        self.opt = torch.optim.AdamW(ns.get_params_groups(self.student))
        self.ns = ns

    def step(self, images) -> float:
        for i, g in enumerate(self.opt.param_groups):
            g["lr"] = LR
            if i == 0:
                g["weight_decay"] = WD
        with torch.autocast("cuda", dtype=torch.bfloat16):
            t = self.teacher(images[:2])
            s = self.student(images)
            loss = self.loss(s, t, 1, None)
        lv = loss.item()
        if not math.isfinite(lv):
            raise RuntimeError(f"reference loss is {lv}")
        self.opt.zero_grad()
        loss.backward()
        self.ns.clip_gradients(self.student, 3.0)
        self.ns.cancel_gradients_last_layer(1, self.student, 1)
        self.opt.step()
        with torch.no_grad():
            for q, k in zip(self.student.parameters(), self.teacher.parameters()):
                k.data.mul_(MOM).add_((1 - MOM) * q.detach().data)
        torch.cuda.synchronize()
        return lv


def run_reference(arch: str, B: int, steps: int, warmup: int) -> dict:
    from esvit_b200.engine import CVT_SPECS
    ref = _ReferenceStep(CVT_SPECS[arch]["cvt_spec"], CVT_SPECS[arch]["drop_path_rate"])
    imgs = crops(B)
    for _ in range(warmup):
        ref.step(imgs)
    ms = _timed(lambda: ref.step(imgs), steps)
    return {"ms_per_step": round(ms, 2), "images_per_s": round(B / ms * 1e3, 1), "precision": "bf16 autocast"}


# arch -> the model and yaml spec named in the metric
SPEC_NAMES = {"cvt_13": "CvT-13 (s1)", "cvt_13_w14": "CvT-13 (win_size/s1)", "cvt_s3": "CvT (s3)",
              "cvt_s3_w14": "CvT (win_size/s3)"}


def largest_fitting(fn, batches):
    """fn(B) at the first batch of `batches` that does not run out of memory -> (B, result) or (None, reason)"""
    for B in batches:
        try:
            return B, fn(B)
        except torch.OutOfMemoryError:
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    return None, "out of memory at every batch tried"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", choices=tuple(SPEC_NAMES), default="cvt_13")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cvt.py measures on a CUDA device; none found")
    from oracle import reference_import as RI
    batches = [b for b in (args.batch, 48, 32, 16) if b <= args.batch]
    B, ours = largest_fitting(lambda b: run_ours(args.arch, b, args.steps, args.warmup), batches)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    if args.no_reference:
        ref = "not run (--no-reference)"
    elif not RI.available():
        ref = "not run (reference tree not installed under oracle/_ref/)"
    else:
        rb, r = largest_fitting(lambda b: run_reference(args.arch, b, args.steps, args.warmup), batches)
        ref = dict(r, batch=rb) if rb is not None else f"not run ({r})"
    line = {"metric": f"multi-crop images/sec, {SPEC_NAMES[args.arch]} pretrain step (2 global 224^2 + 8 local 96^2 crops, "
                      "DDINOLoss, K=65536)",
            "value": ours["images_per_s"] if B else None, "unit": "images/s", "batch": B,
            "steps": args.steps, "warmup": args.warmup, "ours": ours, "reference": ref, "gpu": gpu_info()}
    if B and isinstance(ref, dict):
        line["speedup_vs_reference"] = round(ours["images_per_s"] / ref["images_per_s"], 2)
    print(json.dumps(line))
    import torch.distributed as dist
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
