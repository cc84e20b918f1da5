"""Vision Longformer (vil_2262) pre-training step on one GPU: 2 x 224^2 + 8 x 96^2 crops, DDINOLoss (dense), K = 65 536.

    python bench_vil.py [--batch 64] [--steps 10] [--warmup 3] [--no-reference]

Prints one JSON line:
  * `value`: images/s (batch / step time, as bench.py counts them) of esvit_b200's captured step
    (engine.make_step("vil_2262"), CUDA graph, loss read back every step as train_one_epoch does) at the largest batch of
    --batch, 48, 32, 16 that fits, reported as `batch`;
  * `reference`: the UNMODIFIED reference modules (models.vision_longformer.MsViT built as get_cls_model builds it for
    vil_2262, DINOHead, DDINOLoss from oracle/_ref/, installed by build()) through main_esvit.py:541-590's statement
    sequence under bf16 autocast (bench_cvt._ReferenceStep.step), student and teacher in train mode, at the largest batch
    that fits; "not run" with the reason when the tree is absent or nothing fits;
  * `kernels`: CUDA-event times per step of the ViL attention and assembly entry points from one eager step, with their
    algorithmic bytes and FLOPs (from shapes), achieved TB/s and TFLOP/s, and share of the bound the data sheet gives (the
    larger of FLOPs / 989 TFLOP/s dense bf16 and bytes / 3.35 TB/s);
  * `gpu`: card name, power limit and maximum SM clock, read in the same run.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_cvt as BC  # noqa: E402
from bench_cvt import K, LR, MOM, PEAK_TBS, PEAK_TFLOPS, WD, _timed, crops, gpu_info, largest_fitting  # noqa: E402

NAMES = ("esvit_vil_sc_fwd", "esvit_vil_sc_bwd", "esvit_vil_dense_fwd", "esvit_vil_dense_bwd", "esvit_vil_im2col",
         "esvit_vil_col2im", "esvit_vil_bias_spmv")


def _cost(r) -> tuple:
    """(algorithmic bytes, FLOPs) of one call, from its shapes"""
    n = r["name"]
    if n.startswith("esvit_vil_dense"):
        B, L, C, nH = r["B"], r["L"], r["C"], r["nH"]
        flops = 4.0 * B * L * L * C                      # S = QK^T and O = PV
        io = B * L * 3 * C * 2 + B * L * C * 2 + nH * L * L * 4 + B * nH * L * 4
        if n.endswith("fwd"):
            return io, flops
        # qkv, out, dout in; dqkv out; bias read twice; dS partials written and summed
        parts = min(B, 16)
        return io + B * L * C * 2 + B * L * 3 * C * 2 + nH * L * L * 4 * (2 * parts + 1), 2.5 * flops
    if n.startswith("esvit_vil_sc"):
        B, nx, ny, nH = r["B"], r["nx"], r["ny"], r["nH"]
        N, C = 1 + nx * ny, 32 * nH
        keys = 1 + 2 * 49                                # training modes 1..8: own chunk + one neighbour + global
        flops = 4.0 * B * nx * ny * keys * C + 4.0 * B * N * C
        io = B * N * C * 2 * 2 + B * N * 2 * C * 2
        if n.endswith("fwd"):
            return io, flops
        return 2 * io + B * N * 3 * C * 2, 2.5 * flops
    return 0, 0.0


def _kernel_rates(res) -> dict:
    out = {}
    for name in NAMES:
        rows = [r for r in res if r["name"] == name]
        if not rows:
            continue
        ms = sum(r["ms"] for r in rows)
        nbytes = sum(_cost(r)[0] for r in rows)
        flops = sum(_cost(r)[1] for r in rows)
        d = {"ms_per_step": round(ms, 3), "launches": len(rows)}
        if nbytes:
            bound_ms = max(flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBS * 1e12)) * 1e3
            d.update({"gb": round(nbytes / 1e9, 3), "gflop": round(flops / 1e9, 1),
                      "tb_s": round(nbytes / ms / 1e9, 3), "tflops": round(flops / ms / 1e9, 1),
                      "share_of_bound": round(bound_ms / ms, 3),
                      "bound": "tensor" if flops / PEAK_TFLOPS > nbytes / PEAK_TBS else "hbm"})
        out[name] = d
    return out


def run_ours(B: int, steps: int, warmup: int) -> dict:
    from esvit_b200 import _lib, engine
    step, student, teacher, loss = engine.make_step("vil_2262", out_dim=K, cuda_graph=True)
    imgs = crops(B)
    float(step(imgs, 1, LR, WD, MOM))                    # eager warm-up 1 (module loads, allocator, bias plans)
    _lib.reset_counters()
    _lib.time_entry_point(list(NAMES))
    float(step(imgs, 1, LR, WD, MOM))                    # eager warm-up 2, timed per launch
    torch.cuda.synchronize()
    kernels = _kernel_rates(_lib.timed_results())
    _lib.time_entry_point(None)
    for _ in range(warmup):                              # warm-up 3, then capture + replays
        float(step(imgs, 1, LR, WD, MOM))
    last = [0.0]

    def one():
        last[0] = float(step(imgs, 1, LR, WD, MOM))      # loss.item() every step (main_esvit.py:546)
    ms = _timed(one, steps)
    res = {"ms_per_step": round(ms, 2), "images_per_s": round(B / ms * 1e3, 1), "last_loss": last[0],
           "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), "kernels": kernels}
    del step, student, teacher, loss
    return res


class _ReferenceStep(BC._ReferenceStep):
    """main_esvit.py:257-276 (MsViT student / teacher with DINOHeads on out_planes) and :541-590 (the step of
    bench_cvt._ReferenceStep) on the unmodified modules"""

    def __init__(self):
        from oracle import reference_import as RI
        ns = RI.load()
        import torch.distributed as dist
        if not dist.is_initialized():  # the reference losses all-reduce unconditionally (main_esvit.py:656)
            import socket
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            with socket.socket() as sk:
                sk.bind(("127.0.0.1", 0))
                os.environ.setdefault("MASTER_PORT", str(sk.getsockname()[1]))
            dist.init_process_group("nccl", rank=0, world_size=1,
                                    device_id=torch.device("cuda", torch.cuda.current_device()))
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            from models import vision_longformer as ref_vil
        from esvit_b200.vision_longformer import VIL_2262
        torch.manual_seed(0)
        self.student = ref_vil.MsViT(num_classes=0, use_dense_prediction=True, **dict(VIL_2262, drop_path_rate=0.1))
        self.teacher = ref_vil.MsViT(num_classes=0, use_dense_prediction=True, **dict(VIL_2262, drop_path_rate=0.0))
        for m in (self.student, self.teacher):            # main_esvit.py never calls .eval()
            m.head = ns.DINOHead(m.out_planes, K)
            m.head_dense = ns.DINOHead(m.out_planes, K)
            m.cuda().train()
        self.teacher.load_state_dict(self.student.state_dict())
        for p in self.teacher.parameters():
            p.requires_grad = False
        self.loss = ns.DDINOLoss(K, BC.NCROPS, 0.04, 0.04, 0, 100).cuda()
        self.opt = torch.optim.AdamW(ns.get_params_groups(self.student))
        self.ns = ns


def run_reference(B: int, steps: int, warmup: int) -> dict:
    ref = _ReferenceStep()
    imgs = crops(B)
    for _ in range(warmup):
        ref.step(imgs)
    ms = _timed(lambda: ref.step(imgs), steps)
    return {"ms_per_step": round(ms, 2), "images_per_s": round(B / ms * 1e3, 1), "precision": "bf16 autocast"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_vil.py measures on a CUDA device; none found")
    from oracle import reference_import as RI
    batches = [b for b in (args.batch, 48, 32, 16) if b <= args.batch]
    B, ours = largest_fitting(lambda b: run_ours(b, args.steps, args.warmup), batches)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    if args.no_reference:
        ref = "not run (--no-reference)"
    elif not RI.available():
        ref = "not run (reference tree not installed under oracle/_ref/)"
    else:
        rb, r = largest_fitting(lambda b: run_reference(b, args.steps, args.warmup), batches)
        ref = dict(r, batch=rb) if rb is not None else f"not run ({r})"
    line = {"metric": "multi-crop images/sec, ViL vil_2262 pretrain step (2 global 224^2 + 8 local 96^2 crops, "
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
