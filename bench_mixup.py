"""Throughput of the mixup training step (``--use_mixup``) against the plain step, and the mixing kernel's bandwidth.

    python bench_mixup.py [--batch 64] [--local-crops 8] [--out-dim 65536] [--steps 20] [--warmup 5] [--rounds 3]

Swin-T W7, DINOLoss (the loss that reads the targets; DDINOLoss ignores them), 2 global 224^2 + 8 local 96^2 crops,
CUDA-graph steps with the fused optimiser.  The plain and the mixup step run on one model, in alternating rounds of
``--steps`` replays each; images/s per round and the median are printed.  The mixup step's student crops are timm-style
mixed crops (lambda x + (1 - lambda) x.flip(0)) on the first six views, with per-row-lambda, label-smoothed targets;
the last views get eye(B), as main_esvit.py does past ``num_mixup_views``.  The mixing kernel (esvit_mixup_q) is timed
with CUDA events over eager steps; its bytes are computed from the shapes: the 2B x K fp16 teacher rows read once,
the R x K fp16 mixed rows written, R = ncrops * B.  One JSON line on stdout; nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import time

import torch

HBM_TBPS = 3.35  # H100 SXM data sheet


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        f = [x.strip() for x in out.split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "sm_clock_mhz": float(f[2]), "sm_clock_max_mhz": float(f[3])}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_clock_mhz": None,
                "sm_clock_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--local-crops", type=int, default=8)
    ap.add_argument("--out-dim", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--mixup-views", type=int, default=6)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mixup.py needs a CUDA device"
    from esvit_b200 import _lib, engine
    from oracle import mixup as M

    dev = torch.device("cuda:0")
    B, K, ncrops = args.batch, args.out_dim, 2 + args.local_crops
    lr, wd, mom, epoch = 5e-4 * B / 256.0, 0.04, 0.996, 1
    step, student, teacher, loss_mod = engine.make_step(arch="swin_tiny_w7", out_dim=K, ncrops=ncrops, dense=False,
                                                        device=dev, lr=lr, cuda_graph=True)
    student.train()
    teacher.train()
    g = torch.Generator().manual_seed(0)
    crops = [torch.randn(B, 3, 224, 224, generator=g).to(dev) for _ in range(2)]
    crops += [torch.randn(B, 3, 96, 96, generator=g).to(dev) for _ in range(args.local_crops)]
    lam = [torch.rand(B, generator=g) for _ in range(ncrops)]
    mixed, targets = [], []
    for v, c in enumerate(crops):
        if v < args.mixup_views:
            lv = lam[v].to(dev).view(B, 1, 1, 1)
            mixed.append(c * lv + c.flip(0) * (1 - lv))
            targets.append(M.timm_mixup_target(B, lam[v], 0.1).to(dev))
        else:
            mixed.append(c)
            targets.append(torch.eye(B, device=dev))

    def plain():
        return step.step(crops, epoch, lr, wd, mom)

    def mix():
        return step.step(crops, epoch, lr, wd, mom, student_images=mixed, targets_mixup=targets)

    # mixing kernel: CUDA events around each launch, in eager steps
    step.use_cuda_graph = False
    mix()
    torch.cuda.synchronize()
    _lib.reset_counters()
    _lib.time_entry_point("esvit_mixup_q")
    for _ in range(5):
        mix()
    torch.cuda.synchronize()
    kt = [r["ms"] for r in _lib.timed_results()]
    _lib.time_entry_point(None)
    step.use_cuda_graph = True

    for _ in range(args.warmup):  # eager warm-up, capture, replays of each graph
        plain()
        mix()
    torch.cuda.synchronize()

    rates = {"plain": [], "mixup": []}
    info = card()
    for _ in range(args.rounds):
        for name, fn in (("plain", plain), ("mixup", mix)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                l = fn()
            torch.cuda.synchronize()
            rates[name].append(B * args.steps / (time.perf_counter() - t0))  # images (not crops), as bench.py counts
    assert torch.isfinite(l).item()
    info_after = card()

    R = ncrops * B
    nbytes = 2 * B * K * 2 + R * K * 2
    k_ms = statistics.median(kt)
    res = {
        "metric": "multi-crop images/sec, swin_tiny_w7 DINOLoss step with mixup targets vs the plain step",
        "batch": B, "ncrops": ncrops, "out_dim": K, "mixup_views": args.mixup_views, "steps": args.steps,
        "rounds": args.rounds,
        "plain_images_per_s": round(statistics.median(rates["plain"]), 1),
        "mixup_images_per_s": round(statistics.median(rates["mixup"]), 1),
        "plain_rounds": [round(x, 1) for x in rates["plain"]], "mixup_rounds": [round(x, 1) for x in rates["mixup"]],
        "mixup_over_plain": round(statistics.median(rates["mixup"]) / statistics.median(rates["plain"]), 4),
        "mix_kernel_ms": round(k_ms, 4), "mix_kernel_ms_all": [round(x, 4) for x in kt],
        "mix_kernel_bytes": nbytes, "mix_kernel_tbps": round(nbytes / (k_ms * 1e-3) / 1e12, 3),
        "mix_kernel_frac_of_hbm": round(nbytes / (k_ms * 1e-3) / 1e12 / HBM_TBPS, 3),
        "gpu": info, "gpu_after": info_after,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
