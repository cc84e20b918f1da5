"""Throughput of the training step with ``--optimizer adamw | sgd | lars`` on the fused sweeps, and the sweeps' bandwidth.

    python bench_optim.py [--batch 64] [--local-crops 8] [--out-dim 65536] [--steps 20] [--warmup 5] [--rounds 3]
                          [--sweeps 50]

Swin-T W7, DDINOLoss (`head` and `head_dense`), 2 global 224^2 + 8 local 96^2 crops, CUDA-graph steps.  Three step
objects (FusedAdamWEMA, FusedSGDEMA, FusedSGDEMA(lars=True); same seed) run in alternating rounds of ``--steps``
replays each; images/s per round and the median are printed.

The optimiser entry points are timed with CUDA events around each launch, over ``--sweeps`` eager optimiser steps on the
Swin-T student / teacher parameter set (random gradients, every trainable tensor stepped).  Their bytes are computed
from numel and shadow presence: per stepped element the SGD sweep reads p, g, buf, k and writes p, buf, k (28 B) plus
2 B per bf16 shadow (student, teacher), the AdamW sweep 36 B plus shadows; a frozen element costs the EMA's p read and
k read / write (12 B) plus the teacher shadow; the sum-of-squares pass reads g (4 B), the LARS sums pass also reads p
of every trust-ratio tensor (8 B).  One JSON line on stdout; nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics
import time

import torch

from bench_mixup import HBM_TBPS, card

KINDS = ("adamw", "sgd", "lars")
SWEEP = {"adamw": "esvit_adamw_ema_multi", "sgd": "esvit_sgd_ema_multi", "lars": "esvit_sgd_ema_multi"}
SUMS = {"adamw": "esvit_grad_sumsq_multi", "sgd": "esvit_grad_sumsq_multi", "lars": "esvit_lars_sums_multi"}


def sweep_bytes(opt, kind: str) -> dict:
    """bytes one optimiser step moves, computed from numel and shadow presence (every trainable tensor stepped)"""
    per_step = 36 if kind == "adamw" else 28
    sweep = sums = 0
    for i, p in enumerate(opt.params):
        n = p.numel()
        sk = opt.shadow_k[i] is not None
        if opt.frozen[i]:
            sweep += n * (12 + 2 * sk)
            sums += 4 * n
            continue
        sweep += n * (per_step + 2 * (opt.shadow_p[i] is not None) + 2 * sk)
        sums += n * (8 if kind == "lars" and p.dim() != 1 else 4)
    return {"sweep": sweep, "sums": sums, "params": sum(p.numel() for p in opt.params)}


def time_sweeps(K: int, nsweeps: int, dev) -> dict:
    from esvit_b200 import _lib, engine
    from esvit_b200.optim import FusedAdamWEMA, FusedSGDEMA

    spec = engine.SWIN_SPECS["swin_tiny_w7"]
    torch.manual_seed(0)
    student = engine.build_network(spec, K, True).to(dev)
    teacher = engine.build_network(spec, K, True, is_teacher=True).to(dev)
    teacher.load_state_dict(student.state_dict())
    for p in teacher.parameters():
        p.requires_grad = False
    for p in student.parameters():
        if p.requires_grad:
            p.grad = torch.randn_like(p) * 1e-3
    out = {}
    for kind in KINDS:
        opt = (FusedAdamWEMA(student, teacher) if kind == "adamw"
               else FusedSGDEMA(student, teacher, lars=(kind == "lars")))
        opt.set_hyper(1e-8, 0.04, 0.9999)
        opt.set_skip_last_layer(False)
        for _ in range(3):
            opt.step()
        torch.cuda.synchronize()
        _lib.reset_counters()
        _lib.time_entry_point((SWEEP[kind], SUMS[kind]))
        for _ in range(nsweeps):
            opt.step()
        torch.cuda.synchronize()
        calls = _lib.timed_results()
        _lib.time_entry_point(None)
        b = sweep_bytes(opt, kind)
        ms = {part: statistics.median(c["ms"] for c in calls if c["name"] == name)
              for part, name in (("sweep", SWEEP[kind]), ("sums", SUMS[kind]))}
        ent = {"params": b["params"]}
        for part in ("sweep", "sums"):
            tbps = b[part] / (ms[part] * 1e-3) / 1e12
            ent.update({f"{part}_entry": (SWEEP if part == "sweep" else SUMS)[kind], f"{part}_ms": round(ms[part], 4),
                        f"{part}_bytes": b[part], f"{part}_bytes_per_param": round(b[part] / b["params"], 2),
                        f"{part}_tbps": round(tbps, 3), f"{part}_frac_of_hbm": round(tbps / HBM_TBPS, 3)})
        out[kind] = ent
        del opt
    for p in student.parameters():
        p.grad = None
    del student, teacher
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--local-crops", type=int, default=8)
    ap.add_argument("--out-dim", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweeps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim.py needs a CUDA device"
    from esvit_b200 import engine

    dev = torch.device("cuda:0")
    B, K, ncrops = args.batch, args.out_dim, 2 + args.local_crops
    info = card()
    sweeps = time_sweeps(K, args.sweeps, dev)

    lr, wd, mom, epoch = 5e-4 * B / 256.0, 0.04, 0.996, 1
    steps = {kind: engine.make_step(arch="swin_tiny_w7", out_dim=K, ncrops=ncrops, dense=True, device=dev, lr=lr,
                                    optimizer_type=kind, cuda_graph=True)[0] for kind in KINDS}
    g = torch.Generator().manual_seed(0)
    crops = [torch.randn(B, 3, 224, 224, generator=g).to(dev) for _ in range(2)]
    crops += [torch.randn(B, 3, 96, 96, generator=g).to(dev) for _ in range(args.local_crops)]
    for _ in range(args.warmup):  # eager warm-up, capture, replays of each graph
        for s in steps.values():
            s.step(crops, epoch, lr, wd, mom)
    torch.cuda.synchronize()

    rates = {k: [] for k in KINDS}
    for _ in range(args.rounds):
        for kind, s in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                l = s.step(crops, epoch, lr, wd, mom)
            torch.cuda.synchronize()
            rates[kind].append(B * args.steps / (time.perf_counter() - t0))  # images (not crops), as bench.py counts
            assert torch.isfinite(l).item()
    info_after = card()

    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {
        "metric": "multi-crop images/sec, swin_tiny_w7 DDINO step with the fused adamw / sgd / lars optimiser sweeps",
        "batch": B, "ncrops": ncrops, "out_dim": K, "steps": args.steps, "rounds": args.rounds,
        **{f"{k}_images_per_s": round(med[k], 1) for k in KINDS},
        **{f"{k}_rounds": [round(x, 1) for x in rates[k]] for k in KINDS},
        "sgd_over_adamw": round(med["sgd"] / med["adamw"], 4), "lars_over_adamw": round(med["lars"] / med["adamw"], 4),
        "sweeps": sweeps, "sweep_launches": args.sweeps,
        "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2),
        "gpu": info, "gpu_after": info_after,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
