"""Throughput of the training step with BatchNorm DINO heads (``--use_bn_in_head True``) against plain heads, and the
head BatchNorm kernels' bandwidth.

    python bench_bnhead.py [--batch 64] [--local-crops 8] [--out-dim 65536] [--steps 20] [--warmup 5] [--rounds 3]

Swin-T W7, DDINOLoss (`head` and `head_dense`), 2 global 224^2 + 8 local 96^2 crops, CUDA-graph steps with the fused
optimiser.  Two step objects (plain heads / BN heads, same seed) run in alternating rounds of ``--steps`` replays each;
images/s per round and the median are printed.  The four head-BN entry points (esvit_headbn_*) are timed with CUDA
events over eager steps of the BN-head step; their bytes are computed from the shapes (bf16 [N, C] reads / writes:
fwd_stats 2NC, fwd_apply 4NC, bwd_stats 4NC, bwd_apply 6NC).  One JSON line on stdout; nothing is written to disk.
"""
from __future__ import annotations

import argparse
import json
import statistics
import time

import torch

from bench_mixup import HBM_TBPS, card

BYTES_PER_NC = {"esvit_headbn_fwd_stats": 2, "esvit_headbn_fwd_apply": 4, "esvit_headbn_bwd_stats": 4,
                "esvit_headbn_bwd_apply": 6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--local-crops", type=int, default=8)
    ap.add_argument("--out-dim", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bnhead.py needs a CUDA device"
    from esvit_b200 import _lib, engine

    dev = torch.device("cuda:0")
    B, K, ncrops = args.batch, args.out_dim, 2 + args.local_crops
    lr, wd, mom, epoch = 5e-4 * B / 256.0, 0.04, 0.996, 1
    steps = {}
    for name, hk in (("plain", None), ("bn", dict(use_bn=True))):
        steps[name] = engine.make_step(arch="swin_tiny_w7", out_dim=K, ncrops=ncrops, dense=True, device=dev, lr=lr,
                                       head_kwargs=hk, cuda_graph=True)[0]
    g = torch.Generator().manual_seed(0)
    crops = [torch.randn(B, 3, 224, 224, generator=g).to(dev) for _ in range(2)]
    crops += [torch.randn(B, 3, 96, 96, generator=g).to(dev) for _ in range(args.local_crops)]

    # BN kernels: CUDA events around each launch, in eager steps
    sb = steps["bn"]
    sb.use_cuda_graph = False
    sb.step(crops, epoch, lr, wd, mom)
    torch.cuda.synchronize()
    _lib.reset_counters()
    _lib.time_entry_point(tuple(BYTES_PER_NC))
    nrep = 5
    for _ in range(nrep):
        sb.step(crops, epoch, lr, wd, mom)
    torch.cuda.synchronize()
    calls = _lib.timed_results()
    _lib.time_entry_point(None)
    sb.use_cuda_graph = True
    k_ms = sum(c["ms"] for c in calls) / nrep
    k_bytes = sum(BYTES_PER_NC[c["name"]] * c["N"] * c["C"] for c in calls) / nrep
    per_entry = {n: round(sum(c["ms"] for c in calls if c["name"] == n) / nrep, 4) for n in BYTES_PER_NC}

    for _ in range(args.warmup):  # eager warm-up, capture, replays of each graph
        for s in steps.values():
            s.step(crops, epoch, lr, wd, mom)
    torch.cuda.synchronize()

    rates = {"plain": [], "bn": []}
    info = card()
    for _ in range(args.rounds):
        for name, s in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                l = s.step(crops, epoch, lr, wd, mom)
            torch.cuda.synchronize()
            rates[name].append(B * args.steps / (time.perf_counter() - t0))  # images (not crops), as bench.py counts
            assert torch.isfinite(l).item()
    info_after = card()

    plain, bn = statistics.median(rates["plain"]), statistics.median(rates["bn"])
    res = {
        "metric": "multi-crop images/sec, swin_tiny_w7 DDINO step with BatchNorm DINO heads vs plain heads",
        "batch": B, "ncrops": ncrops, "out_dim": K, "steps": args.steps, "rounds": args.rounds,
        "plain_images_per_s": round(plain, 1), "bn_images_per_s": round(bn, 1),
        "plain_rounds": [round(x, 1) for x in rates["plain"]], "bn_rounds": [round(x, 1) for x in rates["bn"]],
        "bn_over_plain": round(bn / plain, 4),
        "bn_kernels_ms_per_step": round(k_ms, 4), "bn_kernels_ms_by_entry": per_entry,
        "bn_kernels_bytes_per_step": int(k_bytes), "bn_kernels_tbps": round(k_bytes / (k_ms * 1e-3) / 1e12, 3),
        "bn_kernels_frac_of_hbm": round(k_bytes / (k_ms * 1e-3) / 1e12 / HBM_TBPS, 3),
        "bn_kernels_frac_of_step": round(k_ms * 1e-3 / (B / bn), 4),
        "gpu": info, "gpu_after": info_after,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
