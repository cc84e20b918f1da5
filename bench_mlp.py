"""Swin MLP forward at the stage-0/1 shapes of the Swin-T 2 + 8-crop step (B = 64): the two-launch esvit_gemm_bf16 chain
(fc1 + GELU, then fc2) against the back-to-back esvit_mlp_fwd kernel, student (h and gelu' written for the backward)
and teacher (no gradient: y only).

Each case is timed with CUDA events over --iters launches after --warmup launches.  Algorithmic HBM bytes come from the
shapes (bf16 activations; the weights, 16 C^2 bytes, are included but negligible):
  chain   student 28 MC (x, h + gelu' written, h re-read, y)     teacher 20 MC (x, h written and re-read, y)
  fused   student 20 MC (x, h + gelu' written, y)                teacher  4 MC (x, y)
and the share of peak is those bytes over the time against 3.35 TB/s (H100 SXM HBM3 data sheet).  Prints one JSON line
per case and one with the card's name, power limit and maximum SM clock, read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
B = 64
# (stage, C, student tokens, teacher tokens): 2 x 224^2 + 8 x 96^2 crops for the student, the 2 global crops for the teacher
SHAPES = [
    (0, 96, B * (2 * 56 * 56 + 8 * 24 * 24), B * 2 * 56 * 56),
    (1, 192, B * (2 * 28 * 28 + 8 * 12 * 12), B * 2 * 28 * 28),
]


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    import torch
    d = {"device": torch.cuda.get_device_name(0)}
    if out:
        name, power, clk = (s.strip() for s in out[0].split(","))
        d.update(name=name, power_limit=power, clocks_max_sm=clk)
    return d


def bytes_of(M, C, fused, student):
    act = (20 if student else 4) if fused else (28 if student else 20)
    return act * M * C + 16 * C * C


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_mlp.py needs a CUDA device")
    from esvit_b200 import ops
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)

    for stage, C, m_student, m_teacher in SHAPES:
        torch.manual_seed(stage)
        w1 = (torch.randn(4 * C, C, device=dev) / C ** 0.5).to(torch.bfloat16)
        b1 = torch.randn(4 * C, device=dev) * 0.2
        w2 = (torch.randn(C, 4 * C, device=dev) / (4 * C) ** 0.5).to(torch.bfloat16)
        b2 = torch.randn(C, device=dev) * 0.2
        for student, M in ((True, m_student), (False, m_teacher)):
            x = (torch.randn(M, C, device=dev) * 0.5).to(torch.bfloat16)

            def chain():
                if student:
                    h, _ = ops.gemm(x, w1, b1, act=1, want_pre=True)
                else:
                    h = ops.gemm(x, w1, b1, act=1)
                return ops.gemm(h, w2, b2)

            def fused():
                return ops.mlp_fwd(x, w1, b1, w2, b2, want_h=student)

            same = None
            res = {}
            for name, fn in (("chain", chain), ("fused", fused)):
                for _ in range(args.warmup):
                    out = fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    out = fn()
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.iters
                nbytes = bytes_of(M, C, name == "fused", student)
                res[name] = {"ms": round(ms, 4), "GB": round(nbytes / 1e9, 4), "TBps": round(nbytes / ms / 1e9, 3),
                             "hbm_frac": round(nbytes / ms / 1e9 / (HBM_PEAK / 1e12), 3)}
                y = out[0] if isinstance(out, tuple) else out
                same = y if same is None else bool(torch.equal(same, y))
                del out, y
            print(json.dumps({"stage": stage, "C": C, "M": M, "mode": "student" if student else "teacher",
                              **{f"{k}_{n}": v for n, r in res.items() for k, v in r.items()},
                              "speedup": round(res["chain"]["ms"] / res["fused"]["ms"], 3), "y_equal": same}), flush=True)
            del x


if __name__ == "__main__":
    main()
