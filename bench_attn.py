"""ws-7 window-attention core at the launches of one Swin-T W7 2 + 8-crop student step (B = 64): every (stage, crop
size, shift) geometry the step runs, forward (esvit_window_attn_fwd) and backward (esvit_window_attn_bwd), each timed
with CUDA events over --iters launches after --warmup launches.

Algorithmic work comes from the shapes, counted as bench.py counts it:
  bytes  backward 16·tokens·C (qkv 6C + dO 2C + O 2C read, dqkv 6C written), forward 8·tokens·C
  FLOPs  windows·nH·2·2·64²·32 for the forward (QKᵀ + PV over the 64 padded slots), 2.5x that for the backward
The share of peak is bytes over time against 3.35 TB/s (H100 SXM HBM3 data sheet).  Prints one JSON line with the card's
name, power limit and maximum SM clock (read in the same run), one per case, and one per-step total per library and
direction (each geometry times the number of blocks that launch it).

--lib PATH (repeatable) times other builds of libesvit_b200.so next to the tree's own, alternating per case in one
process; --dbg also times every case with ESVIT_ATTN_DBG=2 (gathers only, arithmetic and stores skipped)."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
B = 64
HD = 32
# (stage, C, global map, local map, [(shift, blocks of the step with that shift)]); 2 global + 8 local crops per image.
# Stage 3's global map is one window, so both of its blocks run unshifted.
STAGES = [
    (0, 96, 56, 24, [(0, 1), (3, 1)]),
    (1, 192, 28, 12, [(0, 1), (3, 1)]),
    (2, 384, 14, 6, [(0, 3), (3, 3)]),
    (3, 768, 7, 3, [(0, 2)]),
]


def cases():
    """[(stage, C, maps, side, shift, blocks)]: one entry per distinct launch geometry of the step"""
    out = []
    for stage, C, g, l, shifts in STAGES:
        for shift, blocks in shifts:
            out.append((stage, C, 2 * B, g, shift, blocks))
            out.append((stage, C, 8 * B, l, shift, blocks))
    return out


def work(C, maps, side, backward):
    """(tokens, windows, bytes, flops) of one launch"""
    tokens = maps * side * side
    windows = maps * (-(-side // 7)) ** 2
    nbytes = (16 if backward else 8) * tokens * C
    flops = (2.5 if backward else 1.0) * windows * (C // HD) * 2 * 2 * 64 ** 2 * 32
    return tokens, windows, nbytes, flops


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--lib", action="append", default=[], metavar="PATH",
                    help="another build of libesvit_b200.so to time next to the tree's (repeatable)")
    ap.add_argument("--dbg", action="store_true", help="also time every case with ESVIT_ATTN_DBG=2")
    ap.add_argument("--count-only", action="store_true", help="print the cases and their algorithmic work, run nothing")
    args = ap.parse_args()

    if args.count_only:
        tot = {"fwd": [0, 0.0], "bwd": [0, 0.0]}
        for stage, C, maps, side, shift, blocks in cases():
            for d in ("fwd", "bwd"):
                tokens, windows, nbytes, flops = work(C, maps, side, d == "bwd")
                tot[d][0] += blocks * nbytes
                tot[d][1] += blocks * flops
                print(json.dumps({"stage": stage, "C": C, "maps": maps, "map": side, "shift": shift, "blocks": blocks,
                                  "dir": d, "tokens": tokens, "windows": windows, "items": windows * (C // HD),
                                  "GB": round(nbytes / 1e9, 4), "GFLOP": round(flops / 1e9, 2)}))
        print(json.dumps({"per_step": {d: {"GB": round(v[0] / 1e9, 3), "GFLOP": round(v[1] / 1e9, 1)} for d, v in tot.items()}}))
        return

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_attn.py needs a CUDA device")
    from bench_mlp import card
    from esvit_b200 import _lib
    from esvit_b200.ops import ATTN_WS_FLOATS
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)

    libs = [("tree", _lib.load())]
    for p in args.lib:
        lib = ctypes.CDLL(os.path.abspath(p))
        for name in ("esvit_window_attn_fwd", "esvit_window_attn_bwd"):
            getattr(lib, name).argtypes = _lib.SIGNATURES[name]
            getattr(lib, name).restype = ctypes.c_int
        libs.append((p, lib))
    modes = [None, "2"] if args.dbg else [None]
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    totals = {}

    for stage, C, maps, side, shift, blocks in cases():
        nH = C // HD
        scale = HD ** -0.5
        tokens, windows, _, _ = work(C, maps, side, True)
        torch.manual_seed(stage * 10 + shift)
        qkv = torch.randn(tokens, 3 * C, device=dev).to(torch.bfloat16)
        qb = (torch.randn(3 * C, device=dev) * 0.2).to(torch.bfloat16)
        table = torch.randn(169, nH, device=dev) * 0.5
        dout = torch.randn(tokens, C, device=dev).to(torch.bfloat16)
        out = torch.empty(tokens, C, dtype=torch.bfloat16, device=dev)
        lse = torch.empty(windows * nH * 49, dtype=torch.float32, device=dev)
        dqkv = torch.empty_like(qkv)
        dtable = torch.zeros_like(table)
        dqb = torch.zeros(3 * C, dtype=torch.float32, device=dev)
        bws = torch.empty(nH * ATTN_WS_FLOATS, dtype=torch.float32, device=dev)
        _lib.call("esvit_window_attn_expand_bias", P(table), P(bws), nH, 7, stream())

        def fwd(lib):
            return lib.esvit_window_attn_fwd(P(qkv), P(qb), P(table), P(bws), 1, P(out), P(lse), maps, side, side, C, nH, 7,
                                             shift, scale, stream())

        def bwd(lib):
            return lib.esvit_window_attn_bwd(P(qkv), P(qb), P(table), P(bws), 1, P(out), P(dout), P(lse), P(dqkv), P(dtable),
                                             P(dqb), maps, side, side, C, nH, 7, shift, scale, stream())

        for d, fn in (("fwd", fwd), ("bwd", bwd)):
            _, _, nbytes, flops = work(C, maps, side, d == "bwd")
            for dbg in modes:
                if dbg is None:
                    os.environ.pop("ESVIT_ATTN_DBG", None)
                else:
                    os.environ["ESVIT_ATTN_DBG"] = dbg
                for tag, lib in libs:
                    for _ in range(args.warmup):
                        rc = fn(lib)
                        if rc != 0:
                            sys.exit(f"{d} failed with status {rc} ({tag})")
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        fn(lib)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / args.iters
                    key = (tag, d, dbg or "0")
                    totals[key] = totals.get(key, 0.0) + blocks * ms
                    print(json.dumps({"lib": tag, "dir": d, "dbg": dbg or "0", "stage": stage, "C": C, "maps": maps,
                                      "map": side, "shift": shift, "blocks": blocks, "ms": round(ms, 4),
                                      "GB": round(nbytes / 1e9, 4), "GBps": round(nbytes / ms / 1e6, 1),
                                      "hbm_frac": round(nbytes / ms / 1e9 / (HBM_PEAK / 1e12), 3),
                                      "tflops": round(flops / ms / 1e9, 1)}), flush=True)
            os.environ.pop("ESVIT_ATTN_DBG", None)
            if d == "fwd":
                fn(libs[0][1])  # leave out / lse as the un-debugged forward wrote them for the backward cases
        del qkv, dout, out, lse, dqkv

    step_bytes = {d: sum(blocks * work(C, maps, side, d == "bwd")[2] for _, C, maps, side, _, blocks in cases())
                  for d in ("fwd", "bwd")}
    for (tag, d, dbg), ms in totals.items():
        print(json.dumps({"per_step": True, "lib": tag, "dir": d, "dbg": dbg, "ms": round(ms, 3),
                          "GB": round(step_bytes[d] / 1e9, 3),
                          "hbm_frac": round(step_bytes[d] / ms / 1e9 / (HBM_PEAK / 1e12), 3)}), flush=True)


if __name__ == "__main__":
    main()
