"""GEMM launches of one Swin-T W7 2 + 8-crop student step (K = 65 536, B = 64): every distinct (entry point, M, N, K,
operand majors, epilogue) the bench step runs through hg::gemm_kernel, replayed with CUDA events over --iters launches
after --warmup launches at every tile code (1128, 1256, 2128, 2256) and at the automatic choice (tile 0).

The cases are collected from one eager step of the bench workload (engine.make_step as bench.py builds it) with
_lib.time_entry_point on the GEMM entry points; their arguments are recorded, so the replay runs exactly the launches
of the step (inputs are seeded random tensors of the same shapes).  Algorithmic work, counted as bench.py counts it:
  bytes  bf16 GEMM 2 (MK + NK + MN (1 + gelu')); multiplier GEMM 2 (MK + NK + 2 MN); weight gradient 2 T (N + K) + 4 NK
  FLOPs  2 MNK (weight gradient: 2 T N K)
The bound is the larger of bytes / 3.35 TB/s and FLOPs / 989 TFLOP/s (H100 SXM data sheet); share = bound / time.
Prints one JSON line with the card's name, power limit and maximum SM clock (read in the same run), one per case,
library and tile, and per class (forward, input gradient, fc2-dgrad x GELU', weight gradient) the sums weighted by the
launches per step.

--lib PATH (repeatable) times other builds of libesvit_b200.so next to the tree's own, alternating per case in one
process, and compares their outputs at the automatic tile with the tree's (bf16 outputs bit for bit; column sums and
fp32 weight gradients to fp32 re-association).  --count-only prints the cases of bench_gemm_cases.json (the list a GPU
run collects; the run reports whether the step still launches exactly those) with their bytes and FLOPs, without a GPU."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
BF16_PEAK = 989e12
CASES_FILE = os.path.join(ROOT, "bench_gemm_cases.json")
TILES = [0, 1128, 1256, 2128, 2256]
GEMM_ENTRIES = ["esvit_gemm_bf16", "esvit_gemm_mul_colsum2", "esvit_gemm_wgrad"]
CLASSES = {"fwd": "forward Linears (bias / GELU + GELU')", "dgrad": "input gradients (MN-major B)",
           "mul": "fc2 input gradient x GELU' + fc1 bias gradient", "wgrad": "weight gradients (fp32 split-K + fold)"}


def _set(p):
    """a pointer argument that is not NULL (None or c_void_p(None) is NULL)"""
    return p is not None and getattr(p, "value", p) is not None


def case_of(name, a):
    """the launch's case: a dict of what determines the kernel and its work"""
    if name == "esvit_gemm_bf16":
        return {"kind": "dgrad" if int(a[9]) else "fwd", "M": int(a[5]), "N": int(a[6]), "K": int(a[7]), "a_mn": int(a[8]),
                "b_mn": int(a[9]), "act": int(a[10]), "bias": _set(a[2]),
                "pre": int(a[10]) != 0 and _set(a[4])}
    if name == "esvit_gemm_mul_colsum2":
        return {"kind": "mul", "M": int(a[6]), "N": int(a[7]), "K": int(a[8]), "b_mn": int(a[9])}
    if name == "esvit_gemm_wgrad":
        return {"kind": "wgrad", "T": int(a[4]), "N": int(a[5]), "K": int(a[6]), "accumulate": int(a[7])}
    raise KeyError(name)


def work(c):
    """(bytes, flops) of one launch"""
    if c["kind"] == "wgrad":
        return 2 * c["T"] * (c["N"] + c["K"]) + 4 * c["N"] * c["K"], 2.0 * c["T"] * c["N"] * c["K"]
    M, N, K = c["M"], c["N"], c["K"]
    outs = 2 if c["kind"] == "mul" or c.get("pre") else 1
    return 2 * (M * K + N * K + outs * M * N), 2.0 * M * N * K


def bound_ms(c):
    nbytes, flops = work(c)
    return max(nbytes / HBM_PEAK, flops / BF16_PEAK) * 1e3


def load_cases():
    with open(CASES_FILE) as f:
        return [(d["launches"], {k: v for k, v in d.items() if k != "launches"}) for d in json.load(f)["cases"]]


def collect(dev):
    """[(launches per step, case)] of one eager step of the bench workload"""
    import torch
    from bench import synthetic_crops
    from esvit_b200 import _lib, engine
    B, n_local = 64, 8
    lr = 5e-4 * B / 256.0
    step, student, teacher, _ = engine.make_step(arch="swin_tiny_w7", out_dim=65536, ncrops=2 + n_local, dense=True,
                                                 device=dev, lr=lr, ddp=False, optimizer="fused", cuda_graph=False)
    student.train()
    teacher.train()
    crops = [c.to(dev) for c in synthetic_crops(B, n_local, 0)]
    step(crops, 1, lr, 0.04, 0.996)  # lazy loading and workspace allocation stay out of the recorded step
    torch.cuda.synchronize()
    seen = []
    plain = _lib._plain_call

    def recording(name, *args):
        if name in GEMM_ENTRIES:
            seen.append(case_of(name, args))
        return plain(name, *args)

    _lib._plain_call = recording
    _lib.reset_counters()
    _lib.time_entry_point(GEMM_ENTRIES)
    try:
        step(crops, 1, lr, 0.04, 0.996)
        torch.cuda.synchronize()
    finally:
        _lib._plain_call = plain
        _lib.time_entry_point(None)
    in_step = Counter()
    for t in _lib.timed_results():
        in_step[t["name"]] += t["ms"]
    del step, student, teacher, crops
    torch.cuda.empty_cache()
    counts = Counter(json.dumps(c, sort_keys=True) for c in seen)
    return [(n, json.loads(k)) for k, n in sorted(counts.items())], dict(in_step)


class Replay:
    """inputs of one case and a launcher per (library, tile)"""

    def __init__(self, c, dev, seed):
        import torch
        self.c = c
        g = torch.Generator(device=dev).manual_seed(seed)
        rnd = lambda *s, scale=1.0: (torch.randn(*s, device=dev, generator=g) * scale).to(torch.bfloat16)
        bf = dict(dtype=torch.bfloat16, device=dev)
        if c["kind"] == "wgrad":
            T, N, K = c["T"], c["N"], c["K"]
            self.dy, self.x = rnd(T, N), rnd(T, K)
            self.dw = torch.zeros(N, K, dtype=torch.float32, device=dev)
            self.ws = None
        else:
            M, N, K = c["M"], c["N"], c["K"]
            self.a = rnd(K, M) if c.get("a_mn") else rnd(M, K)
            self.b = rnd(K, N, scale=K ** -0.5) if c["b_mn"] else rnd(N, K, scale=K ** -0.5)
            self.out = torch.empty(M, N, **bf)
            if c["kind"] == "mul":
                self.mult = rnd(M, N, scale=0.5)
                self.colsum = torch.zeros(N, dtype=torch.float32, device=dev)
                self.ws = torch.empty(160 * N, dtype=torch.float32, device=dev)
            else:
                self.bias = torch.randn(N, device=dev, generator=g) * 0.2 if c["bias"] else None
                self.pre = torch.empty(M, N, **bf) if c.get("pre") else None

    def prepare(self, lib):
        """wgrad: the split-K workspace for this library's sizing"""
        import torch
        c = self.c
        if c["kind"] == "wgrad" and self.ws is None:
            n = lib.esvit_gemm_wgrad_ws_floats(c["N"], c["K"])
            self.ws = torch.empty(n, dtype=torch.float32, device=self.dw.device)

    def run(self, lib, tile):
        P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(None)
        import torch
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        c = self.c
        if c["kind"] == "wgrad":
            return lib.esvit_gemm_wgrad(P(self.dy), P(self.x), P(self.dw), P(self.ws), c["T"], c["N"], c["K"],
                                        c["accumulate"], tile, s)
        if c["kind"] == "mul":
            return lib.esvit_gemm_mul_colsum2(P(self.a), P(self.b), P(self.mult), P(self.out), P(self.colsum), P(self.ws),
                                              c["M"], c["N"], c["K"], c["b_mn"], tile, s)
        return lib.esvit_gemm_bf16(P(self.a), P(self.b), P(self.bias), P(self.out), P(self.pre), c["M"], c["N"], c["K"],
                                   c["a_mn"], c["b_mn"], c["act"], tile, s)

    def outputs(self, lib, tile):
        """fresh outputs of one launch"""
        c = self.c
        if c["kind"] == "wgrad":
            self.dw.zero_()
        elif c["kind"] == "mul":
            self.colsum.zero_()
        rc = self.run(lib, tile)
        if rc != 0:
            raise RuntimeError(f"launch failed with status {rc}")
        if c["kind"] == "wgrad":
            return {"dw": self.dw.clone()}
        if c["kind"] == "mul":
            return {"out": self.out.clone(), "colsum": self.colsum.clone()}
        o = {"out": self.out.clone()}
        if self.pre is not None:
            o["pre"] = self.pre.clone()
        return o


def compare(ref, got):
    """bf16 tensors bit for bit; fp32 (column sums, weight gradients) to fp32 re-association"""
    import torch
    res = {}
    for k, r in ref.items():
        g = got[k]
        if r.dtype == torch.bfloat16:
            res[k] = bool(torch.equal(r, g))
        else:
            err = ((g.double() - r.double()).norm() / r.double().norm().clamp_min(1e-30)).item()
            # another tile shape or split count adds the fp32 partials in another order: over T = 696 320 tokens that
            # moves the result by ~2e-5 (rel. L2); the weight-gradient tests gate at 1e-4 against fp64
            res[k] = err < 1e-4
            res[k + "_rel_l2"] = float(f"{err:.3g}")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--lib", action="append", default=[], metavar="PATH",
                    help="another build of libesvit_b200.so to time next to the tree's (repeatable)")
    ap.add_argument("--tiles", default=",".join(map(str, TILES)), help="tile codes to time (0 = automatic)")
    ap.add_argument("--count-only", action="store_true", help="print the cases and their algorithmic work, run nothing")
    args = ap.parse_args()
    tiles = [int(t) for t in args.tiles.split(",")]

    if args.count_only:
        tot = Counter()
        for n, c in load_cases():
            nbytes, flops = work(c)
            tot[c["kind"], "GB"] += n * nbytes / 1e9
            tot[c["kind"], "GFLOP"] += n * flops / 1e9
            tot[c["kind"], "bound_ms"] += n * bound_ms(c)
            print(json.dumps({**c, "launches": n, "GB": round(nbytes / 1e9, 4), "GFLOP": round(flops / 1e9, 2),
                              "bound_ms": round(bound_ms(c), 4)}))
        for k in CLASSES:
            print(json.dumps({"per_step": k, "class": CLASSES[k], "GB": round(tot[k, "GB"], 3),
                              "GFLOP": round(tot[k, "GFLOP"], 1), "bound_ms": round(tot[k, "bound_ms"], 3)}))
        return

    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_gemm.py needs a CUDA device")
    from bench_mlp import card
    from esvit_b200 import _lib
    torch.cuda.set_device(0)
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)

    cases, in_step = collect(dev)
    committed = None
    if os.path.isfile(CASES_FILE):
        committed = sorted(json.dumps([n, c], sort_keys=True) for n, c in load_cases())
    found = sorted(json.dumps([n, c], sort_keys=True) for n, c in cases)
    print(json.dumps({"cases": [dict(c, launches=n) for n, c in cases], "matches_cases_file": committed == found,
                      "in_step_ms": {k: round(v, 3) for k, v in in_step.items()}}), flush=True)

    libs = [("tree", _lib.load())]
    for p in args.lib:
        lib = ctypes.CDLL(os.path.abspath(p))
        for name in ("esvit_gemm_bf16", "esvit_gemm_mul_colsum2", "esvit_gemm_wgrad", "esvit_gemm_wgrad_ws_floats"):
            getattr(lib, name).argtypes = _lib.SIGNATURES[name]
            getattr(lib, name).restype = ctypes.c_int
        libs.append((p, lib))

    totals = Counter()
    for idx, (n, c) in enumerate(cases):
        r = Replay(c, dev, seed=idx)
        for _, lib in libs:
            r.prepare(lib)
        if len(libs) > 1:
            ref = r.outputs(libs[0][1], 0)
            for tag, lib in libs[1:]:
                print(json.dumps({"compare": tag, "case": idx, **c, **compare(ref, r.outputs(lib, 0))}), flush=True)
            del ref
        nbytes, flops = work(c)
        for tile in tiles:
            for tag, lib in libs:
                for _ in range(args.warmup):
                    rc = r.run(lib, tile)
                    if rc != 0:
                        sys.exit(f"case {idx} tile {tile} failed with status {rc} ({tag})")
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    r.run(lib, tile)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.iters
                totals[tag, c["kind"], tile] += n * ms
                print(json.dumps({"lib": tag, "case": idx, **c, "launches": n, "tile": tile, "ms": round(ms, 4),
                                  "TBps": round(nbytes / ms / 1e9, 3), "TFLOPs": round(flops / ms / 1e9, 1),
                                  "share": round(bound_ms(c) / ms, 3)}), flush=True)
        del r
        torch.cuda.empty_cache()

    for tag, _ in libs:
        for k in CLASSES:
            sel = [(n, c) for n, c in cases if c["kind"] == k]
            nbytes = sum(n * work(c)[0] for n, c in sel)
            flops = sum(n * work(c)[1] for n, c in sel)
            bms = sum(n * bound_ms(c) for n, c in sel)
            for tile in tiles:
                ms = totals[tag, k, tile]
                if not ms:
                    continue
                print(json.dumps({"per_step": k, "class": CLASSES[k], "lib": tag, "tile": tile,
                                  "launches": sum(n for n, _ in sel), "ms": round(ms, 3),
                                  "TBps": round(nbytes / ms / 1e9, 3), "TFLOPs": round(flops / ms / 1e9, 1),
                                  "share": round(bms / ms, 3)}), flush=True)


if __name__ == "__main__":
    main()
