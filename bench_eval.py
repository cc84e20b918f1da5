"""Measure the evaluation entry points on one GPU and print one JSON line.

    python bench_eval.py probe   # forward_return_n_last_blocks(x, 4, False, depths), Swin-T W7, 224^2, B = 128
    python bench_eval.py knn     # knn_classifier on synthetic ImageNet-shaped features, k in {10, 20, 100, 200}
    python bench_eval.py attn    # forward_selfattention(x, n=2), Swin-T W7, 224^2, B = 1 and 64 (analyze_models.py)

probe: images/s of the CUDA path against the unmodified reference modules (oracle/_ref/, fp32, what eval_linear.py runs)
on the same GPU and the same seeded weights, with the rel-L2 difference of their outputs.

knn: seconds per knn_classifier call and its split into GEMM / select / vote (CUDA events around each launch); the
unmodified eval_knn.knn_classifier (AST-extracted from oracle/_ref/eval_knn.py, on the GPU as with --use_cuda) on the
first --ref-test-rows test rows, with the top-1 / top-5 agreement and neighbour disagreements on those rows; the largest
candidate count and the rerun rows; GEMM TFLOP/s against 989 (dense bf16) and select bytes/s against 3.35 TB/s, computed
from shapes.

attn: images/s of forward_selfattention(x, 2) against the unmodified reference modules (fp32, same seeded weights), the
rel-L2 and max-abs difference of every map, and the probability kernel's time per image (CUDA events around every
esvit_window_attn_probs launch) with its bytes/s against 3.35 TB/s; the bytes are the maps written plus the q/k rows read,
computed from shapes.

Writes nothing in the tree; card name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from functools import partial

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

PEAK_BF16_TFLOPS = 989.0   # H100 SXM data sheet, dense
PEAK_HBM_TBPS = 3.35


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:  # the query is informational; the torch device name is always there
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def _time(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / steps


def probe(args) -> dict:
    from esvit_b200.swin_transformer import SwinTransformer
    from oracle import golden as GD
    from oracle import reference_import as R
    from oracle import swin as S
    spec = dict(S.SWIN_T_W7)
    depths = list(spec["depths"])
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6), **spec)
    sd = GD.seeded_state_dict(GD.recipe(m.state_dict()), 0)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    x = torch.randn(args.batch, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
    res = {"mode": "probe", "arch": "swin_tiny_w7", "batch": args.batch, "n": 4}
    with torch.no_grad():
        t = _time(lambda: m.forward_return_n_last_blocks(x, 4, False, depths), args.steps, args.warmup)
        out = m.forward_return_n_last_blocks(x, 4, False, depths)
    res.update(esvit_b200={"s_per_batch": t, "images_per_s": args.batch / t}, width=out.shape[1])
    if R.available():
        ns = R.load()
        ref = ns.SwinTransformer(img_size=224, in_chans=3, num_classes=0, embed_dim=spec["embed_dim"], depths=depths,
                                 num_heads=list(spec["num_heads"]), window_size=spec["window_size"], drop_path_rate=0.0,
                                 norm_layer=partial(nn.LayerNorm, eps=1e-6))
        ref.load_state_dict(sd)
        ref = ref.cuda().eval()
        with torch.no_grad():
            tr = _time(lambda: ref.forward_return_n_last_blocks(x, 4, False, depths), args.steps, args.warmup)
            ro = ref.forward_return_n_last_blocks(x, 4, False, depths)
        res["reference_fp32"] = {"s_per_batch": tr, "images_per_s": args.batch / tr}
        res["speedup"] = tr / t
        res["rel_l2"] = float((out.double() - ro.double()).norm() / ro.double().norm())
    else:
        res["reference_fp32"] = "oracle/_ref not installed"
    return res


def attn(args) -> dict:
    from esvit_b200 import _lib
    from esvit_b200.swin_transformer import SwinTransformer
    from oracle import golden as GD
    from oracle import reference_import as R
    from oracle import swin as S
    spec = dict(S.SWIN_T_W7)
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6), **spec)
    sd = GD.seeded_state_dict(GD.recipe(m.state_dict()), 0)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    ref = None
    if R.available():
        ns = R.load()
        ref = ns.SwinTransformer(img_size=224, in_chans=3, num_classes=0, embed_dim=spec["embed_dim"],
                                 depths=list(spec["depths"]), num_heads=list(spec["num_heads"]),
                                 window_size=spec["window_size"], drop_path_rate=0.0,
                                 norm_layer=partial(nn.LayerNorm, eps=1e-6))
        ref.load_state_dict(sd)
        ref = ref.cuda().eval()
    res = {"mode": "attn", "arch": "swin_tiny_w7", "n": 2, "per_batch": {}}
    for B in [int(b) for b in args.batches.split(",")]:
        x = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(1)).cuda()
        with torch.no_grad():
            t = _time(lambda: m.forward_selfattention(x, 2), args.steps, args.warmup)
            _lib.reset_counters()
            _lib.time_entry_point("esvit_window_attn_probs")
            out = m.forward_selfattention(x, 2)
            torch.cuda.synchronize()
            _lib.time_entry_point(None)
            calls = _lib.timed_results()
        k_s = sum(c["ms"] for c in calls) / 1e3
        k_bytes = sum(c["windows"] * c["nH"] * c["ws"] ** 4 * 4 + c["tokens"] * 2 * c["C"] * 2 for c in calls)
        r = {"esvit_b200": {"s_per_batch": t, "images_per_s": B / t}, "maps": len(out),
             "map_bytes_per_image": sum(o.numel() * 4 for o in out) / B,
             "probs_kernel": {"launches": len(calls), "s_per_image": k_s / B, "bytes_per_image": k_bytes / B,
                              "tbps": k_bytes / k_s / 1e12, "share_of_3.35": k_bytes / k_s / 1e12 / PEAK_HBM_TBPS}}
        if ref is not None:
            with torch.no_grad():
                tr = _time(lambda: ref.forward_selfattention(x, 2), args.steps, args.warmup)
                ro = ref.forward_selfattention(x, 2)
            assert [o.shape for o in out] == [o.shape for o in ro]
            num = sum(float((a.double() - b.double()).norm() ** 2) for a, b in zip(out, ro))
            den = sum(float(b.double().norm() ** 2) for b in ro)
            r["reference_fp32"] = {"s_per_batch": tr, "images_per_s": B / tr}
            r["speedup"] = tr / t
            r["rel_l2"] = (num / den) ** 0.5
            r["max_abs"] = max(float((a - b).abs().max()) for a, b in zip(out, ro))
        else:
            r["reference_fp32"] = "oracle/_ref not installed"
        res["per_batch"][B] = r
        del out
    return res


def knn(args) -> dict:
    from esvit_b200 import _lib
    from esvit_b200 import knn as K
    from oracle import eval as E
    from oracle import reference_import as R
    N, M, D, C, T = args.train_rows, args.test_rows, args.dim, args.classes, args.temperature
    ks = [int(k) for k in args.ks.split(",")]
    xtr, ytr, xte, yte = E.clustered_features(args.seed, N, M, D, C, noise=args.noise, device="cuda")
    n_pad = -(-N // 8) * 8
    res = {"mode": "knn", "train_rows": N, "test_rows": M, "dim": D, "classes": C, "T": T}
    K.knn_classifier(xtr, ytr, xte[:256], yte[:256], max(ks), T, C)  # loads modules, warms every kernel
    names = ["esvit_knn_prep", "esvit_gemm_bf16", "esvit_knn_select", "esvit_knn_vote"]
    per_k = {}
    for k in ks:
        _lib.reset_counters()
        _lib.time_entry_point(names)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        top1, top5 = K.knn_classifier(xtr, ytr, xte, yte, k, T, C)
        wall = time.perf_counter() - t0
        _lib.time_entry_point(None)
        split = {n: 0.0 for n in names}
        for r in _lib.timed_results():
            split[r["name"]] += r["ms"] / 1e3
        gemm_flop = 2.0 * M * n_pad * D
        sel_bytes = 3.0 * M * N * 2  # the select's three passes over the bf16 similarities
        per_k[k] = {"s_per_call": wall, "top1": top1, "top5": top5, "split_s": split,
                    "max_candidates": K.last_stats["max_candidates"], "rerun_rows": K.last_stats["rerun_rows"],
                    "gemm_tflops": gemm_flop / split["esvit_gemm_bf16"] / 1e12,
                    "gemm_share_of_989": gemm_flop / split["esvit_gemm_bf16"] / 1e12 / PEAK_BF16_TFLOPS,
                    "select_tbps": sel_bytes / split["esvit_knn_select"] / 1e12,
                    "select_share_of_3.35": sel_bytes / split["esvit_knn_select"] / 1e12 / PEAK_HBM_TBPS}
    res["esvit_b200"] = per_k
    if R.available() and args.ref_test_rows > 0:
        ref = E.reference_knn_classifier()
        Mr = min(M, args.ref_test_rows)
        sub, ysub = xte[:Mr], yte[:Mr]
        kmax = max(ks)
        ref_idx = torch.cat([torch.mm(sub[i:i + 64], xtr.t()).topk(kmax, largest=True, sorted=True)[1]
                             for i in range(0, Mr, 64)])
        ref_vals = torch.cat([torch.mm(sub[i:i + 64], xtr.t()).topk(kmax, largest=True, sorted=True)[0]
                              for i in range(0, Mr, 64)])
        our_sims, our_idx = K.knn_topk(xtr, sub, kmax)
        rk = {}
        for k in ks:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r1, r5 = ref(xtr, ytr, sub, ysub, k, T, C)
            torch.cuda.synchronize()
            tr = time.perf_counter() - t0
            o1, o5 = K.knn_classifier(xtr, ytr, sub, ysub, k, T, C)
            rk[k] = {"s_per_call": tr, "top1": r1, "top5": r5, "esvit_b200_top1": o1, "esvit_b200_top5": o5,
                     "agree": (r1, r5) == (o1, o5),
                     "neighbour_disagreements": int((our_idx[:, :k] != ref_idx[:, :k]).sum()),
                     # largest difference of the k sorted similarities: summation-order noise when the neighbour
                     # disagreements are swaps of near-equal values
                     "max_sim_diff": float((our_sims[:, :k] - ref_vals[:, :k]).abs().max()),
                     "esvit_b200_s_per_test_row": per_k[k]["s_per_call"] / M, "reference_s_per_test_row": tr / Mr}
        res["reference_fp32"] = {"test_rows": Mr, "per_k": rk}
    else:
        res["reference_fp32"] = "oracle/_ref not installed" if not R.available() else "skipped"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["probe", "knn", "attn"])
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--batches", default="1,64", help="attn: batch sizes")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--train-rows", type=int, default=1281167)
    ap.add_argument("--test-rows", type=int, default=50000)
    ap.add_argument("--ref-test-rows", type=int, default=50000, help="test rows the fp32 reference runs on (>= 100)")
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--ks", default="10,20,100,200")
    ap.add_argument("--temperature", type=float, default=0.07)
    ap.add_argument("--noise", type=float, default=5.0)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_eval.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False  # the reference arms run fp32
    before = card()
    res = {"probe": probe, "knn": knn, "attn": attn}[args.mode](args)
    res["card"] = before
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
