"""Device multi-crop augmentation (esvit_b200.augment, csrc/augment.cu) on one GPU; prints one JSON line.

    python bench_augment.py [--steps 20] [--warmup 3] [--step-iters 10]

* `device`: images/s of MultiCropAugment (2 x 224^2 + 8 x 96^2 crops per image) at B = 64 and 128 from pinned collated
  batches, host -> device copy included, on a seeded mix of 500x375, 375x500, 800x600 and 1600x1200 sources (ImageNet's
  mean size plus larger photos); per-kernel times from the _lib entry-point timers, with bytes counted from shapes (box
  reads and the uint8 intermediate of the horizontal pass, its re-read, the fp32 writes) against 3.35 TB/s.
* `host_per_image_ms`: the work that stays on DataLoader workers (JPEG decode + convert('RGB'), parameter sampling,
  collate), one thread.
* `reference_per_core`: the unmodified DataAugmentationDINO (oracle/_ref/, AST-extracted) on the same decoded images,
  one thread, when build() installed the reference.
* `swin_t_step`: images/s of the Swin-T 2 + 8-crop DDINO step (bench.py's configuration, B = 64) with the augmentation
  inside the timed loop against the step alone, alternating in one session.
Card name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import io
import json
import random
import subprocess
import time

import numpy as np
import torch
from PIL import Image

from esvit_b200 import _lib
from esvit_b200 import augment as AG
from oracle import augment as A

PEAK_HBM_TBPS = 3.35
SHAPES = [(375, 500), (500, 375), (600, 800), (1200, 1600)]  # (H, W)
KERNELS = ["esvit_augment_coeffs", "esvit_augment_resize_h", "esvit_augment_color"]


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def sources(n: int, seed: int = 0):
    rng = np.random.default_rng(seed)
    return [A.synthetic_image(int(rng.integers(1 << 30)), *SHAPES[i % len(SHAPES)]) for i in range(n)]


def algorithmic_bytes(batch, sizes) -> dict:
    B = batch.index.shape[0]
    p = batch.params.transpose(0, 1).reshape(-1, AG.NPARAM)
    S = torch.tensor(sizes, dtype=torch.float64).repeat_interleave(B)
    h, w = p[:, 2], p[:, 3]
    return {"esvit_augment_resize_h": float((h * w * 3 + h * S * 3).sum()),
            "esvit_augment_color": float((h * S * 3 + 3 * S * S * 4).sum())}


def device_rate(images, B: int, steps: int, warmup: int) -> dict:
    t = AG.MultiCropParams((0.4, 1.0), (0.05, 0.4), (8,), (96,))
    aug = AG.MultiCropAugment()
    batches = []
    for k in range(4):
        imgs = [images[(k * B + i) % len(images)] for i in range(B)]
        items = [((torch.from_numpy(im), t.sample(*im.shape[:2])), 0) for im in imgs]
        batches.append(AG.collate_multicrop(items, pin_memory=True)[0])
    out = aug(batches[0])
    for i in range(warmup):
        aug(batches[i % 4], out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        aug(batches[i % 4], out=out)
    e1.record()
    torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3 / steps
    # one more pass per batch with the entry points bracketed by events
    _lib.reset_counters()
    _lib.time_entry_point(KERNELS)
    for b in batches:
        aug(b, out=out)
    torch.cuda.synchronize()
    _lib.time_entry_point(None)
    ms = {k: 0.0 for k in KERNELS}
    for r in _lib.timed_results():
        ms[r["name"]] += r["ms"]
    nbytes = {k: 0.0 for k in KERNELS}
    for b in batches:
        for k, v in algorithmic_bytes(b, t.sizes).items():
            nbytes[k] += v
    kern = {}
    for k in KERNELS:
        d = {"ms_per_batch": round(ms[k] / len(batches), 3)}
        if k in algorithmic_bytes(batches[0], t.sizes):
            tbps = nbytes[k] / (ms[k] / 1e3) / 1e12
            d.update(bytes_per_batch=nbytes[k] / len(batches), tb_per_s=round(tbps, 3),
                     share_of_3_35=round(tbps / PEAK_HBM_TBPS, 3))
        kern[k] = d
    src_mb = float(sum(b.pixels.numel() for b in batches)) / len(batches) / 1e6
    return {"B": B, "ms_per_batch": round(s * 1e3, 3), "images_per_s": round(B / s, 1),
            "source_mb_per_batch": round(src_mb, 1), "kernels": kern}


def host_cost(images, n: int) -> dict:
    torch.set_num_threads(1)
    jpegs = []
    for im in images[:n]:
        buf = io.BytesIO()
        Image.fromarray(im).save(buf, "JPEG", quality=90)
        jpegs.append(buf.getvalue())
    t = AG.MultiCropParams((0.4, 1.0), (0.05, 0.4), (8,), (96,))
    t0 = time.perf_counter()
    items = [(t(Image.open(io.BytesIO(j)).convert("RGB")), 0) for j in jpegs]
    t1 = time.perf_counter()
    AG.collate_multicrop(items)
    t2 = time.perf_counter()
    res = {"images": n, "decode_and_sample_ms": round((t1 - t0) / n * 1e3, 3),
           "collate_ms": round((t2 - t1) / n * 1e3, 3), "total_ms": round((t2 - t0) / n * 1e3, 3)}
    from oracle import reference_import as R
    if R.available():
        ref = A.reference_transform(R.REF_ROOT)
        pils = [Image.open(io.BytesIO(j)).convert("RGB") for j in jpegs]
        ref(pils[0])
        t0 = time.perf_counter()
        for p in pils:
            ref(p)
        s = (time.perf_counter() - t0) / n
        res["reference_per_core"] = {"ms_per_image": round(s * 1e3, 2), "images_per_s": round(1 / s, 1),
                                     "note": "DataAugmentationDINO (2 + 8 crops) on decoded images, one thread"}
    else:
        res["reference_per_core"] = "oracle/_ref not installed"
    torch.set_num_threads(max(1, torch.get_num_threads()))
    return res


def swin_step(images, iters: int, rounds: int) -> dict:
    from esvit_b200 import engine
    B = 64
    t = AG.MultiCropParams((0.4, 1.0), (0.05, 0.4), (8,), (96,))
    aug = AG.MultiCropAugment()
    batches = []
    for k in range(2):
        items = [((torch.from_numpy(images[(k * B + i) % len(images)]),
                   t.sample(*images[(k * B + i) % len(images)].shape[:2])), 0) for i in range(B)]
        batches.append(AG.collate_multicrop(items, pin_memory=True)[0])
    step, student, teacher, _ = engine.make_step(out_dim=65536, ncrops=10, dense=True, lr=5e-4 * B / 256,
                                                 cuda_graph=True)
    crops = aug(batches[0])
    wd, mom = 0.04, 0.996
    for _ in range(3):
        float(step(crops, 1, 5e-4, wd, mom))

    def timed(with_aug: bool) -> float:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(iters):
            if with_aug:
                aug(batches[i % 2], out=crops)
            float(step(crops, 1, 5e-4, wd, mom))  # loss read back every step, as main_esvit.py does
        torch.cuda.synchronize()
        return B * iters / (time.perf_counter() - t0)

    alone, with_aug = [], []
    for _ in range(rounds):
        alone.append(timed(False))
        with_aug.append(timed(True))
    return {"B": B, "step_alone_images_per_s": [round(v, 1) for v in alone],
            "step_with_augment_images_per_s": [round(v, 1) for v in with_aug],
            "median_ratio": round(float(np.median(with_aug) / np.median(alone)), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--step-iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-images", type=int, default=40)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_augment.py measures on a CUDA device"
    random.seed(0)
    torch.manual_seed(0)
    images = sources(64)
    res = {"metric": "device multi-crop augmentation, images/s (2 x 224^2 + 8 x 96^2 crops)", "card": card()}
    res["device"] = [device_rate(images, B, args.steps, args.warmup) for B in (64, 128)]
    res["host_per_image_ms"] = host_cost(images, args.host_images)
    res["swin_t_step"] = swin_step(images, args.step_iters, args.rounds)
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
