"""Write tests/golden/esvit_eval_augment.pt from the UNMODIFIED reference evaluation transforms (CPU, Pillow).

    python -m oracle.make_golden_eval_augment

The transforms are eval_linear.py's ``train_transform`` (RandomResizedCrop(224), RandomHorizontalFlip) and
``val_transform`` (Resize(256, interpolation=3), CenterCrop(224)) and eval_knn.py's ``transform`` (the same as
``val_transform``), each followed by ToTensor + Normalize, AST-extracted by oracle.eval_augment.reference_eval_transforms.

Sources are seeded synthetic images (oracle.augment.synthetic_image), stored as seed, shape and SHA-256 as in
esvit_augment.pt: the four shapes of that fixture (500 x 375, 375 x 500, 200 x 160, 1600 x 1200, W x H), a short side of
exactly 256 (384 x 256: Resize is the identity), a short side below 224 (150 x 100: both transforms upsample),
257 x 256 (Resize is the identity and the horizontal crop offset round(16.5) is 16), and 1200 x 40 and 40 x 1200
(RandomResizedCrop falls back to its centre crop, and Resize makes a 7680 px long side).

For every source:
  * under a fixed torch seed the reference ``train_transform`` runs TRAIN_CROPS times; esvit_b200.augment's
    LinearTrainParams samples as many records from the same seed and must leave the torch and Python RNGs where the
    reference left them;
  * ``val_transform`` and ``transform`` run once each, must agree, and CenterCropParams gives the record; it must not
    touch the RNGs.
Every reference crop must equal ToTensor + Normalize of oracle.eval_augment.apply_eval_u8 on its record bit for bit.  Each
crop is stored as the SHA-256 of its uint8 bytes plus a seeded sample of its values (oracle.golden.sample).
"""
from __future__ import annotations

import hashlib
import os
import random

import torch
from PIL import Image

from esvit_b200.augment import CenterCropParams, LinearTrainParams
from oracle import augment as A
from oracle import eval_augment as EA
from oracle import reference_import as R
from oracle.make_golden_augment import crop_record

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "esvit_eval_augment.pt")
SOURCES = [(11, 375, 500), (12, 500, 375), (13, 160, 200), (14, 1200, 1600),  # (seed, H, W)
           (15, 256, 384), (16, 100, 150), (17, 256, 257), (18, 40, 1200), (19, 1200, 40)]
TRAIN_CROPS = 3


def _seed(s: int) -> None:
    torch.manual_seed(s)
    random.seed(s)


def _rng():
    return torch.get_rng_state(), random.getstate()


def _same_rng(a, b) -> bool:
    return torch.equal(a[0], b[0]) and a[1] == b[1]


def _check(pil, record, ref: torch.Tensor, what) -> dict:
    u8 = EA.apply_eval_u8(pil, record)
    assert torch.equal(A.normalize(u8), ref), (what, record.tolist())
    return crop_record(torch.from_numpy(u8), what[0])


def main() -> None:
    assert R.available(), f"reference tree not found at {R.REF_ROOT}"
    torch.set_num_threads(1)
    ref = EA.reference_eval_transforms(R.REF_ROOT)
    G = {"meta": {"train_crops": TRAIN_CROPS, "sources": []}, "cases": []}
    for seed, H, W in SOURCES:
        img = A.synthetic_image(seed, H, W)
        pil = Image.fromarray(img, "RGB")
        G["meta"]["sources"].append({"seed": seed, "H": H, "W": W, "sha256": hashlib.sha256(img.tobytes()).hexdigest()})
        tseed = 3000 + seed
        _seed(tseed)
        train_ref = [ref["train_transform"](pil) for _ in range(TRAIN_CROPS)]
        state = _rng()
        _seed(tseed)
        sampler = LinearTrainParams()
        train = torch.stack([sampler.sample(H, W) for _ in range(TRAIN_CROPS)])
        assert _same_rng(_rng(), state), ("LinearTrainParams RNG streams diverge", seed)
        train_crops = [_check(pil, r, x, (seed * 10 + k, "train")) for k, (r, x) in enumerate(zip(train, train_ref))]

        state = _rng()
        val_ref, knn_ref = ref["val_transform"](pil), ref["transform"](pil)
        assert torch.equal(val_ref, knn_ref), seed
        center = CenterCropParams().sample(H, W)
        assert _same_rng(_rng(), state), ("the centre-crop path consumed RNG", seed)
        center_crop = _check(pil, center, val_ref, (seed * 10 + 9, "center"))
        G["cases"].append({"train_seed": tseed, "train": train, "train_crops": train_crops,
                           "center": center, "center_crop": center_crop})
        print(f"source {seed} {W}x{H}: {TRAIN_CROPS} train crops {[r[:4].int().tolist() for r in train]}, centre crop "
              f"{center[4:8].int().tolist()}: reproduced bit for bit by the oracle")
    torch.save(G, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
