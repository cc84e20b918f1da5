"""Write tests/golden/esvit_augment.pt from the UNMODIFIED reference DataAugmentationDINO (CPU, Pillow).

    python -m oracle.make_golden_augment

Sources are seeded synthetic images (oracle.augment.synthetic_image: numpy integer ops, no codec), regenerated from
their seeds by the tests; the fixture stores their seeds, shapes and a SHA-256 of their bytes.  Shapes: a landscape
(500 x 375) and a portrait (375 x 500) of ImageNet's mean size, one smaller than 224 on a side (200 x 160, the global
crops upsample), and a 1600 x 1200 source for long resampling filters.

For every source, under fixed torch and Python seeds:
  * the reference runs with 2 global + 2 local crops.  Each crop is kept as uint8 (its ToTensor + Normalize is asserted
    to equal the reference's fp32 bit for bit) in compact form: the SHA-256 of all its bytes, which pins every value,
    plus a seeded sample of its values (oracle.golden.sample), which shows the size of a difference.  The fixture also
    stores the parameters esvit_b200.augment.MultiCropParams draws from the same seeds;
  * the reference runs again with its default 2 + 8 crops under a second seed; only the parameters are stored.
Both times the generator asserts that the sampler leaves the torch and Python RNGs where the reference left them, and
that oracle.augment.apply reproduces every reference crop bit for bit.
"""
from __future__ import annotations

import hashlib
import os
import random

import numpy as np
import torch
from PIL import Image

from esvit_b200.augment import MultiCropParams
from oracle import augment as A
from oracle import golden
from oracle import reference_import as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_augment.pt")
SOURCES = [(11, 375, 500), (12, 500, 375), (13, 160, 200), (14, 1200, 1600)]  # (seed, H, W)
GLOBAL_SCALE, LOCAL_SCALE = (0.4, 1.0), (0.05, 0.4)


def _seed(s: int) -> None:
    torch.manual_seed(s)
    random.seed(s)


def _run(root, pil, H, W, seed, n_local):
    ref = A.reference_transform(root, GLOBAL_SCALE, LOCAL_SCALE, (n_local,), (96,))
    _seed(seed)
    crops = ref(pil)
    state = (torch.get_rng_state(), random.getstate())
    _seed(seed)
    params = MultiCropParams(GLOBAL_SCALE, LOCAL_SCALE, (n_local,), (96,)).sample(H, W)
    assert torch.equal(torch.get_rng_state(), state[0]) and random.getstate() == state[1], "RNG streams diverge"
    sizes = [224, 224] + [96] * n_local
    u8 = []
    for k, (crop, p, S) in enumerate(zip(crops, params, sizes)):
        u = A.apply_u8(pil, p, S)
        assert torch.equal(A.normalize(u), crop), (seed, k, p.tolist())
        u8.append(crop_record(torch.from_numpy(u), k))
    return params, u8


def crop_record(u8: torch.Tensor, seed: int) -> dict:
    """a uint8 [S, S, 3] crop as its SHA-256 and a seeded sample of its values"""
    return {"shape": tuple(u8.shape), "sha256": A.digest(u8.numpy()),
            "sample": golden.sample(u8, seed)}


def main() -> None:
    assert R.available(), f"reference tree not found at {R.REF_ROOT}"
    torch.set_num_threads(1)
    G = {"meta": {"global_crops_scale": GLOBAL_SCALE, "local_crops_scale": LOCAL_SCALE, "local_crops_size": 96,
                  "sources": []}, "cases": []}
    for seed, H, W in SOURCES:
        img = A.synthetic_image(seed, H, W)
        pil = Image.fromarray(img, "RGB")
        G["meta"]["sources"].append({"seed": seed, "H": H, "W": W, "sha256": hashlib.sha256(img.tobytes()).hexdigest()})
        params, u8 = _run(R.REF_ROOT, pil, H, W, 1000 + seed, 2)
        params8, _ = _run(R.REF_ROOT, pil, H, W, 2000 + seed, 8)
        G["cases"].append({"seed": 1000 + seed, "params": params, "crops": u8,
                           "seed8": 2000 + seed, "params8": params8})
        print(f"source {seed} {W}x{H}: {len(u8)} + 10 reference crops reproduced bit for bit by the oracle")
    torch.save(G, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
