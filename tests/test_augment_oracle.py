"""CPU checks of the multi-crop augmentation's host side against tests/golden/esvit_augment.pt (written from the
unmodified reference DataAugmentationDINO by oracle/make_golden_augment.py)."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch
from PIL import Image

from esvit_b200 import augment as AG
from oracle import augment as A
from oracle import golden as GD

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_augment.pt")


@pytest.fixture(scope="module")
def golden():
    G = torch.load(GOLDEN, map_location="cpu", weights_only=False)
    G["images"] = []
    for src in G["meta"]["sources"]:
        img = A.synthetic_image(src["seed"], src["H"], src["W"])
        assert hashlib.sha256(img.tobytes()).hexdigest() == src["sha256"], "synthetic source changed"
        G["images"].append(img)
    return G


def _sample(G, seed, n_local, H, W):
    torch.manual_seed(seed)
    random.seed(seed)
    m = G["meta"]
    return AG.MultiCropParams(m["global_crops_scale"], m["local_crops_scale"], (n_local,), (96,)).sample(H, W)


def test_sampler_reproduces_fixture_parameters(golden):
    for src, case in zip(golden["meta"]["sources"], golden["cases"]):
        assert torch.equal(_sample(golden, case["seed"], 2, src["H"], src["W"]), case["params"])
        assert torch.equal(_sample(golden, case["seed8"], 8, src["H"], src["W"]), case["params8"])


def test_worker_transform_returns_image_and_parameters(golden):
    img = golden["images"][0]
    m = golden["meta"]
    t = AG.MultiCropParams(m["global_crops_scale"], m["local_crops_scale"], (2,), (96,))
    torch.manual_seed(golden["cases"][0]["seed"])
    random.seed(golden["cases"][0]["seed"])
    u8, p = t(Image.fromarray(img, "RGB"))
    assert u8.dtype == torch.uint8 and tuple(u8.shape) == img.shape and np.array_equal(u8.numpy(), img)
    assert torch.equal(p, golden["cases"][0]["params"])
    assert t.sizes == [224, 224, 96, 96]
    with pytest.raises(ValueError):
        t(np.zeros((4, 4, 4), np.uint8))
    with pytest.raises(ValueError):
        t(np.zeros((0, 4, 3), np.uint8))


def test_oracle_reproduces_fixture_crops(golden):
    for img, case in zip(golden["images"], golden["cases"]):
        pil = Image.fromarray(img, "RGB")
        for p, ref in zip(case["params"], case["crops"]):
            u8 = A.apply_u8(pil, p, ref["shape"][0])
            got, want = GD.at_golden(torch.from_numpy(u8), ref["sample"])
            assert torch.equal(got, want)
            assert A.digest(u8) == ref["sha256"]


def test_normalisation_round_trip_is_exact(golden):
    case = golden["cases"][0]
    u8 = A.apply_u8(Image.fromarray(golden["images"][0], "RGB"), case["params"][0], 224)
    assert A.digest(u8) == case["crops"][0]["sha256"]
    got = A.normalize(u8)
    mean = torch.tensor(A.MEAN, dtype=torch.float32)[:, None, None]
    std = torch.tensor(A.STD, dtype=torch.float32)[:, None, None]
    want = (torch.from_numpy(u8).permute(2, 0, 1).float() / 255 - mean) / std
    assert torch.equal(got, want)
    # every uint8 value maps to a distinct fp32 per channel, so a crop kept as uint8 loses nothing
    allv = A.normalize(np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, 2))
    assert all(len(torch.unique(allv[c])) == 256 for c in range(3))


def test_collate_packs_images_and_parameters(golden):
    imgs = [torch.from_numpy(i) for i in golden["images"][:3]]
    params = [c["params"] for c in golden["cases"][:3]]
    batch, targets = AG.collate_multicrop([((im, p), k) for k, (im, p) in enumerate(zip(imgs, params))])
    assert torch.equal(targets, torch.arange(3))
    assert batch.pixels.dtype == torch.uint8 and batch.pixels.dim() == 1
    assert batch.index.dtype == torch.int64 and batch.params.dtype == torch.float64
    off = 0
    for k, im in enumerate(imgs):
        assert batch.index[k].tolist() == [off, im.shape[0], im.shape[1]]
        assert torch.equal(batch.pixels[off:off + im.numel()].view(im.shape), im)
        off += im.numel()
    assert batch.pixels.numel() == off
    assert torch.equal(batch.params, torch.stack(params))
    assert hasattr(batch, "pin_memory")  # DataLoader(pin_memory=True) pins both buffers through it
    with pytest.raises(ValueError):
        AG.collate_multicrop([((torch.zeros(4, 4, 3, dtype=torch.float32), params[0]), 0)])
