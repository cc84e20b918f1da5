"""CPU checks of the evaluation transforms' host side (esvit_b200.augment LinearTrainParams / CenterCropParams) and oracle
against tests/golden/esvit_eval_augment.pt (written from the unmodified eval_linear.py / eval_knn.py transforms by
oracle/make_golden_eval_augment.py) and against torchvision's own Resize + CenterCrop."""
import hashlib
import os

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision import transforms as T

from esvit_b200 import augment as AG
from oracle import augment as A
from oracle import eval_augment as EA
from oracle import golden as GD

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_eval_augment.pt")
_E = {k: i for i, k in enumerate(AG.EVAL_FIELDS)}


@pytest.fixture(scope="module")
def golden():
    G = torch.load(GOLDEN, map_location="cpu", weights_only=False)
    G["images"] = []
    for src in G["meta"]["sources"]:
        img = A.synthetic_image(src["seed"], src["H"], src["W"])
        assert hashlib.sha256(img.tobytes()).hexdigest() == src["sha256"], "synthetic source changed"
        G["images"].append(img)
    return G


def _check_crop(pil, record, ref):
    u8 = EA.apply_eval_u8(pil, record)
    got, want = GD.at_golden(torch.from_numpy(u8), ref["sample"])
    assert torch.equal(got, want)
    assert A.digest(u8) == ref["sha256"]


def test_oracle_reproduces_fixture_crops(golden):
    for img, case in zip(golden["images"], golden["cases"]):
        pil = Image.fromarray(img, "RGB")
        for r, ref in zip(case["train"], case["train_crops"]):
            _check_crop(pil, r, ref)
        _check_crop(pil, case["center"], case["center_crop"])


def test_samplers_reproduce_fixture_records(golden):
    for src, case in zip(golden["meta"]["sources"], golden["cases"]):
        torch.manual_seed(case["train_seed"])
        t = AG.LinearTrainParams()
        got = torch.stack([t.sample(src["H"], src["W"]) for _ in range(golden["meta"]["train_crops"])])
        assert torch.equal(got, case["train"])
        assert torch.equal(AG.CenterCropParams().sample(src["H"], src["W"]), case["center"])


def test_fixture_covers_the_edge_geometries(golden):
    by_shape = {(s["H"], s["W"]): c for s, c in zip(golden["meta"]["sources"], golden["cases"])}
    c = by_shape[(256, 384)]["center"]                    # short side 256: Resize is the identity
    assert c[_E["resize_h"]:_E["resize_w"] + 1].tolist() == [256, 384]
    c = by_shape[(256, 257)]["center"]                    # (257 - 224) / 2 = 16.5 rounds to even
    assert c[_E["resize_w"]] == 257 and c[_E["win_left"]] == 16
    for shape in ((40, 1200), (1200, 40)):                # RandomResizedCrop's fallback: a 40 x 53 centre box
        case = by_shape[shape]
        assert all(sorted(r[_E["height"]:_E["width"] + 1].int().tolist()) == [40, 53] for r in case["train"])
        assert max(case["center"][_E["resize_h"]:_E["resize_w"] + 1].tolist()) == 7680
    assert {int(r[_E["flip"]]) for c in golden["cases"] for r in c["train"]} == {0, 1}


@pytest.mark.parametrize("H,W", [(H, W) for H in (1, 97, 223, 224, 255, 256, 257, 300, 333, 481, 1024)
                                 for W in (1, 100, 224, 256, 257, 258, 375, 500, 999)])
def test_center_crop_geometry_matches_torchvision(H, W):
    """resized size from torchvision's Resize(256, bicubic) on a PIL image, window offsets from CenterCrop(224) on a
    tensor whose values are their own coordinates"""
    r = AG.CenterCropParams().sample(H, W)
    resized = T.Resize(256, interpolation=T.InterpolationMode.BICUBIC)(Image.new("RGB", (W, H)))
    rw, rh = resized.size
    coords = torch.arange(rh * rw, dtype=torch.int64).view(1, rh, rw)
    win = T.CenterCrop(224)(coords)
    assert tuple(win.shape) == (1, 224, 224)
    oy, ox = divmod(int(win[0, 0, 0]), rw)
    assert r.tolist() == [0, 0, H, W, rh, rw, oy, ox, 224, 0, AG.PIL_BICUBIC]


def test_worker_transforms_and_collate_with_index_targets(golden):
    """the records ride on the unchanged collate; ReturnIndexDataset's (img, idx) index goes through as the target"""
    imgs = golden["images"][:3]
    for t in (AG.LinearTrainParams(), AG.CenterCropParams()):
        torch.manual_seed(0)
        items = [(t(Image.fromarray(im, "RGB")), idx) for idx, im in zip((7, 3, 11), imgs)]
        for (u8, rec), _ in items:
            assert u8.dtype == torch.uint8 and rec.dtype == torch.float64 and tuple(rec.shape) == (AG.NEVAL,)
        batch, targets = AG.collate_multicrop(items)
        assert targets.tolist() == [7, 3, 11]
        assert torch.equal(batch.params, torch.stack([rec for (_, rec), _ in items]))
        off = 0
        for k, im in enumerate(imgs):
            assert batch.index[k].tolist() == [off, im.shape[0], im.shape[1]]
            assert np.array_equal(batch.pixels[off:off + im.size].view(im.shape).numpy(), im)
            off += im.size
    with pytest.raises(ValueError):
        AG.CenterCropParams()(np.zeros((4, 4, 4), np.uint8))
    with pytest.raises(ValueError):
        AG.CenterCropParams(resize=200, crop=224)
