"""Device evaluation transforms (csrc/augment.cu eval kernels via esvit_b200.augment.EvalAugment) against Pillow.

Every comparison is torch.equal on the fp32 tensor: the oracle (oracle.eval_augment.apply_eval_u8, the reference's
torchvision / Pillow calls on the same record) followed by torchvision's ToTensor + Normalize, which on the fixture's
records is pinned to the unmodified reference transforms by the SHA-256 of each crop."""
import hashlib
import os
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn as nn
from PIL import Image

from esvit_b200 import augment as AG
from oracle import augment as A
from oracle import eval_augment as EA

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_eval_augment.pt")
_E = {k: i for i, k in enumerate(AG.EVAL_FIELDS)}


@pytest.fixture(scope="module")
def golden():
    G = torch.load(GOLDEN, map_location="cpu", weights_only=False)
    G["images"] = []
    for src in G["meta"]["sources"]:
        img = A.synthetic_image(src["seed"], src["H"], src["W"])
        assert hashlib.sha256(img.tobytes()).hexdigest() == src["sha256"]
        G["images"].append(img)
    return G


def batch_of(images, records, **kw):
    return AG.collate_multicrop([((torch.from_numpy(im), r), 0) for im, r in zip(images, records)], **kw)[0]


def oracle(images, records) -> torch.Tensor:
    return torch.stack([A.normalize(EA.apply_eval_u8(Image.fromarray(im, "RGB"), r)) for im, r in zip(images, records)])


def assert_equal_oracle(images, records, out):
    want = oracle(images, records)
    got = out.cpu()
    for b in range(len(images)):
        assert torch.equal(got[b], want[b]), (b, records[b].tolist())


def test_fixture_crops_equal_reference(golden):
    """one batch of every train record (sources of nine sizes) and one of every centre record"""
    images, records, refs = [], [], []
    for im, case in zip(golden["images"], golden["cases"]):
        images += [im] * len(case["train"])
        records += list(case["train"])
        refs += case["train_crops"]
    centre = [c["center"] for c in golden["cases"]]
    aug = AG.EvalAugment()
    centre_crops = [c["center_crop"] for c in golden["cases"]]
    for ims, recs, crops in ((images, records, refs), (golden["images"], centre, centre_crops)):
        out = aug(batch_of(ims, recs)).cpu()
        for b, (im, r, ref) in enumerate(zip(ims, recs, crops)):
            u8 = EA.apply_eval_u8(Image.fromarray(im, "RGB"), r)
            assert A.digest(u8) == ref["sha256"]               # the oracle's crop is the reference's
            assert torch.equal(out[b], A.normalize(u8)), (b, r.tolist())


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_sweep_mixed_sizes_and_filters(seed):
    """random sources of mixed sizes in one batch, LinearTrainParams at several scales and CenterCropParams records side
    by side (each record carries its filter)"""
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    S = [224, 96, 61][seed]
    train = AG.LinearTrainParams(size=S, scale=[(0.08, 1.0), (0.005, 0.05), (0.5, 1.0)][seed])
    centre = AG.CenterCropParams(resize=[256, 112, 61][seed], crop=S)
    images, records = [], []
    for k in range(12):
        H, W = int(rng.integers(1, 700)), int(rng.integers(1, 700))
        if k % 5 == 4:
            H, W = (H, 3 + W % 30) if k % 2 else (3 + H % 30, W)  # elongated
        images.append(A.synthetic_image(int(rng.integers(1 << 30)), H, W))
        records.append((train if k % 2 else centre).sample(H, W))
    out = AG.EvalAugment()(batch_of(images, records))
    assert tuple(out.shape) == (12, 3, S, S)
    assert_equal_oracle(images, records, out)


def test_flip_on_and_off(golden):
    images = golden["images"][:4]
    base = [golden["cases"][k]["train"][0].clone() for k in range(4)]
    aug = AG.EvalAugment()
    outs = []
    for flip in (0, 1):
        recs = [r.clone() for r in base]
        for r in recs:
            r[_E["flip"]] = flip
        out = aug(batch_of(images, recs))
        assert_equal_oracle(images, recs, out)
        outs.append(out)
    assert torch.equal(outs[1], outs[0].flip(-1))


def test_out_buffer_pinned_batch_on_side_stream(golden):
    recs = [c["center"] for c in golden["cases"]]
    batch = batch_of(golden["images"], recs, pin_memory=True)
    aug = AG.EvalAugment()
    want = aug(batch)
    buf = torch.full((len(recs), 3, 224, 224), float("nan"), device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = aug(batch, out=buf)
    side.synchronize()
    assert got is buf and torch.equal(buf, want)
    again = aug(batch)
    assert torch.equal(again, want)
    with pytest.raises(ValueError):
        aug(batch, out=torch.empty(len(recs), 3, 224, 223, device="cuda"))
    with pytest.raises(ValueError):
        aug(batch, out=torch.empty(len(recs), 3, 224, 224, device="cuda", dtype=torch.float16))


def test_invalid_input_raises(golden):
    im = golden["images"][0]
    good = batch_of([im, im], [golden["cases"][0]["train"][0], golden["cases"][0]["center"]])
    aug = AG.EvalAugment()
    aug(good)

    def with_field(field, value, row=0):
        p = good.params.clone()
        p[row, _E[field]] = value
        return good._replace(params=p)

    H, W = im.shape[:2]
    bad = [good._replace(pixels=good.pixels.float()),
           good._replace(params=good.params.float()),
           good._replace(params=good.params[:, :-1]),
           good._replace(params=good.params[None]),
           good._replace(index=torch.tensor([[0, 0, 10], [0, 10, 10]])),
           good._replace(index=good.index * torch.tensor([1, 2, 1])),
           with_field("top", -1), with_field("left", W), with_field("height", H + 1), with_field("width", 0),
           with_field("top", 0.5), with_field("resize_h", 1.5, row=1), with_field("flip", 2), with_field("flip", -1),
           with_field("interpolation", 1), with_field("interpolation", 0), with_field("size", 96),
           with_field("win_left", 1000, row=1), with_field("win_top", -1, row=1), with_field("resize_w", 100, row=1),
           with_field("height", float("nan")), with_field("resize_h", 2.0 ** 40)]
    for b in bad:
        with pytest.raises(ValueError):
            aug(b)


def test_swin_t_features_from_device_crops_equal_reference_crops(golden):
    """the linear probe's features and the k-NN features of Swin-T from device crops and from the reference-transformed
    tensor copied to the GPU: the inputs are bit-identical, so the outputs are"""
    from esvit_b200.swin_transformer import SwinTransformer
    from oracle import golden as GD
    from oracle import swin as S
    spec = dict(S.SWIN_T_W7)
    depths = list(spec["depths"])
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                        **spec)
    m.load_state_dict(GD.seeded_state_dict(GD.recipe(m.state_dict()), 0))
    m = m.cuda().eval()
    images = golden["images"][:8]
    recs = [c["center"] for c in golden["cases"][:8]]
    dev = AG.EvalAugment()(batch_of(images, recs))
    host = oracle(images, recs).pin_memory().cuda(non_blocking=True)
    assert torch.equal(dev, host)
    with torch.no_grad():
        assert torch.equal(m.forward_return_n_last_blocks(dev, 4, False, depths),
                           m.forward_return_n_last_blocks(host, 4, False, depths))
        assert torch.equal(m(dev), m(host))
