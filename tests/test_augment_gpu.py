"""Device multi-crop augmentation (csrc/augment.cu via esvit_b200.augment.MultiCropAugment) against Pillow.

Per-op cases compare with oracle.augment (the reference's Pillow / torchvision calls on the same parameters) in uint8
steps: the device fp32 crop is mapped back to uint8 by inverting Normalize, then compared with the oracle's uint8 crop;
wherever the uint8 values agree, the fp32 values must equal torchvision's ToTensor + Normalize bit for bit."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch
from PIL import Image

from esvit_b200 import augment as AG
from oracle import augment as A

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_augment.pt")
MEAN = torch.tensor(A.MEAN, dtype=torch.float32)[:, None, None]
STD = torch.tensor(A.STD, dtype=torch.float32)[:, None, None]
_F = {k: i for i, k in enumerate(AG.PARAM_FIELDS)}


def to_u8(x: torch.Tensor) -> torch.Tensor:
    """[3, S, S] normalised fp32 -> uint8-valued int [S, S, 3]"""
    return torch.round((x.cpu() * STD + MEAN) * 255).to(torch.int32).permute(1, 2, 0)


def batch_of(images, params):
    return AG.collate_multicrop([((torch.from_numpy(im), p), 0) for im, p in zip(images, params)])[0]


def run(images, params, sizes, **kw):
    """images: uint8 HWC arrays; params: [ncrops, NPARAM] per image; sizes: output side per crop position"""
    n_local = len(sizes) - 2
    aug = AG.MultiCropAugment(local_crops_number=(n_local,), local_crops_size=(sizes[2],), global_crops_size=sizes[0])
    return aug(batch_of(images, params), **kw)


def compare(images, params, sizes, out):
    """(max |delta| in uint8 steps, exact fraction); asserts the fp32 is torchvision's wherever the uint8 agrees"""
    worst, exact, total = 0, 0, 0
    for b, (im, P) in enumerate(zip(images, params)):
        pil = Image.fromarray(im, "RGB")
        for k, S in enumerate(sizes):
            ref = A.apply_u8(pil, P[k], S)
            got = out[k][b].cpu()
            d = (to_u8(got) - torch.from_numpy(ref).to(torch.int32)).abs()
            worst = max(worst, int(d.max()))
            exact += int((d == 0).sum())
            total += d.numel()
            if int(d.max()) == 0:
                assert torch.equal(got, A.normalize(ref)), (b, k)
    return worst, exact / total


def base_row(H, W, S, rng):
    """a crop that only resizes: a random box of aspect within [3/4, 4/3] (or the whole image)"""
    h = int(rng.integers(1, H + 1))
    w = int(min(W, max(1, round(h * rng.uniform(0.75, 4 / 3)))))
    return [int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w, int(rng.integers(0, 2)), 0,
            0, 1, 2, 3, 1.0, 1.0, 1.0, 0.0, 0, 0, 0.0, 0]


def random_image(rng, H, W):
    return A.synthetic_image(int(rng.integers(0, 1 << 30)), H, W)


# ---- per op -----------------------------------------------------------------------------------------------------------
def test_resize_and_flip():
    rng = np.random.default_rng(1)
    sizes = [224, 224, 96, 96]
    shapes = [(375, 500), (500, 375), (160, 200), (1200, 1600), (97, 130), (224, 224), (96, 300)]
    images, params = [], []
    for H, W in shapes:
        rows = [base_row(H, W, S, rng) for S in sizes]
        rows[0][:4] = [0, 0, H, W]                                   # whole image
        rows[1][:4] = [H - min(H, 150), W - min(W, 200), min(H, 150), min(W, 200)]  # bottom-right corner, 4:3
        rows[2][:4] = [0, W - min(W, H) * 3 // 4, min(W, H), min(W, H) * 3 // 4]    # top-right, 3:4 (portrait box)
        rows[3][:4] = [H // 3, W // 5, min(40, H - H // 3), min(30, W - W // 5)]    # smaller than S: upsampling
        images.append(random_image(rng, H, W))
        params.append(torch.tensor(rows, dtype=torch.float64))
    out = run(images, params, sizes)
    worst, frac = compare(images, params, sizes, out)
    print(f"resize+flip: max |d| {worst}, exact {frac:.6f}")
    assert worst <= 1


def _identity_case(rng, S, n, edit):
    """n source images of exactly S x S cropped whole (Pillow's resize returns a copy), then `edit(row, i)`"""
    images = [random_image(rng, S, S) for _ in range(n)]
    params = []
    for i in range(n):
        rows = []
        for k in range(4):
            r = [0, 0, S, S, int(rng.integers(0, 2)), 0, 0, 1, 2, 3, 1.0, 1.0, 1.0, 0.0, 0, 0, 0.0, 0]
            edit(r, i * 4 + k)
            rows.append(r)
        params.append(torch.tensor(rows, dtype=torch.float64))
    return images, params


@pytest.mark.parametrize("S", [224, 96])
def test_colour_jitter(S):
    rng = np.random.default_rng(2 + S)
    ends = {"b": [0.6, 1.4], "c": [0.6, 1.4], "s": [0.8, 1.2], "h": [-0.1, 0.1, -0.5, 0.5, -0.001, 0.002]}

    def edit(r, t):
        r[_F["jitter"]] = 1
        r[_F["perm0"]:_F["perm3"] + 1] = [int(v) for v in rng.permutation(4)]
        for j, key in enumerate("bcs"):
            lo, hi = ends[key]
            r[_F["brightness"] + j] = [lo, hi, float(rng.uniform(lo, hi))][t % 3]
        r[_F["hue"]] = ends["h"][t % 6] if t < 12 else float(rng.uniform(-0.1, 0.1))

    sizes = [S] * 4
    images, params = _identity_case(rng, S, 6, edit)
    out = run(images, params, sizes, )
    worst, frac = compare(images, params, sizes, out)
    print(f"colour jitter S={S}: max |d| {worst}, exact {frac:.6f}")
    assert worst <= 1


@pytest.mark.parametrize("op", ["brightness", "contrast", "saturation"])
def test_blend_ops_exact_without_hue_error(op):
    """brightness / contrast / saturation as the only jitter op that changes pixels (hue 0 still runs Pillow's HSV
    round trip, which the hue test covers); gated bit-exact whenever the hue round trip is"""
    rng = np.random.default_rng(3)
    lo, hi = {"brightness": (0.6, 1.4), "contrast": (0.6, 1.4), "saturation": (0.8, 1.2)}[op]

    def edit(r, t):
        r[_F["jitter"]] = 1
        r[_F["perm0"]:_F["perm3"] + 1] = [3, 0, 1, 2] if t % 2 else [0, 1, 2, 3]
        r[_F[op]] = [lo, hi, float(rng.uniform(lo, hi)), 0.0][t % 4]

    images, params = _identity_case(rng, 96, 4, edit)
    out = run(images, params, [96] * 4)
    worst, frac = compare(images, params, [96] * 4, out)
    print(f"{op}: max |d| {worst}, exact {frac:.6f}")
    assert worst == 0


def test_grayscale_then_solarize_exact():
    rng = np.random.default_rng(4)

    def edit(r, t):
        r[_F["grayscale"]] = t % 2
        r[_F["solarize"]] = 1 if t % 4 < 3 else 0

    images, params = _identity_case(rng, 224, 3, edit)
    out = run(images, params, [224] * 4)
    worst, _ = compare(images, params, [224] * 4, out)
    assert worst == 0


@pytest.mark.parametrize("S", [224, 96])
def test_blur(S):
    rng = np.random.default_rng(5 + S)
    radii = [0.1, 2.0, 1.0, 0.5]

    def edit(r, t):
        r[_F["blur"]] = 1
        r[_F["radius"]] = radii[t] if t < 4 else float(rng.uniform(0.1, 2.0))

    images, params = _identity_case(rng, S, 4, edit)
    out = run(images, params, [S] * 4)
    worst, frac = compare(images, params, [S] * 4, out)
    print(f"blur S={S}: max |d| {worst}, exact {frac:.6f}")
    assert worst <= 1


def test_sampled_parameters_many_sizes():
    """the sampler's own parameter stream over random source sizes, every op at once"""
    rng = np.random.default_rng(6)
    t = AG.MultiCropParams((0.4, 1.0), (0.05, 0.4), (8,), (96,))
    images, params = [], []
    torch.manual_seed(6)
    random.seed(6)
    for _ in range(6):
        H, W = int(rng.integers(120, 900)), int(rng.integers(120, 900))
        images.append(random_image(rng, H, W))
        params.append(t.sample(H, W))
    out = run(images, params, t.sizes)
    worst, frac = compare(images, params, t.sizes, out)
    print(f"sampled 2+8 crops: max |d| {worst}, exact {frac:.6f}")
    assert worst <= 1


# ---- end to end against the reference fixture -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    G = torch.load(GOLDEN, map_location="cpu", weights_only=False)
    G["images"] = []
    for src in G["meta"]["sources"]:
        img = A.synthetic_image(src["seed"], src["H"], src["W"])
        assert hashlib.sha256(img.tobytes()).hexdigest() == src["sha256"]
        G["images"].append(img)
    return G


def test_fixture_end_to_end(golden):
    """the fixture pins each reference crop by the SHA-256 of its uint8 bytes and a seeded sample of its values; the
    oracle (checked against both on CPU) supplies the full crop for the difference"""
    from oracle import golden as GD
    sizes = [224, 224, 96, 96]
    params = [c["params"] for c in golden["cases"]]
    out = run(golden["images"], params, sizes)
    worst, exact, total, same_digest = 0, 0, 0, 0
    for b, (img, case) in enumerate(zip(golden["images"], golden["cases"])):
        pil = Image.fromarray(img, "RGB")
        for k, (p, ref) in enumerate(zip(case["params"], case["crops"])):
            got = to_u8(out[k][b])
            sampled, want = GD.at_golden(got, ref["sample"])
            assert int((sampled - want.to(torch.int32)).abs().max()) <= 2, (b, k)
            full = torch.from_numpy(A.apply_u8(pil, p, sizes[k]))
            assert A.digest(full.numpy()) == ref["sha256"]
            d = (got - full.to(torch.int32)).abs()
            worst = max(worst, int(d.max()))
            exact += int((d == 0).sum())
            total += d.numel()
            same_digest += A.digest(got.to(torch.uint8).numpy()) == ref["sha256"]
    print(f"reference fixture: max |d| {worst}, exact {exact / total:.6f} of {total} values, "
          f"{same_digest} of {len(sizes) * len(params)} crops with the reference's SHA-256")
    assert worst <= 2


def test_mixed_batch_equals_each_image_alone_and_reruns_are_identical(golden):
    sizes = [224, 224, 96, 96]
    params = [c["params"] for c in golden["cases"]]
    out = run(golden["images"], params, sizes)
    again = run(golden["images"], params, sizes)
    for a, b in zip(out, again):
        assert torch.equal(a, b)
    for b, (im, p) in enumerate(zip(golden["images"], params)):
        alone = run([im], [p], sizes)
        for k in range(len(sizes)):
            assert torch.equal(alone[k][0], out[k][b]), (b, k)


def test_source_buffer_past_2_31_bytes():
    side = 14000
    n_img = 4  # 4 x 588 MB: the last image starts at 1.76e9 and ends past 2^31 bytes
    g = torch.Generator(device="cuda").manual_seed(0)
    small = torch.randint(0, 256, (side // 10, side // 10, 3), dtype=torch.uint8, device="cuda", generator=g)
    img = torch.nn.functional.interpolate(small.permute(2, 0, 1)[None].float(), size=(side, side), mode="nearest")
    img = img[0].permute(1, 2, 0).to(torch.uint8).contiguous()
    nbytes = img.numel()
    pixels = torch.empty(n_img * nbytes, dtype=torch.uint8, device="cuda")
    for i in range(n_img):
        pixels[i * nbytes:(i + 1) * nbytes] = img.view(-1)
    del small
    index = torch.tensor([[i * nbytes, side, side] for i in range(n_img)], dtype=torch.int64)
    rows = [[side - 3000, side - 4000, 3000, 4000, 1, 0, 0, 1, 2, 3, 1.0, 1.0, 1.0, 0.0, 0, 1, 1.3, 0],
            [0, 0, side, side, 0, 1, 3, 2, 1, 0, 1.2, 0.7, 1.1, 0.05, 0, 0, 0.0, 1],
            [side - 900, side - 700, 900, 700, 0, 0, 0, 1, 2, 3, 1.0, 1.0, 1.0, 0.0, 1, 0, 0.0, 0]]
    params = torch.tensor([rows] * n_img, dtype=torch.float64)
    aug = AG.MultiCropAugment(local_crops_number=(1,), local_crops_size=(96,))
    out = aug(AG.MultiCropBatch(pixels, index, params))
    alone = aug(AG.MultiCropBatch(img.view(-1), index[:1] * torch.tensor([0, 1, 1]), params[:1]))
    assert int(index[-1, 0]) + nbytes > 2 ** 31
    for k in range(3):
        for b in range(n_img):
            assert torch.equal(out[k][b], alone[k][0]), (k, b)


# ---- interface ---------------------------------------------------------------------------------------------------------
def _good(golden):
    return [golden["images"][0]], [golden["cases"][0]["params"]]


def test_invalid_input_raises(golden):
    images, params = _good(golden)
    aug = AG.MultiCropAugment(local_crops_number=(2,), local_crops_size=(96,))
    good = batch_of(images, params)
    aug(good)

    def with_param(field, value, crop=0):
        p = good.params.clone()
        p[0, crop, _F[field]] = value
        return good._replace(params=p)

    bad = [good._replace(pixels=good.pixels.float()),
           good._replace(params=good.params[:, :3]),
           good._replace(params=good.params.float()),
           good._replace(index=torch.tensor([[0, 0, 10]])),
           good._replace(index=torch.tensor([[0, 10 ** 6, 10]])),
           with_param("height", 10 ** 5), with_param("top", -1), with_param("width", 0), with_param("left", 0.5),
           with_param("flip", 2), with_param("perm0", 1), with_param("hue", 0.7), with_param("brightness", -0.1),
           with_param("radius", 0.0, crop=0) if bool(good.params[0, 0, _F["blur"]]) else with_param("blur", 1),
           with_param("saturation", float("nan"))]
    for b in bad:
        with pytest.raises(ValueError):
            aug(b)
    with pytest.raises(ValueError):
        aug(good, out=[torch.empty(1, 3, 224, 224, device="cuda")] * 3)
    with pytest.raises(ValueError):
        AG.collate_multicrop([((torch.zeros(8, 8, 4, dtype=torch.uint8), params[0]), 0)])
    with pytest.raises(ValueError):
        AG.MultiCropAugment(global_crops_size=256)


def test_pinned_collate_and_out_buffers_on_current_stream(golden):
    params = [c["params"] for c in golden["cases"]]
    items = [((torch.from_numpy(im), p), 0) for im, p in zip(golden["images"], params)]
    batch, _ = AG.collate_multicrop(items, pin_memory=True)
    assert batch.pixels.is_pinned() and batch.params.is_pinned()
    assert batch.pin_memory().pixels.is_pinned()
    aug = AG.MultiCropAugment(local_crops_number=(2,), local_crops_size=(96,))
    want = aug(batch)
    side = torch.cuda.Stream()
    bufs = [torch.full((4, 3, s, s), float("nan"), device="cuda") for s in (224, 224, 96, 96)]
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        got = aug(batch, out=bufs)
    side.synchronize()
    assert all(g is b for g, b in zip(got, bufs))
    for g, w in zip(bufs, want):
        assert torch.equal(g, w)


def test_swin_step_fed_device_crops_equals_host_round_trip():
    from esvit_b200 import engine
    rng = np.random.default_rng(7)
    t = AG.MultiCropParams((0.4, 1.0), (0.05, 0.4), (8,), (96,))
    torch.manual_seed(7)
    random.seed(7)
    images = [random_image(rng, 375, 500), random_image(rng, 500, 375)]
    params = [t.sample(*im.shape[:2]) for im in images]
    crops = AG.MultiCropAugment()(batch_of(images, params))
    host = [c.cpu().pin_memory().cuda(non_blocking=True) for c in crops]
    assert all(torch.equal(a, b) for a, b in zip(crops, host))
    losses, weights = [], []
    for feed in (crops, host):
        step, student, _, _ = engine.make_step(out_dim=4096, ncrops=10, device="cuda", seed=0)
        losses.append(float(step(feed, 0, 5e-4, 0.04, 0.996)))
        weights.append(torch.cat([p.detach().reshape(-1).cpu() for p in student.parameters()]))
    assert abs(losses[0] - losses[1]) <= 1e-6 * abs(losses[1]), losses
    assert torch.allclose(weights[0], weights[1], rtol=0, atol=1e-6)
