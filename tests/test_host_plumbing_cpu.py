"""Host-side autograd plumbing of the module mirror, exercised WITHOUT a GPU: every C-ABI call is replaced by a no-op
(outputs stay uninitialised), so only the wiring is checked - fused pending residuals, the x-less add+LN after
PatchMerging, the per-row DropPath scales, the one-group standalone entry points, the shared gradient accumulators of
the two crop groups, MlpFn.  The numerics of the same paths are the -m gpu tests."""
import torch

from esvit_b200 import _lib, backbone, engine, ops


def _patch(monkeypatch):
    monkeypatch.setattr(_lib, "call", lambda name, *a: None)
    monkeypatch.setattr(ops, "_stream", lambda: 0)

    def chk(t, dtype, name):
        if t is None:
            return None
        assert t.dtype == dtype, (name, t.dtype, dtype)
        return t if t.is_contiguous() else t.contiguous()

    monkeypatch.setattr(ops, "_chk", chk)


import pytest


def _stages_224_96(name):
    """name -> (the rows per image of every stage for 224^2 and 96^2 crops, blocks per stage) of _backbone(name)"""
    if name == "deit_small_p16":
        return [(1 + 14 * 14, 1 + 6 * 6)], [12]
    sides = [(56, 24), (28, 12), (14, 6), (7, 3)]
    if name == "swin_tiny_w7":
        return [(a * a, b * b) for a, b in sides], [1, 1, 2, 1]
    if name == "cvt_13":
        return [(a * a, b * b) for a, b in sides], [2, 2, 6, 2]
    return [(g + a * a, g + b * b) for (a, b), g in zip(sides, [1, 1, 1, 0])], [2, 2, 6, 2]  # vil_2262


def _backbone(name, dense=False):
    """one of the four backbones with its DINO head(s), small where the depth is free, in train mode"""
    spec = dict({**engine.SWIN_SPECS, **engine.VIT_SPECS, **engine.CVT_SPECS, **engine.VIL_SPECS}[name])
    if name == "swin_tiny_w7":
        spec["depths"] = [1, 1, 2, 1]
    torch.manual_seed(0)
    return engine.build_network(spec, 256, dense, False, True, 224, None).train()


BACKBONES = ["swin_tiny_w7", "deit_small_p16", "cvt_13", "vil_2262"]


def _backward_gives_one_gradient_each(params, loss):
    """loss.backward() inside a step: every parameter that requires grad gets exactly one fp32 gradient of its shape"""
    ops.begin_step("cpu", 1 << 22)
    try:
        loss.backward()
        n_shared = len(ops._Arena.accs)
    finally:
        ops.end_step()
    assert ops._Arena.accs is None
    missing = [n for n, p in params if p.requires_grad and p.grad is None]
    assert not missing, missing
    for n, p in params:
        if p.grad is not None:
            assert p.grad.shape == p.shape and p.grad.dtype == torch.float32, n
    return n_shared


# tokens per image of a 224^2 and a 96^2 crop at the last stage, the backbone's width, and its probe widths:
# (n, return_patch_avgpool) -> width of forward_return_n_last_blocks
_ENTRY = {
    "swin_tiny_w7": ([49, 9], 768, {(1, False): 768, (2, False): 384 + 768, (5, False): 96 + 192 + 384 + 384 + 768}),
    "deit_small_p16": ([196, 36], 384, {(1, False): 384, (2, False): 2 * 384, (2, True): 3 * 384, (12, False): 12 * 384}),
    "cvt_13": ([49, 9], 768, {(1, False): 768, (5, False): 3 * 384 + 2 * 768,
                              (12, False): 2 * 64 + 2 * 192 + 6 * 384 + 2 * 768}),
    "vil_2262": ([49, 9], 768, {(1, False): 768, (5, False): 3 * 384 + 2 * 768,
                                (12, False): 2 * 96 + 2 * 192 + 6 * 384 + 2 * 768}),
}


@pytest.mark.parametrize("name,dense", [
    pytest.param(n, d, id=("" if n == "swin_tiny_w7" else n + "-") + ("dense" if d else "view"))
    for n in BACKBONES for d in (True, False)])
def test_every_parameter_gets_one_gradient(monkeypatch, name, dense):
    _patch(monkeypatch)
    net = _backbone(name, dense)
    ntok, width, _ = _ENTRY[name]
    B = 2
    crops = [torch.randn(B, 3, 224, 224) for _ in range(2)] + [torch.randn(B, 3, 96, 96) for _ in range(3)]
    if dense:
        cls, region, fea, npatch = net(crops)
        assert npatch == ntok
        rows = B * (2 * ntok[0] + 3 * ntok[1])
        assert region.shape == (rows, 256) and fea.shape == (rows, width)
        loss = (cls.float() ** 2).sum() + (region.float() ** 2).sum()
    else:
        cls = net(crops)
        loss = (cls.float() ** 2).sum()
    assert cls.shape == (5 * B, 256)
    n_shared = _backward_gives_one_gradient_each(list(net.named_parameters()), loss)
    assert n_shared > 20  # LN / bias / rel-pos-table accumulators


def test_standalone_entry_points_wiring(monkeypatch):
    """The entry points outside the multi-crop forward run the same resolution-group path on one group: shapes, and
    the gradients of forward_features (train mode, DropPath, dense) and of a standalone block."""
    _patch(monkeypatch)
    B = 2
    x = torch.randn(B, 3, 224, 224)
    for name in BACKBONES:
        net = _backbone(name, True)
        ntok, width, probes = _ENTRY[name]
        pooled, region = net.forward_features(x)
        assert pooled.shape == (B, width) and region.shape == (B, ntok[0], width), name
        params = [(n, p) for n, p in net.named_parameters() if not n.startswith("head")]
        _backward_gives_one_gradient_each(params, (pooled ** 2).sum() + (region ** 2).sum())

        net.eval()
        depths = _stages_224_96(name)[1]
        vit = name == "deit_small_p16"  # the ViT probe ignores `depth`, as the reference does
        for (n, avgpool), w in probes.items():
            assert net.forward_return_n_last_blocks(x, n, avgpool, [] if vit else depths).shape == (B, w), (name, n)
        for n in (0, sum(depths) + 1):
            with pytest.raises(ValueError):
                net.forward_return_n_last_blocks(x, n, False, depths)
        if not vit:
            with pytest.raises(ValueError):
                net.forward_return_n_last_blocks(x, 1, False, depths[:-1])

    net = _backbone("swin_tiny_w7", True).eval()
    last = net.forward_selfattention(x, 1)
    assert last.shape == (B, 24, 49, 49) and not last.requires_grad
    maps = net.forward_selfattention(x, 2)
    assert [tuple(m.shape) for m in maps] == [(B * 64, 3, 49, 49), (B * 16, 6, 49, 49), (B * 4, 12, 49, 49),
                                              (B * 4, 12, 49, 49), (B, 24, 49, 49)]

    layer, xs = net.layers[2], torch.randn(B, 14 * 14, 384)
    y, fea = layer.forward_with_features(xs)
    assert y.shape == (B, 49, 768) and [tuple(f.shape) for f in fea] == [(B, 196, 384)] * 2
    y, maps = layer.forward_with_attention(xs)
    assert y.shape == (B, 49, 768) and [tuple(m.shape) for m in maps] == [(B * 4, 12, 49, 49)] * 2

    blk = layer.blocks[1].train()
    assert blk.shift_size == 3 and blk.drop_prob > 0
    xs.requires_grad_(True)
    y, attn = blk(xs)
    assert y.shape == xs.shape and y.dtype == torch.float32 and attn is None
    _backward_gives_one_gradient_each(list(blk.named_parameters()), (y ** 2).sum())
    assert xs.grad.shape == xs.shape


@pytest.mark.parametrize("name", BACKBONES)
def test_drop_path_draw_order_under_a_seed(monkeypatch, name):
    """The DropPath scales a train-mode multi-crop forward hands to the residual adds, bit for bit the timm rule
    floor(keep + U) / keep drawn in each backbone's order: Swin and ViT one [2 * blocks, images] draw, CvT one
    [2 * depth_i, images] draw per stage, ViL its sliding-chunk modes randint(1, 9, [modules, groups]) and then one draw
    per stage; every scale is spread to the rows of its image."""
    _patch(monkeypatch)
    recorded = []
    for fn in ("add_layer_norm", "residual_add"):
        orig = getattr(ops, fn)

        def rec(*a, _orig=orig, **k):
            keep = k["keep"] if "keep" in k else a[2]
            if keep is not None:
                recorded.append(keep.clone())
            return _orig(*a, **k)
        monkeypatch.setattr(ops, fn, rec)
    net = _backbone(name)
    stages, depths = _stages_224_96(name)
    B = 2
    crops = [torch.randn(B, 3, 224, 224) for _ in range(2)] + [torch.randn(B, 3, 96, 96) for _ in range(3)]
    torch.manual_seed(1234)
    net(crops)

    torch.manual_seed(1234)
    images = [2 * B, 3 * B]
    dpr = [float(p) for p in torch.linspace(0, 0.1, sum(depths))]  # drop_path_rate 0.1 of every spec used here
    if name == "vil_2262":
        torch.randint(1, 9, (depths[0] + depths[1], len(images)), dtype=torch.int32)

    def draw(probs):
        kp = torch.tensor([[1.0 - p] for p in probs for _ in range(2)], dtype=torch.float32)
        return torch.rand(kp.shape[0], sum(images), dtype=torch.float32).add_(kp).floor_().div_(kp)

    one_draw = name in ("swin_tiny_w7", "deit_small_p16")
    scales = draw(dpr) if one_draw else None
    expected, b0 = [], 0
    for rows, d in zip(stages, depths):
        s = scales[2 * b0:2 * (b0 + d)] if one_draw else draw(dpr[b0:b0 + d])
        counts = torch.tensor([r for r, n in zip(rows, images) for _ in range(n)])
        for j in range(d):
            if dpr[b0 + j] > 0:
                expected += [s[2 * j].repeat_interleave(counts), s[2 * j + 1].repeat_interleave(counts)]
        b0 += d
    assert len(recorded) == len(expected)
    for i, (got, want) in enumerate(zip(recorded, expected)):
        assert got.dtype == torch.float32 and torch.equal(got, want), i


def test_accumulators_are_private_outside_a_step(monkeypatch):
    _patch(monkeypatch)
    a, first_a = ops._acc(("k", 1), (4,), "cpu")
    b, first_b = ops._acc(("k", 1), (4,), "cpu")
    assert first_a and first_b and a.data_ptr() != b.data_ptr()
    ops.begin_step("cpu", 1 << 10)
    try:
        a, first_a = ops._acc(("k", 1), (4,), "cpu")
        b, first_b = ops._acc(("k", 1), (4,), "cpu")
        assert first_a and not first_b and a.data_ptr() == b.data_ptr()
    finally:
        ops.end_step()


def test_row_samples_and_group_geometry_of_the_concatenated_layout():
    """rows -> samples map and the per-stage geometry the group-aware Functions receive (pure host logic)."""
    spec = dict(engine.SWIN_SPECS["swin_tiny_w7"])
    spec["depths"] = [1, 1, 1, 1]
    net = engine.build_network(spec, 64, True, False, True, 224, None)
    grp = [(2, 56, 56, 0), (3, 24, 24, 2 * 56 * 56)]
    counts = [(B, H * W) for B, H, W, _ in grp]
    rs = backbone.row_samples(net, counts, torch.device("cpu"))
    assert rs.numel() == 2 * 56 * 56 + 3 * 24 * 24
    assert rs[0] == 0 and rs[56 * 56 - 1] == 0 and rs[56 * 56] == 1 and rs[2 * 56 * 56] == 2 and rs[-1] == 4
    assert backbone.row_samples(net, counts, torch.device("cpu")) is rs  # cached per geometry
    merged = []
    row0 = 0
    for B, H, W, _ in grp:  # what PatchMerging.fused hands to the next stage
        merged.append((B, (H + 1) // 2, (W + 1) // 2, row0))
        row0 += B * ((H + 1) // 2) * ((W + 1) // 2)
    assert merged == [(2, 28, 28, 0), (3, 12, 12, 2 * 28 * 28)]


def test_loss_row_order_is_an_image_major_permutation():
    """losses._order: the CTA -> student-row map of the CE kernels is a permutation of the (crop, image, token) storage
    order that visits all rows of image 0, then image 1, ... (so the CTAs resident together share teacher rows)."""
    from esvit_b200.losses import DDINOLoss
    B, ncrops, Tg, Tl = 3, 5, 4, 2
    m = DDINOLoss(64, ncrops, 0.04, 0.04, 0, 10)
    o = m._order(B, [(2, Tg), (ncrops - 2, Tl)], "cpu").tolist()
    R = B * (2 * Tg + (ncrops - 2) * Tl)
    assert sorted(o) == list(range(R))

    def image_of(r):
        if r < 2 * B * Tg:
            return (r // Tg) % B
        return ((r - 2 * B * Tg) // Tl) % B
    imgs = [image_of(r) for r in o]
    assert imgs == sorted(imgs)                      # image-major
    per = 2 * Tg + (ncrops - 2) * Tl
    assert all(imgs[i * per] == i for i in range(B))
    oc = m._order(B, [(ncrops, 1)], "cpu").tolist()  # cls rows: (crop, image) -> (image, crop)
    assert oc == [v * B + b for b in range(B) for v in range(ncrops)]


def test_cat_adjacent_views_back_to_back_crops():
    """ops.cat_adjacent == torch.cat; a view (no copy) exactly when the tensors lie back to back in one storage."""
    import torch
    from esvit_b200 import ops
    buf = torch.randn(3, 4, 3, 8, 8)
    ts = [buf[k] for k in range(3)]
    v = ops.cat_adjacent(ts)
    assert torch.equal(v, torch.cat(ts)) and v.data_ptr() == buf.data_ptr()
    gap = ops.cat_adjacent([buf[0], buf[2]])                       # not adjacent: a real concatenation
    assert torch.equal(gap, torch.cat([buf[0], buf[2]])) and gap.data_ptr() != buf.data_ptr()
    sep = [torch.randn(4, 3, 8, 8) for _ in range(2)]               # separate allocations
    assert torch.equal(ops.cat_adjacent(sep), torch.cat(sep))
    assert ops.cat_adjacent([buf[1]]) is not None and ops.cat_adjacent([buf[1]]).shape == buf[1].shape
