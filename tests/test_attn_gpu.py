"""GPU: attention-map extraction - SwinTransformer.forward_selfattention and the esvit_window_attn_probs kernel behind it -
against the pinned reference fixture (tests/golden/esvit_attn.pt), fp32 torch softmax of the same bf16 qkv at real
geometries, and the CPU oracle at real model shapes."""
import os
from functools import partial

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import TOL_BF16_ACT, TOL_FP32_KERNEL, assert_close, at_golden
from oracle import attn as A
from oracle import eval as E
from oracle import swin as S

pytestmark = pytest.mark.gpu

GOLDEN_ATTN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_attn.pt")
MAX_ABS = 5e-5                    # probabilities are <= 1; ex2.approx and the fp32 mma sum give ~1e-6 relative
ROWSUM = {7: 1e-5, 14: 4e-5}      # |sum_j P_ij - 1|; measured maxima in DESIGN.md §4.5


@pytest.fixture(scope="module")
def G():
    return A.load_golden_attn(GOLDEN_ATTN)


def _model(img_size, spec, sd=None, seed=0):
    from esvit_b200.swin_transformer import SwinTransformer
    from oracle import golden as GD
    m = SwinTransformer(img_size=img_size, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                        **spec)
    sd = sd if sd is not None else GD.seeded_state_dict(GD.recipe(m.state_dict()), seed)
    m.load_state_dict(sd)
    return m.cuda().eval(), sd


# ---- 1. the reference's own maps ---------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["w7_112", "w7_96", "w14_112", "w14_96"])
def test_selfattention_matches_reference_fixture(G, name):
    C = G["cases"][name]
    sp = dict(C["spec"])
    img = sp.pop("img_size")
    m, _ = _model(img, sp, sd=C["state_dict"])
    x = C["images"].cuda()
    for n, refs in C["maps"].items():
        out = m.forward_selfattention(x, n)
        outs = [out] if n == 1 else out
        assert isinstance(outs, list) and len(outs) == len(refs), n
        for i, (a, ref) in enumerate(zip(outs, refs)):
            shape = tuple(ref["shape"]) if isinstance(ref, dict) else tuple(ref.shape)
            assert tuple(a.shape) == shape and a.dtype == torch.float32 and not a.requires_grad, (n, i)
            a, r = at_golden(a, ref)
            assert_close(a, r, TOL_BF16_ACT, f"{name} n={n} block {i}")


# ---- 2./3. the kernel alone against fp32 torch on the same bf16 qkv ---------------------------------------------
def _torch_probs(qkv, qkv_bias, table, B, H, W, nH, ws, shift, scale):
    """fp64 softmax of the reference's scores (models/swin_transformer.py:120-147, :283-308) from the SAME bf16 qkv;
    padded slots hold the bf16 qkv bias."""
    C = qkv.shape[-1] // 3
    Hp, Wp = -(-H // ws) * ws, -(-W // ws) * ws
    x = qkv_bias.to(torch.bfloat16).double().view(1, 1, 1, 3 * C).repeat(B, Hp, Wp, 1)
    x[:, :H, :W] = qkv.view(B, H, W, 3 * C).double()
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    N = ws * ws
    xw = x.view(B, Hp // ws, ws, Wp // ws, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(-1, N, 3, nH, 32)
    q, k = xw[:, :, 0].transpose(1, 2), xw[:, :, 1].transpose(1, 2)
    s = (q * scale) @ k.transpose(-2, -1)
    s = s + table.double()[S.rel_pos_index(ws).to(table.device).view(-1)].view(N, N, nH).permute(2, 0, 1)
    if shift:
        mask = S.shift_mask(H, W, ws, shift).to(s.device).double()
        s = (s.view(B, -1, nH, N, N) + mask[None, :, None]).view(-1, nH, N, N)
    return s.softmax(-1)


W7 = [(96, m) for m in (56, 24)] + [(192, m) for m in (28, 12)] + [(384, m) for m in (14, 6)] + [(768, 7)]
W14 = [(128, m) for m in (56, 24)] + [(256, m) for m in (28, 12)] + [(512, 14), (1024, 14)]
KERNEL_CASES = ([(C, m, 7, s) for C, m in W7 for s in (0, 3)] + [(C, m, 14, s) for C, m in W14 for s in (0, 7)])


def _kernel_case(C, side, ws, shift):
    from esvit_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C * 1000 + side * 10 + shift)
    nH = C // 32
    B = 1 if side * side * C > 56 * 56 * 128 else 2
    qkv = torch.randn(B, side * side, 3 * C, device="cuda", generator=g).to(torch.bfloat16)
    qkv_bias = torch.randn(3 * C, device="cuda", generator=g)
    table = torch.randn((2 * ws - 1) ** 2, nH, device="cuda", generator=g)
    scale = 32 ** -0.5
    p = ops.window_attention_probs(qkv, qkv_bias, table, side, side, nH, ws, shift, scale)
    ref = _torch_probs(qkv, qkv_bias, table, B, side, side, nH, ws, shift, scale)
    return p, ref


def _check_kernel_case(C, side, ws, shift):
    p, ref = _kernel_case(C, side, ws, shift)
    tag = f"C={C} map={side} ws={ws} shift={shift}"
    assert p.shape == ref.shape and p.dtype == torch.float32, tag
    assert_close(p, ref, TOL_FP32_KERNEL, tag)
    err = float((p.double() - ref).abs().max())
    assert err < MAX_ABS, (tag, err)
    rs = float((p.double().sum(-1) - 1).abs().max())
    assert rs < ROWSUM[ws], (tag, rs)
    print(f"attn-probs {tag}: max|dP| {err:.2e} max|rowsum-1| {rs:.2e}")


@pytest.mark.parametrize("C,side,ws,shift", KERNEL_CASES)
def test_probs_kernel_matches_torch(C, side, ws, shift):
    _check_kernel_case(C, side, ws, shift)


@pytest.mark.parametrize("C,side,ws,shift", [c for c in KERNEL_CASES if c[1] in (56, 24, 28)])
def test_probs_kernel_multi_window_ctas(monkeypatch, C, side, ws, shift):
    monkeypatch.setenv("ESVIT_ATTN_GY", "2")  # two CTAs per head: each walks many windows
    _check_kernel_case(C, side, ws, shift)


# ---- 4. real models against the CPU oracle -----------------------------------------------------------------------
@pytest.mark.parametrize("arch,nblk", [("swin_t_w7", 12), ("swin_b_w14", 24)])
def test_selfattention_real_models_match_oracle(arch, nblk):
    spec = dict(S.SWIN_T_W7 if arch == "swin_t_w7" else S.SWIN_B_W14)
    m, sd = _model(224, spec, seed=5)
    x = E.probe_images(2, 224, 9)
    maps = m.forward_selfattention(x.cuda(), 2)
    with torch.no_grad():
        refs = A.selfattention(x, sd, S.SwinSpec(img_size=224, **spec), 2)
    assert len(maps) == len(refs) == nblk
    for i, (a, r) in enumerate(zip(maps, refs)):
        assert a.shape == r.shape, (i, tuple(a.shape), tuple(r.shape))
        assert_close(a, r, TOL_BF16_ACT, f"{arch} block {i}")
    if arch == "swin_t_w7":
        assert [tuple(t.shape) for t in maps] == ([(128, 3, 49, 49)] * 2 + [(32, 6, 49, 49)] * 2 + [(8, 12, 49, 49)] * 6
                                                  + [(2, 24, 49, 49)] * 2)
    else:
        assert tuple(maps[0].shape) == (32, 4, 196, 196)
    last = m.forward_selfattention(x.cuda(), 1)
    assert torch.equal(last, maps[-1])


# ---- 5. the residual stream is unchanged; results are reproducible -----------------------------------------------
def test_forward_with_attention_keeps_the_stream():
    m, _ = _model(224, dict(S.SWIN_T_W7), seed=6)
    x = torch.randn(2, 56 * 56, 96, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    layer = m.layers[0]
    with torch.no_grad():
        y, maps = layer.forward_with_attention(x)
        ref = layer(x)
    assert len(maps) == 2 and tuple(maps[0].shape) == (128, 3, 49, 49)
    assert_close(y, ref, TOL_FP32_KERNEL, "stream")
    img = E.probe_images(2, 96, 3).cuda()
    a, b = m.forward_selfattention(img, 2), m.forward_selfattention(img, 2)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    tokens = m.patch_embed(img)
    assert all(torch.equal(p, q) for p, q in zip(a, m.forward_all_selfattention(tokens)))
    assert torch.equal(a[-1], m.forward_last_selfattention(tokens))


# ---- 6. invalid input --------------------------------------------------------------------------------------------
def test_invalid_input_raises():
    from esvit_b200 import ops
    m, _ = _model(112, dict(embed_dim=32, depths=(2, 2, 2), num_heads=(1, 2, 4), window_size=7))
    with pytest.raises(ValueError):
        m.forward_selfattention(torch.randn(1, 3, 96, 112, device="cuda"))
    with pytest.raises(ValueError):
        m.forward_selfattention(torch.randn(1, 3, 98, 98, device="cuda"))
    with pytest.raises(ValueError):
        m.forward_last_selfattention(torch.randn(1, 24 * 25, 32, device="cuda"))
    qkv = torch.zeros(1, 49, 3 * 64, dtype=torch.bfloat16, device="cuda")
    bias, table = torch.zeros(3 * 64, device="cuda"), torch.zeros(13 * 13, 2, device="cuda")
    for nH, ws, shift in ((2, 5, 0), (3, 7, 0), (2, 7, 7), (2, 7, -1)):
        with pytest.raises(ValueError):
            ops.window_attention_probs(qkv, bias, table, 7, 7, nH, ws, shift, 0.1)
