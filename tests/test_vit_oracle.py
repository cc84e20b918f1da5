"""CPU: oracle.vit reproduces what the UNMODIFIED reference's VisionTransformer produced (tests/golden/esvit_vit.pt,
written by oracle/make_golden_vit.py): the dense multi-crop forward and forward_return_n_last_blocks at patch 16 and 8."""
import os

import pytest
import torch

from oracle import golden as GD
from oracle import make_golden_vit as MG
from oracle import vit as V


@pytest.fixture(scope="module")
def G():
    return MG.load()


def test_fixture_is_small():
    assert os.path.getsize(MG.OUT) < 1 << 20


@pytest.mark.parametrize("name", ["p16", "p8"])
def test_oracle_matches_reference(G, name):
    C = G["cases"][name]
    nH = G["spec"]["num_heads"]
    with torch.no_grad():
        cls, region, npatch = V.forward_dense(C["state_dict"], C["crops"], C["patch"], nH)
        nlast = V.n_last_blocks(C["state_dict"], torch.cat(C["crops"][:2]), C["patch"], nH, 2, True)
    assert npatch == C["npatch"]
    for key, a in (("cls", cls), ("region", region), ("n_last", nlast)):
        a, r = GD.at_golden(a, C[key])
        assert torch.allclose(a, r, atol=2e-5, rtol=0), (key, float((a - r).abs().max()))


def test_state_dict_interchanges_with_reference(G):
    """the port's state_dict has exactly the reference's keys and shapes (the fixture's recipe is the reference's
    state_dict layout), and loads the reference's weights with strict=True"""
    from functools import partial

    import torch.nn as nn

    from esvit_b200 import vision_transformer as VT
    for C in G["cases"].values():
        m = VT.VisionTransformer(patch_size=C["patch"], mlp_ratio=4, qkv_bias=True,
                                 norm_layer=partial(nn.LayerNorm, eps=1e-6), **G["spec"])
        assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, s) for k, s, _ in C["state_recipe"]]
        m.load_state_dict(C["state_dict"], strict=True)
    for f, D in ((VT.deit_tiny, 192), (VT.deit_small, 384), (VT.vit_base, 768)):
        assert f(patch_size=16).embed_dim == D


@pytest.mark.parametrize("name", ["ddino_p16", "dino_p16", "ddino_p8"])
def test_oracle_training_step_matches_reference(G, name):
    """DINOHead heads at K = 4096 and the reference's DDINOLoss / DINOLoss: head outputs, loss and every parameter
    gradient of the oracle (oracle/vit.py + oracle/losses.py) against the reference's own backward"""
    from oracle import losses as LO
    C = G["train"][name]
    nH, K = G["spec"]["num_heads"], G["K"]
    temp, stemp = G["temps"]
    x = C["crops"]
    sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g"))
          for k, v in C["state_dict"].items()}
    with torch.no_grad():
        t = V.multicrop_forward({k: v.detach() for k, v in sd.items()}, x[:2], C["patch"], nH, C["dense"])
    s = V.multicrop_forward(sd, x, C["patch"], nH, C["dense"])
    zero = torch.zeros(1, K)
    if C["dense"]:
        loss = LO.ddino_loss(s, t, zero, zero, len(x), temp, stemp)
    else:
        loss = LO.dino_loss(s, t, zero, len(x), temp, stemp)
    loss.backward()
    assert abs(float(loss) - C["loss"]) <= 1e-5 * abs(C["loss"])
    for i, o in enumerate(list(s[:3]) if C["dense"] else [s]):
        a, r = GD.at_golden(o.detach(), C["outputs"][i])
        assert torch.allclose(a, r, atol=2e-5, rtol=0), i
    assert sorted(C["grads"]) == sorted(k for k, v in sd.items() if v.grad is not None)
    for k, ref in C["grads"].items():
        a, r = GD.at_golden(sd[k].grad, ref)
        assert torch.allclose(a, r, atol=1e-6, rtol=1e-4), (k, float((a - r).abs().max()))
