"""Generate tests/golden/esvit_vit.pt by RUNNING THE UNMODIFIED REFERENCE's VisionTransformer.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_vit

models.vision_transformer.VisionTransformer (head dim 64, 2 blocks, embed 128, 2 heads) at patch 16 and patch 8, with
seeded weights (oracle.golden.seeded_state_dict) and seeded crops: 2 x 224^2 + 2 x 96^2 at B = 2, so the local crops
exercise interpolate_pos_encoding.  Stored: the dense forward's cls and region features and npatch (:186-217), and
forward_return_n_last_blocks(x, 2, True) (:339-360) of the 224^2 crops.  Then the training sequence of main_esvit.py
:541-567 with DINOHead heads at K = 4096: teacher(crops[:2]) under no_grad, student(crops), the reference's DDINOLoss
(dense, `head` + `head_dense`) and DINOLoss (view, `head` only) at epoch 1, loss.backward(): the student's head
outputs, the loss and every parameter gradient.  Tensors of more than GD.SAMPLE elements are stored as a seeded sample.
oracle/vit.py + oracle/losses.py are asserted against every stored value while the file is written.
"""
from __future__ import annotations

import os
import sys
import warnings
from functools import partial

import torch
import torch.nn as nn

from . import golden as GD
from . import losses as LO
from . import reference_import as R
from . import vit as V

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_vit.pt")

SPEC = dict(embed_dim=128, depth=2, num_heads=2)
WEIGHT_SEED = 7
BATCH = 2
CASES = {"p16": 16, "p8": 8}  # name -> patch size
K = 4096
TEMP, STUDENT_TEMP = 0.04, 0.1      # teacher temperature at epoch 1 (warm-up 0 epochs), main_esvit.py defaults
TRAIN = {"ddino_p16": (16, True), "dino_p16": (16, False), "ddino_p8": (8, True)}  # name -> (patch, dense)


def crops(seed: int):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(BATCH, 3, s, s, generator=g) for s in (224, 224, 96, 96)]


def reference_model(patch: int):
    R.load()
    ref_vit = sys.modules["models.vision_transformer"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = ref_vit.VisionTransformer(patch_size=patch, mlp_ratio=4, qkv_bias=True,
                                      norm_layer=partial(nn.LayerNorm, eps=1e-6), use_dense_prediction=True, **SPEC)
    m.head, m.head_dense = nn.Identity(), nn.Identity()
    rec = GD.recipe(m.state_dict())
    sd = GD.seeded_state_dict(rec, WEIGHT_SEED)
    m.load_state_dict(sd)
    return m.eval(), rec, sd


def case(patch: int, crop_seed: int) -> dict:
    m, rec, sd = reference_model(patch)
    x = crops(crop_seed)
    with torch.no_grad():
        cls, region, _, npatch = m(x)
        o_cls, o_region, o_np = V.forward_dense(sd, x, patch, SPEC["num_heads"])
        nlast = m.forward_return_n_last_blocks(torch.cat(x[:2]), 2, True)
        o_nlast = V.n_last_blocks(sd, torch.cat(x[:2]), patch, SPEC["num_heads"], 2, True)
    assert list(npatch) == list(o_np), (npatch, o_np)
    for name, a, b in (("cls", cls, o_cls), ("region", region, o_region), ("n_last", nlast, o_nlast)):
        assert a.shape == b.shape, name
        assert torch.allclose(b, a, atol=2e-5, rtol=0), (name, float((b - a).abs().max()))
    return dict(patch=patch, state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed, npatch=list(npatch),
                cls=GD.sample(cls, 0), region=GD.sample(region, 1), n_last=GD.sample(nlast, 2))


def train_case(patch: int, dense: bool, crop_seed: int) -> dict:
    ns = R.load()
    R.ensure_process_group()
    ref_vit = sys.modules["models.vision_transformer"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = ref_vit.VisionTransformer(patch_size=patch, mlp_ratio=4, qkv_bias=True,
                                      norm_layer=partial(nn.LayerNorm, eps=1e-6), use_dense_prediction=dense, **SPEC)
        m.head = ns.DINOHead(SPEC["embed_dim"], K)
        if dense:
            m.head_dense = ns.DINOHead(SPEC["embed_dim"], K)
    rec = GD.recipe(m.state_dict())
    sd = GD.seeded_state_dict(rec, WEIGHT_SEED)
    m.load_state_dict(sd)
    m.train()
    x = crops(crop_seed)
    ncrops = len(x)
    Loss = ns.DDINOLoss if dense else ns.DINOLoss
    loss_mod = Loss(K, ncrops, TEMP, TEMP, 0, 10, STUDENT_TEMP, 0.9)
    with torch.no_grad():
        t_out = m(x[:2])
    s_out = m(x)
    loss = loss_mod(s_out, t_out, 1, None)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

    osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g")) for k, v in sd.items()}
    with torch.no_grad():
        ot = V.multicrop_forward({k: v.detach() for k, v in osd.items()}, x[:2], patch, SPEC["num_heads"], dense)
    os_ = V.multicrop_forward(osd, x, patch, SPEC["num_heads"], dense)
    zero = torch.zeros(1, K)
    if dense:
        ol = LO.ddino_loss(os_, ot, zero, zero, ncrops, TEMP, STUDENT_TEMP)
    else:
        ol = LO.dino_loss(os_, ot, zero, ncrops, TEMP, STUDENT_TEMP)
    ol.backward()
    assert abs(float(ol) - float(loss)) <= 1e-5 * abs(float(loss)), (float(ol), float(loss))
    outs = list(s_out[:3]) if dense else [s_out]
    oouts = list(os_[:3]) if dense else [os_]
    for i, (a, b) in enumerate(zip(outs, oouts)):
        assert torch.allclose(b, a, atol=2e-5, rtol=0), (i, float((b - a).abs().max()))
    assert set(grads) == {k for k, v in osd.items() if v.grad is not None}
    for k, g in grads.items():
        assert torch.allclose(osd[k].grad, g, atol=1e-6, rtol=1e-4), (k, float((osd[k].grad - g).abs().max()))
    return dict(patch=patch, dense=dense, state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed,
                loss=float(loss), outputs=[GD.sample(o, 10 + i) for i, o in enumerate(outs)],
                grads={k: GD.sample(g, 100 + i) for i, (k, g) in enumerate(sorted(grads.items()))})


def load(path: str = OUT) -> dict:
    """the fixture with each case's seeded weights and crops rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    for C in G["cases"].values():
        C["state_dict"] = GD.seeded_state_dict(C["state_recipe"], C["weight_seed"])
        C["crops"] = crops(C["crop_seed"])
    for C in G["train"].values():
        C["state_dict"] = GD.seeded_state_dict(C["state_recipe"], C["weight_seed"])
        C["crops"] = crops(C["crop_seed"])
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    out = dict(spec=SPEC, cases={name: case(p, 20 + i) for i, (name, p) in enumerate(CASES.items())},
               train={name: train_case(p, d, 30 + i) for i, (name, (p, d)) in enumerate(TRAIN.items())},
               K=K, temps=(TEMP, STUDENT_TEMP),
               generator="oracle/make_golden_vit.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
