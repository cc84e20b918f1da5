"""Generate tests/golden/esvit_cvt.pt by RUNNING THE UNMODIFIED REFERENCE's CvT (models/cvt_v4_transformer.py).

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_cvt

A head-dim-64 CvT (dims 64/128/192/256, heads 1/2/3/4, depths 1/1/2/1, s1's kernels / strides / window 7) built by the
reference's get_cls_model layers (QuickGELU, LayerNorm eps 1e-5), seeded weights and BatchNorm buffers, seeded crops
2 x 224^2 + 2 x 96^2 at B = 2: the 96^2 maps are padded 24 -> 28 and 12 -> 14 and use windows 6 and 3.  Stored: the
dense train-mode forward (pooled, region, npatch) and the BatchNorm running statistics after it,
forward_return_n_last_blocks(x, 3, depth) in eval mode, and the training sequence of main_esvit.py:541-567 with
DINOHead heads at K = 4096 (teacher and student both in train mode, as main_esvit.py never calls .eval()): DDINOLoss
(dense) and DINOLoss (view) at epoch 1 -> the loss, the student's head outputs and every parameter gradient.  Tensors of
more than GD.SAMPLE elements are stored as a seeded sample.  oracle/cvt.py + oracle/losses.py are asserted against
every stored value while the file is written.
"""
from __future__ import annotations

import os
import sys
import warnings
from functools import partial

import torch
import torch.nn as nn

from . import cvt as O
from . import golden as GD
from . import losses as LO
from . import reference_import as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_cvt.pt")

SPEC = dict(INIT='trunc_norm', NUM_STAGES=4, REL_POS_EMBED=False, SHIFT=[False] * 4, DROP_PATH_RATE=0.0,
            PATCH_SIZE=[7, 3, 3, 3], PATCH_STRIDE=[4, 2, 2, 2], PATCH_PADDING=[2, 1, 1, 1], WINDOW_SIZE=[7] * 4,
            DIM_EMBED=[64, 128, 192, 256], NUM_HEADS=[1, 2, 3, 4], DEPTH=[1, 1, 2, 1], MLP_RATIO=[4.0] * 4,
            QKV_BIAS=[True] * 4, KERNEL_QKV=[3] * 4, PADDING_QKV=[1] * 4)
WEIGHT_SEED = 11
BATCH = 2
K = 4096
TEMP, STUDENT_TEMP = 0.04, 0.1
N_LAST = 3


def crops(seed: int):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(BATCH, 3, s, s, generator=g) for s in (224, 224, 96, 96)]


def seeded(rec, seed: int) -> dict:
    """GD.seeded_state_dict for the float tensors, with BatchNorm-shaped values: gamma 1 + N(0, 0.1), running mean
    N(0, 0.1), running var 1 + U(0, 1), num_batches_tracked 0"""
    fl = [r for r in rec if r[2]]
    sd = GD.seeded_state_dict(fl, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for name, shape, is_float in rec:
        if name.endswith("num_batches_tracked"):
            sd[name] = torch.zeros(shape, dtype=torch.long)
        elif name.endswith("running_mean"):
            sd[name] = torch.randn(shape, generator=g) * 0.1
        elif name.endswith("running_var"):
            sd[name] = 1 + torch.rand(shape, generator=g)
        elif ".bn.weight" in name:
            sd[name] = 1 + torch.randn(shape, generator=g) * 0.1
    return {name: sd[name] for name, _, _ in rec}


def reference_model(dense: bool, head: bool):
    ns = R.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import cvt_v4_transformer as ref_cvt  # noqa
        m = ref_cvt.CvT(num_classes=0, act_layer=ref_cvt.QuickGELU, norm_layer=partial(ref_cvt.LayerNorm, eps=1e-5),
                        init='trunc_norm', use_dense_prediction=dense, spec=dict(SPEC))
        if head:
            m.head = ns.DINOHead(SPEC["DIM_EMBED"][-1], K)
            if dense:
                m.head_dense = ns.DINOHead(SPEC["DIM_EMBED"][-1], K)
        else:
            m.head = nn.Identity()
            if dense:
                m.head_dense = nn.Identity()
    rec = GD.recipe(m.state_dict())
    sd = seeded(rec, WEIGHT_SEED)
    m.load_state_dict(sd)
    return m, rec, sd


def close(name, a, b, atol=2e-5):
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.allclose(b, a, atol=atol, rtol=0), (name, float((b - a).abs().max()))


def features_case(crop_seed: int) -> dict:
    m, rec, sd = reference_model(True, False)
    x = crops(crop_seed)
    m.train()
    with torch.no_grad():
        pooled, region, _, npatch = m(x)
    bufs = O.buffers(sd)
    with torch.no_grad():
        o_pooled, o_region, o_np = O.forward_dense(sd, bufs, x, True)
    assert list(npatch) == list(o_np), (npatch, o_np)
    close("pooled", pooled, o_pooled)
    close("region", region, o_region)
    ref_bufs = {k: v for k, v in m.state_dict().items() if k in bufs}
    for k, v in ref_bufs.items():
        close(k, v.double(), bufs[k].double(), 1e-6)
    m.eval()
    depth = SPEC["DEPTH"]
    with torch.no_grad():
        nlast = m.forward_return_n_last_blocks(torch.cat(x[:2]), N_LAST, False, depth)
        o_nlast = O.n_last_blocks(sd, {k: v.clone() for k, v in bufs.items()}, torch.cat(x[:2]), N_LAST)
    close("n_last", nlast, o_nlast)
    return dict(state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed, npatch=list(npatch),
                pooled=GD.sample(pooled, 0), region=GD.sample(region, 1),
                buffers={k: v.clone() for k, v in ref_bufs.items()}, n_last=GD.sample(nlast, 2))


def train_case(dense: bool, crop_seed: int) -> dict:
    ns = R.load()
    R.ensure_process_group()
    m, rec, sd = reference_model(dense, True)
    m.train()
    x = crops(crop_seed)
    ncrops = len(x)
    Loss = ns.DDINOLoss if dense else ns.DINOLoss
    loss_mod = Loss(K, ncrops, TEMP, TEMP, 0, 10, STUDENT_TEMP, 0.9)
    with torch.no_grad():
        t_out = m(x[:2])      # the teacher: the same weights, train-mode BN (its own running statistics are not stored)
    m.load_state_dict(sd)     # the student starts from the same buffers
    s_out = m(x)
    loss = loss_mod(s_out, t_out, 1, None)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

    osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running_" not in k and not k.endswith("weight_g"))
           for k, v in sd.items()}
    with torch.no_grad():
        ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, O.buffers(sd), x[:2], dense)
    os_ = O.multicrop_forward(osd, O.buffers(sd), x, dense)
    zero = torch.zeros(1, K)
    ol = LO.ddino_loss(os_, ot, zero, zero, ncrops, TEMP, STUDENT_TEMP) if dense else \
        LO.dino_loss(os_, ot, zero, ncrops, TEMP, STUDENT_TEMP)
    ol.backward()
    assert abs(float(ol) - float(loss)) <= 1e-5 * abs(float(loss)), (float(ol), float(loss))
    outs = list(s_out[:3]) if dense else [s_out]
    oouts = list(os_[:3]) if dense else [os_]
    for i, (a, b) in enumerate(zip(outs, oouts)):
        close(f"out{i}", a, b)
    assert set(grads) == {k for k, v in osd.items() if v.grad is not None}, set(grads) ^ {
        k for k, v in osd.items() if v.grad is not None}
    for k, g in grads.items():
        assert torch.allclose(osd[k].grad, g, atol=1e-6, rtol=1e-4), (k, float((osd[k].grad - g).abs().max()))
    return dict(dense=dense, state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed, loss=float(loss),
                outputs=[GD.sample(o, 10 + i) for i, o in enumerate(outs)],
                grads={k: GD.sample(g, 100 + i) for i, (k, g) in enumerate(sorted(grads.items()))})


def load(path: str = OUT) -> dict:
    """the fixture with each case's seeded weights and crops rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    for C in [G["features"]] + list(G["train"].values()):
        C["state_dict"] = seeded(C["state_recipe"], C["weight_seed"])
        C["crops"] = crops(C["crop_seed"])
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    out = dict(spec=SPEC, features=features_case(40), n_last=N_LAST,
               train={"ddino": train_case(True, 41), "dino": train_case(False, 42)}, K=K, temps=(TEMP, STUDENT_TEMP),
               generator="oracle/make_golden_cvt.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
