"""Generate tests/golden/esvit_vil.pt by RUNNING THE UNMODIFIED REFERENCE's Vision Longformer (models/vision_longformer.py
MsViT with layers/longformer2d.py).

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/; needs `einops`):

    python -m oracle.make_golden_vil

A reduced vil_2262 (ARCH below: every stage kind, head dim 32, MODE 1, the vil_small base.yaml switches, DROP_PATH 0)
with seeded weights, seeded crops 2 x 224^2 + 4 x 96^2 at B = 2.  `random.randrange` is wrapped with a seeded generator
so the sliding-chunk modes the reference draws are reproducible; every drawn sequence is stored.  Stored: the dense
train-mode forward (x_cls, region, npatch), forward_return_n_last_blocks(x, 3, depth) in eval mode (stage-3 global-row
taps and the stage-4 tap), and the training sequence of main_esvit.py:541-567 with DINOHead heads at K = 4096 (teacher
and student in train mode, as main_esvit.py never calls .eval()): DDINOLoss (dense) and DINOLoss (view) at epoch 1 ->
loss, the student's head outputs and every parameter gradient.  Tensors of more than GD.SAMPLE elements are stored as a
seeded sample.  oracle/vil.py + oracle/losses.py are asserted against every stored value while the file is written.
"""
from __future__ import annotations

import os
import random
import sys
import warnings

import torch
import torch.nn as nn

from . import golden as GD
from . import losses as LO
from . import reference_import as R
from . import vil as O

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_vil.pt")

ARCH = 'l1,h1,d32,n1,s1,g1,p4,f7,a0_l2,h2,d64,n1,s1,g1,p2,f7,a0_l3,h3,d96,n2,s0,g1,p2,f7,a0_l4,h4,d128,n1,s0,g0,p2,f7,a0'
ARGS = dict(arch=ARCH, img_size=224, drop_rate=0.0, drop_path_rate=0.0, norm_embed=True, avg_pool=False, sharew=True,
            attn_type='longformerhand', share_kv=True, only_glo=False, sw_exact=0, ln_eps=1e-6, mode=1,
            pool_method=None, with_se=False)
OUT_DIM = 128
WEIGHT_SEED = 21
BATCH = 2
K = 4096
TEMP, STUDENT_TEMP = 0.04, 0.1
N_LAST = 3
DEPTH = [1, 1, 2, 1]


def crops(seed: int):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(BATCH, 3, s, s, generator=g) for s in (224, 224, 96, 96, 96, 96)]


def reference_model(dense: bool, head: bool):
    ns = R.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import vision_longformer as RV  # noqa
        m = RV.MsViT(num_classes=0, use_dense_prediction=dense, **ARGS)
        if head:
            m.head = ns.DINOHead(OUT_DIM, K)
            if dense:
                m.head_dense = ns.DINOHead(OUT_DIM, K)
        else:
            m.head = nn.Identity()
            if dense:
                m.head_dense = nn.Identity()
    rec = GD.recipe(m.state_dict())
    sd = O.seeded(rec, WEIGHT_SEED)
    m.load_state_dict(sd, strict=True)
    return m, rec, sd


class Draws:
    """random.randrange replaced by a seeded generator that records what the reference draws"""

    def __init__(self, seed: int):
        self.rng, self.seq = random.Random(seed), []

    def __enter__(self):
        self.orig = random.randrange

        def draw(a, b):
            v = self.rng.randrange(a, b)
            self.seq.append(v)
            return v
        random.randrange = draw
        return self

    def __exit__(self, *exc):
        random.randrange = self.orig


def close(name, a, b, atol=2e-5):
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.allclose(b, a, atol=atol, rtol=0), (name, float((b - a).abs().max()))


def features_case(crop_seed: int) -> dict:
    m, rec, sd = reference_model(True, False)
    x = crops(crop_seed)
    m.train()
    with Draws(crop_seed) as d, torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cls, region, _, npatch = m(x)
    with torch.no_grad():
        o_cls, o_region, o_np = O.forward_dense(sd, x, iter(d.seq), True)
    assert list(npatch) == list(o_np) == [49, 9], (npatch, o_np)
    close("x_cls", cls, o_cls)
    close("region", region, o_region)
    m.eval()
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nlast = m.forward_return_n_last_blocks(torch.cat(x[:2]), N_LAST, False, DEPTH)
        o_nlast = O.n_last_blocks(sd, torch.cat(x[:2]), N_LAST)
    close("n_last", nlast, o_nlast)
    return dict(state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed, modes=list(d.seq), npatch=list(npatch),
                x_cls=GD.sample(cls, 0), region=GD.sample(region, 1), n_last=GD.sample(nlast, 2))


def train_case(dense: bool, crop_seed: int) -> dict:
    ns = R.load()
    R.ensure_process_group()
    m, rec, sd = reference_model(dense, True)
    m.train()
    x = crops(crop_seed)
    ncrops = len(x)
    Loss = ns.DDINOLoss if dense else ns.DINOLoss
    loss_mod = Loss(K, ncrops, TEMP, TEMP, 0, 10, STUDENT_TEMP, 0.9)
    with Draws(crop_seed) as d, warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with torch.no_grad():
            t_out = m(x[:2])          # the teacher: the same weights, train mode
        n_teacher = len(d.seq)
        s_out = m(x)
    loss = loss_mod(s_out, t_out, 1, None)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}

    osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g")) for k, v in sd.items()}
    with torch.no_grad():
        ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, x[:2], dense, iter(d.seq[:n_teacher]))
    os_ = O.multicrop_forward(osd, x, dense, iter(d.seq[n_teacher:]))
    zero = torch.zeros(1, K)
    ol = LO.ddino_loss(os_, ot, zero, zero, ncrops, TEMP, STUDENT_TEMP) if dense else \
        LO.dino_loss(os_, ot, zero, ncrops, TEMP, STUDENT_TEMP)
    ol.backward()
    assert abs(float(ol) - float(loss)) <= 1e-5 * abs(float(loss)), (float(ol), float(loss))
    outs = list(s_out[:3]) if dense else [s_out]
    oouts = list(os_[:3]) if dense else [os_]
    for i, (a, b) in enumerate(zip(outs, oouts)):
        close(f"out{i}", a, b)
    named = dict(m.named_parameters())   # the aliased *_global modules are one parameter under its first name
    ograds = {k: osd[k].grad for k in named if osd[k].grad is not None}
    assert set(grads) == set(ograds), set(grads) ^ set(ograds)
    for k, g in grads.items():
        assert torch.allclose(ograds[k], g, atol=1e-6, rtol=1e-4), (k, float((ograds[k] - g).abs().max()))
    return dict(dense=dense, state_recipe=rec, weight_seed=WEIGHT_SEED, crop_seed=crop_seed, modes=list(d.seq),
                n_teacher_modes=n_teacher, loss=float(loss), outputs=[GD.sample(o, 10 + i) for i, o in enumerate(outs)],
                grads={k: GD.sample(g, 100 + i) for i, (k, g) in enumerate(sorted(grads.items()))})


def load(path: str = OUT) -> dict:
    """the fixture with each case's seeded weights and crops rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    for C in [G["features"]] + list(G["train"].values()):
        C["state_dict"] = O.seeded(C["state_recipe"], C["weight_seed"])
        C["crops"] = crops(C["crop_seed"])
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    torch.set_num_threads(1)  # the table gradient's index backward sums in thread order: one thread, one order
    out = dict(args=ARGS, depth=DEPTH, features=features_case(50), n_last=N_LAST,
               train={"ddino": train_case(True, 51), "dino": train_case(False, 52)}, K=K, temps=(TEMP, STUDENT_TEMP),
               generator="oracle/make_golden_vil.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
