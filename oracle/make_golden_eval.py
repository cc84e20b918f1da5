"""Generate tests/golden/esvit_eval.pt by RUNNING THE UNMODIFIED REFERENCE's evaluation code.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_eval

  * probe: the reference's SwinTransformer.forward_return_n_last_blocks (models/swin_transformer.py:799-837) on the
    SMALL spec of make_golden.py (112^2, depths 2/2/2) with seeded weights (oracle.golden.seeded_state_dict) and seeded
    images, for n in {1, 2, 3, 6};
  * knn: eval_knn.knn_classifier (eval_knn.py:193-232), AST-extracted, on seeded clustered features (4000 train x 64,
    300 test - its 100 chunks need at least 100 test rows -, 50 classes), k in {10, 20, 100, 200}, T = 0.07, on CPU
    with Tensor.cuda mapped to identity; plus the top-200 indices of the reference's expression
    ``torch.mm(test, train.t()).topk(k, largest=True, sorted=True)`` (eval_knn.py:209-210).

Features and weights are regenerated from their seeds on load.  oracle/eval.py is asserted against every stored value
while the file is written.
"""
from __future__ import annotations

import os
import sys
import warnings
from functools import partial

import torch
import torch.nn as nn

from . import eval as E
from . import golden as GD
from . import reference_import as R
from . import swin as S
from .make_golden import SMALL, WEIGHT_SEED

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_eval.pt")

PROBE_NS = (1, 2, 3, 6)
IMAGE_SEED, BATCH = 7, 2
# 50 classes: with 20, two test rows at k = 10 have a true class of score 0 and fewer than 5 classes of positive score,
# so whether they are top-5 hits depends on how the reference's unstable descending sort orders equal (zero) scores
KNN = dict(seed=3, n_train=4000, n_test=300, dim=64, num_classes=50, noise=3.0)
KS = (10, 20, 100, 200)
TEMP = 0.07


def probe():
    ns = R.load()
    spec = S.SwinSpec(**SMALL)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m = ns.SwinTransformer(img_size=spec.img_size, in_chans=3, num_classes=0, patch_size=spec.patch_size,
                               embed_dim=spec.embed_dim, depths=list(spec.depths), num_heads=list(spec.num_heads),
                               window_size=spec.window_size, mlp_ratio=spec.mlp_ratio, qkv_bias=True, drop_rate=0.0,
                               attn_drop_rate=0.0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                               ape=False, patch_norm=True)
    rec = GD.recipe(m.state_dict())
    sd = GD.seeded_state_dict(rec, WEIGHT_SEED)
    m.load_state_dict(sd)
    m.eval()
    x = E.probe_images(BATCH, spec.img_size, IMAGE_SEED)
    feats = {}
    with torch.no_grad():
        for n in PROBE_NS:
            f = m.forward_return_n_last_blocks(x, n, False, list(spec.depths))
            o = E.n_last_blocks(x, sd, spec, n)
            assert f.shape == o.shape and torch.allclose(o, f, atol=2e-5, rtol=0), (n, float((o - f).abs().max()))
            feats[n] = f.clone()
    return dict(spec=dict(SMALL), state_recipe=rec, weight_seed=WEIGHT_SEED, image_seed=IMAGE_SEED, batch=BATCH,
                features=feats)


def knn():
    ref = E.reference_knn_classifier()
    xtr, ytr, xte, yte = E.clustered_features(**KNN)
    acc = {}
    with E.cpu_cuda_shim():
        for k in KS:
            # no row's top-5 outcome may depend on the order of tied scores, which the reference leaves unspecified
            sims, idx = E.knn_topk(xtr, xte, k)
            probs = torch.zeros(len(yte), KNN["num_classes"]).scatter_add_(1, ytr[idx], sims.div(TEMP).exp())
            tied = (probs.gather(1, yte.view(-1, 1)).view(-1) == 0) & ((probs > 0).sum(1) < 5)
            assert not bool(tied.any()), (k, int(tied.sum()))
            acc[k] = ref(xtr, ytr, xte, yte, k, TEMP, KNN["num_classes"])
            o = E.knn_classifier(xtr, ytr, xte, yte, k, TEMP, KNN["num_classes"])
            assert o == acc[k], (k, o, acc[k])
    kmax = max(KS)
    _, idx = torch.mm(xte, xtr.t()).topk(kmax, largest=True, sorted=True)
    _, oidx = E.knn_topk(xtr, xte, kmax)
    assert torch.equal(idx, oidx)
    return dict(params=dict(KNN), ks=list(KS), T=TEMP, accuracy=acc, idx=idx.to(torch.int16))


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    out = dict(probe=probe(), knn=knn(),
               generator="oracle/make_golden_eval.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB; accuracy", out["knn"]["accuracy"])
