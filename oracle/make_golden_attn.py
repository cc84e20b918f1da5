"""Generate tests/golden/esvit_attn.pt by RUNNING THE UNMODIFIED REFERENCE's SwinTransformer.forward_selfattention.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_attn

forward_selfattention(x, 1) and (x, 2) (models/swin_transformer.py:766-796) of the SMALL (ws 7) and SMALL_W14 specs of
make_golden.py, both built at img_size 112, with seeded weights (oracle.golden.seeded_state_dict) and seeded images:
  * 112^2: shifted windows, the single clamped window of the last stage and (W14) the un-shifted ws-14 stage 1;
  * 96^2 (the local-crop geometry): maps of 24 -> 28, 12 -> 14 and 6 -> 7 tokens, so padded slots under a shift mask.
Maps of more than GD.SAMPLE elements are stored as a seeded sample.  oracle/attn.py is asserted against every stored
value while the file is written.
"""
from __future__ import annotations

import os
import sys
import warnings
from functools import partial

import torch
import torch.nn as nn

from . import attn as A
from . import eval as E
from . import golden as GD
from . import reference_import as R
from . import swin as S
from .make_golden import SMALL, SMALL_W14, WEIGHT_SEED

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_attn.pt")

BATCH = 2
CASES = {  # name -> (spec, input side, image seed)
    "w7_112": (SMALL, 112, 11),
    "w7_96": (SMALL, 96, 12),
    "w14_112": (SMALL_W14, 112, 13),
    "w14_96": (SMALL_W14, 96, 14),
}
NS = (1, 2)


def reference_model(small: dict):
    ns = R.load()
    spec = S.SwinSpec(**small)
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
    return m.eval(), spec, rec, sd


def case(small: dict, side: int, image_seed: int) -> dict:
    m, spec, rec, sd = reference_model(small)
    x = E.probe_images(BATCH, side, image_seed)
    maps = {}
    with torch.no_grad():
        for n in NS:
            ref = m.forward_selfattention(x, n)
            o = A.selfattention(x, sd, spec, n)
            refs, os_ = ([ref], [o]) if n == 1 else (ref, o)
            assert len(refs) == len(os_) == (1 if n == 1 else sum(spec.depths)), n
            for i, (a, b) in enumerate(zip(refs, os_)):
                assert a.shape == b.shape and a.dtype == b.dtype == torch.float32, (n, i)
                assert torch.allclose(b, a, atol=2e-5, rtol=0), (n, i, float((b - a).abs().max()))
            maps[n] = [GD.sample(a, seed=i) for i, a in enumerate(refs)]
    return dict(spec=dict(small), state_recipe=rec, weight_seed=WEIGHT_SEED, side=side, image_seed=image_seed,
                batch=BATCH, maps=maps)


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    out = dict(cases={name: case(*c) for name, c in CASES.items()},
               generator="oracle/make_golden_attn.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
