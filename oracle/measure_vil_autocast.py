"""How far the UNMODIFIED reference Vision Longformer moves under bf16 autocast (what main_esvit.py runs with
--use_fp16) from its own fp32 run: the yardstick for the gates of tests/test_vil_gpu.py.

TEST INFRASTRUCTURE (needs a CUDA device, the reference under oracle/_ref/ and `einops`):

    python -m oracle.measure_vil_autocast

Two cases, the sliding-chunk modes forced to the same sequence in both runs:
  * fixture: the reduced arch, seeded weights, crops and recorded modes of tests/golden/esvit_vil.pt (train case
    "ddino"), the training sequence of main_esvit.py:541-567 at K = 4096 -> rel-L2(bf16-autocast grad, fp32 grad) per
    parameter: the relative-position bias parameters (`g2l` / `g2g` / tables), and the largest over all others;
  * real: vil_2262 with the seeded weights of tests/test_vil_gpu.py (seed 5), one 224^2 + one 96^2 crop, train-mode
    dense forward -> rel-L2 of x_cls and x_region.
Prints one JSON line per case.
"""
from __future__ import annotations

import json
import random
import statistics
import sys
import warnings

import torch

from . import golden as GD
from . import make_golden_vil as MG
from . import reference_import as R
from . import vil as O


def _forced(seq):
    it = iter(seq)
    orig = random.randrange
    random.randrange = lambda a, b: next(it)
    return orig


def _ref(args, dense=True, head_k=None):
    ns = R.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import vision_longformer as RV  # noqa
        m = RV.MsViT(num_classes=0, use_dense_prediction=dense, **args)
        if head_k:
            m.head = ns.DINOHead(m.out_planes, head_k)
            m.head_dense = ns.DINOHead(m.out_planes, head_k)
        else:
            m.head = torch.nn.Identity()
            m.head_dense = torch.nn.Identity()
    return m


def _grads(m, sd, x, K, seq, autocast):
    ns = R.load()
    m.load_state_dict(sd)
    m.zero_grad(set_to_none=True)
    loss_mod = ns.DDINOLoss(K, len(x), MG.TEMP, MG.TEMP, 0, 10, MG.STUDENT_TEMP, 0.9).cuda()
    orig = _forced(seq)
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            with torch.no_grad():
                t = m(x[:2])
            s = m(x)
            loss = loss_mod(s, t, 1, None)
    finally:
        random.randrange = orig
    loss.backward()
    return {k: p.grad.detach().double().clone() for k, p in m.named_parameters() if p.grad is not None}


def fixture_case():
    R.ensure_process_group()
    G = MG.load()
    C = G["train"]["ddino"]
    m = _ref(MG.ARGS, head_k=G["K"]).cuda().train()
    sd = {k: v.cuda() for k, v in C["state_dict"].items()}
    x = [c.cuda() for c in C["crops"]]
    g32 = _grads(m, sd, x, G["K"], C["modes"], False)
    g16 = _grads(m, sd, x, G["K"], C["modes"], True)
    rel = {k: float((g16[k] - g32[k]).norm() / g32[k].norm().clamp_min(1e-30)) for k in g32}
    rpb = {k: v for k, v in rel.items() if "relative_position" in k}
    other = {k: v for k, v in rel.items() if k not in rpb}
    return {"rel_pos_bias_max": max(rpb.values()), "rel_pos_bias_worst": max(rpb, key=rpb.get),
            "rel_pos_bias": {k: round(v, 4) for k, v in sorted(rpb.items())},
            "other_max": max(other.values()), "other_worst": max(other, key=other.get),
            "median_all": statistics.median(rel.values())}


def real_case():
    from esvit_b200.vision_longformer import VIL_2262
    m = _ref(dict(VIL_2262, drop_path_rate=0.0))
    sd = O.seeded(GD.recipe(m.state_dict()), 5)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    g = torch.Generator().manual_seed(5)
    x = [torch.randn(1, 3, 224, 224, generator=g).cuda(), torch.randn(1, 3, 96, 96, generator=g).cuda()]
    seq = [2, 7, 4, 6, 1, 8, 3, 5]
    out = {}
    for ac in (False, True):
        orig = _forced(seq)
        try:
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                o = m(x)
        finally:
            random.randrange = orig
        out[ac] = (o[0].double(), o[2].double())
    return {name: float((out[True][i] - out[False][i]).norm() / out[False][i].norm())
            for i, name in enumerate(("x_cls", "x_region"))}


def main():
    if not (torch.cuda.is_available() and R.available()):
        sys.exit("needs a CUDA device and the reference under oracle/_ref/")
    print(json.dumps(dict(case="fixture", **fixture_case())))
    print(json.dumps(dict(case="real", **real_case())))


if __name__ == "__main__":
    main()
