"""How far the UNMODIFIED reference CvT's own gradients move under bf16 autocast (what main_esvit.py runs with
--use_fp16) from its fp32 gradients, per parameter: the yardstick for the gradient gates of tests/test_cvt_gpu.py.

TEST INFRASTRUCTURE (needs a CUDA device and the reference under oracle/_ref/):

    python -m oracle.measure_cvt_autocast

Two cases, each the training sequence of main_esvit.py:541-567 (teacher and student in train mode, DDINOLoss):
  * fixture: the spec, seeded weights and crops of tests/golden/esvit_cvt.pt (train case "ddino"), K = 4096;
  * real: CvT-13 s1, K = 65 536, 2 + 8 crops at B = 2, seeded weights (oracle.make_golden_cvt.seeded).
Prints one JSON line per case: rel-L2(bf16-autocast grad, fp32 grad) of the attention PreNorm LayerNorm affine
(`layers.j.0.norm.*`), of stage0.0.proj.weight, and the median over all parameters.
"""
from __future__ import annotations

import json
import statistics
import sys
import warnings
from functools import partial

import torch

from . import make_golden_cvt as MG
from . import reference_import as R


def _grads(m, sd, x, K, autocast):
    ns = R.load()
    m.load_state_dict(sd)
    m.zero_grad(set_to_none=True)
    loss_mod = ns.DDINOLoss(K, len(x), MG.TEMP, MG.TEMP, 0, 10, MG.STUDENT_TEMP, 0.9).cuda()
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        with torch.no_grad():
            t = m(x[:2])
        m.load_state_dict(sd)
        s = m(x)
        loss = loss_mod(s, t, 1, None)
    loss.backward()
    return {k: p.grad.detach().double().clone() for k, p in m.named_parameters() if p.grad is not None}


def _case(spec, K, sd_seed, crops):
    ns = R.load()
    R.ensure_process_group()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import cvt_v4_transformer as ref_cvt  # noqa
        m = ref_cvt.CvT(num_classes=0, act_layer=ref_cvt.QuickGELU, norm_layer=partial(ref_cvt.LayerNorm, eps=1e-5),
                        init='trunc_norm', use_dense_prediction=True, spec=dict(spec, DROP_PATH_RATE=0.0))
        m.head = ns.DINOHead(spec["DIM_EMBED"][-1], K)
        m.head_dense = ns.DINOHead(spec["DIM_EMBED"][-1], K)
    sd = MG.seeded(MG.GD.recipe(m.state_dict()), sd_seed)
    m = m.cuda().train()
    sd = {k: v.cuda() for k, v in sd.items()}
    x = [c.cuda() for c in crops]
    g32 = _grads(m, sd, x, K, False)
    g16 = _grads(m, sd, x, K, True)
    rel = {k: float((g16[k] - g32[k]).norm() / g32[k].norm().clamp_min(1e-30)) for k in g32}
    ln = {k: v for k, v in rel.items() if ".1.layers." in k and (k.endswith(".0.norm.weight") or k.endswith(".0.norm.bias"))}
    return {"prenorm_ln_max": max(ln.values()), "prenorm_ln_median": statistics.median(ln.values()),
            "prenorm_ln_worst": max(ln, key=ln.get), "stage0_proj_weight": rel["stage0.0.proj.weight"],
            "median_all": statistics.median(rel.values()), "max_other": max(v for k, v in rel.items() if k not in ln)}


def main():
    if not (torch.cuda.is_available() and R.available()):
        sys.exit("needs a CUDA device and the reference under oracle/_ref/")
    from esvit_b200.cvt_v4_transformer import S1_SPEC
    G = MG.load()
    C = G["train"]["ddino"]
    print(json.dumps(dict(case="fixture", **_case(MG.SPEC, G["K"], C["weight_seed"], C["crops"]))))
    g = torch.Generator().manual_seed(5)
    crops = [torch.randn(2, 3, 224, 224, generator=g) for _ in range(2)] + \
            [torch.randn(2, 3, 96, 96, generator=g) for _ in range(8)]
    print(json.dumps(dict(case="real", **_case(S1_SPEC, 65536, 11, crops))))


if __name__ == "__main__":
    main()
