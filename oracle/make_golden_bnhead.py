"""Generate tests/golden/esvit_bnhead.pt by RUNNING THE UNMODIFIED REFERENCE with DINOHead(use_bn=True) heads.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_bnhead

Three cases, every head built with use_bn=True (main_esvit.py:336-358 with --use_bn_in_head True), single process, so
the BatchNorm1d layers stay BatchNorm1d:
  * swin_dense: oracle/make_golden.py's small Swin (SMALL, HEAD, K), DDINOLoss, 2 x 112^2 + 3 x 48^2 crops at B = 2;
  * swin_view:  the same backbone, DINOLoss, the two global crops;
  * vit_dense:  oracle/make_golden_vit.py's ViT (SPEC) at patch 16, DDINOLoss, 2 x 224^2 + 2 x 96^2 crops at B = 2.
Each runs make_golden.reference_steps (main_esvit.py:541-590 on CPU fp32: teacher and student in train mode, loss,
backward, clip, cancel last layer, AdamW, EMA) for NSTEPS steps.  Stored per step: the loss, the student and teacher head
outputs, the raw student gradients (seeded samples of the head gradients, (sum, norm) of all), the running statistics
of every student and teacher BatchNorm1d after the step.  Then one eval-mode output of the student `head`: the initial
weights with the running statistics after the last step, on seeded rows.  oracle/bnhead.py is asserted against every
stored value while the file is written.
"""
from __future__ import annotations

import os
import sys
import warnings
from functools import partial

import torch
import torch.nn as nn

from . import bnhead as BH
from . import golden as GD
from . import make_golden as MG
from . import make_golden_vit as MV
from . import reference_import as R
from . import step as ST
from . import swin as S

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_bnhead.pt")

NSTEPS = 2
WEIGHT_SEED = 11
EVAL_ROWS, EVAL_SEED = 16, 5
GRAD_ATOL = 1e-4  # of the largest gradient norm
CASES = {"swin_dense": ("swin", True), "swin_view": ("swin", False), "vit_dense": ("vit", True)}


def crops(kind: str, dense: bool):
    if kind == "vit":
        return MV.crops(30)
    c = ST.synthetic_crops(2, 3, seed=1234, global_size=112, local_size=48)
    return c if dense else c[:2]


def arch(kind: str, dense: bool) -> dict:
    if kind == "vit":
        return {"kind": "vit", "patch": 16, "num_heads": MV.SPEC["num_heads"]}
    return {"kind": "swin", "spec": S.SwinSpec(use_dense_prediction=dense, **MG.SMALL)}


def reference_model(kind: str, dense: bool):
    ns = R.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if kind == "vit":
            ref_vit = sys.modules["models.vision_transformer"]
            m = ref_vit.VisionTransformer(patch_size=16, mlp_ratio=4, qkv_bias=True,
                                          norm_layer=partial(nn.LayerNorm, eps=1e-6), use_dense_prediction=dense,
                                          **MV.SPEC)
        else:
            m = R.build_swin(arch(kind, dense)["spec"], MG.K)
        m.head = ns.DINOHead(m.num_features, MG.K, use_bn=True, **MG.HEAD)
        if dense:
            m.head_dense = ns.DINOHead(m.num_features, MG.K, use_bn=True, **MG.HEAD)
    return m


def _close(a: torch.Tensor, b: torch.Tensor, tol: float, name: str, atol: float = 0.0) -> None:
    """||a - b|| < tol ||b|| + atol"""
    d, n = float((a.double() - b.double()).norm()), float(b.double().norm())
    assert d < tol * n + atol, (name, d, n)


def case(kind: str, dense: bool) -> dict:
    ns = R.load()
    R.ensure_process_group()
    student, teacher = reference_model(kind, dense), reference_model(kind, dense)
    rec = GD.recipe(student.state_dict())
    sd0 = BH.seeded_state_dict(rec, WEIGHT_SEED)
    student.load_state_dict(sd0)
    teacher.load_state_dict(sd0)
    student.train()
    teacher.train()
    for p in teacher.parameters():
        p.requires_grad = False
    x = crops(kind, dense)
    ncrops = len(x)
    Loss = ns.DDINOLoss if dense else ns.DINOLoss
    loss_mod = Loss(MG.K, ncrops, 0.04, MG.HP["teacher_temp"], 0, 10, MG.HP["student_temp"], MG.HP["center_momentum"])
    # the running statistics after each step: every BatchNorm1d runs once per network forward
    seen = {}
    for net, tag in ((student, "student"), (teacher, "teacher")):
        for name, mod in net.named_modules():
            if isinstance(mod, nn.BatchNorm1d):
                mod.register_forward_hook(lambda m, i, o, key=(tag, name): seen.setdefault(key, []).append(
                    {b: getattr(m, b).detach().clone() for b in ("running_mean", "running_var", "num_batches_tracked")}))
    ref = MG.reference_steps(ns, student, teacher, loss_mod, x, NSTEPS, dense)
    run = [{f"{net}.{name}.{b}": v for (net, name), lst in seen.items() for b, v in lst[it].items()}
           for it in range(NSTEPS)]

    # ---- the oracle must reproduce all of it ----------------------------------------------------------------------
    hp = {k: v for k, v in MG.HP.items()}
    orc = BH.OracleBnStep(sd0, arch(kind, dense), dense, ncrops, MG.K, **hp)
    steps = []
    for it in range(NSTEPS):
        r = ref[it]
        lo, so, to, go = orc.step(x, epoch=0)
        # step 0 runs on identical weights; later steps on AdamW updates that agree to ~lr where a gradient is ~0
        tol = 2e-5 if it == 0 else 2e-3
        assert abs(lo - r["loss"]) < tol * max(1.0, abs(r["loss"])), (kind, it, lo, r["loss"])
        s_ref = list(r["student_output"][:2]) if dense else [r["student_output"]]
        t_ref = list(r["teacher_output"][:2]) if dense else [r["teacher_output"]]
        s_orc = list(so[:2]) if dense else [so]
        t_orc = list(to[:2]) if dense else [to]
        for i, (a, b) in enumerate(zip(s_orc + t_orc, s_ref + t_ref)):
            _close(a.detach(), b.detach(), 1e-5 if it == 0 else 2e-3, f"{kind} step {it} output {i}")
        assert set(go) == set(r["grads"]), (kind, set(go) ^ set(r["grads"]))
        gmax = max(float(g.norm()) for g in r["grads"].values())
        for k, g in r["grads"].items():
            # atol: gradients the head BNs cancel (a shift common to all rows, e.g. the final norm's bias) are
            # rounding noise in both
            _close(go[k], g, 1e-4 if it == 0 else 2e-2, f"{kind} step {it} grad {k}", atol=GRAD_ATOL * gmax)
        o_run = {f"{net}.{k}": v for net, d in (("student", orc.student), ("teacher", orc.teacher))
                 for k, v in BH.running_stats(d).items()}
        assert set(o_run) == set(run[it]), set(o_run) ^ set(run[it])
        for k, v in run[it].items():
            if v.dtype == torch.long:
                assert torch.equal(o_run[k], v), k
            else:
                _close(o_run[k], v, 1e-5 if it == 0 else 2e-3, f"{kind} step {it} {k}")
        heads = [k for k in r["grads"] if k.startswith("head")]
        steps.append(dict(
            loss=r["loss"],
            student_outputs=[GD.sample(o, 10 + i) for i, o in enumerate(s_ref)],
            teacher_outputs=[GD.sample(o, 20 + i) for i, o in enumerate(t_ref)],
            grads_stats=MG.stats(r["grads"]),
            grads_head={k: GD.sample(r["grads"][k], 100 + i) for i, k in enumerate(sorted(heads))},
            running={k: v.clone() for k, v in run[it].items()}))

    # ---- eval mode: the initial `head` with the running statistics of the last step ---------------------------------
    rows = torch.randn(EVAL_ROWS, student.num_features, generator=torch.Generator().manual_seed(EVAL_SEED))
    head_sd = {k[len("head."):]: v for k, v in sd0.items() if k.startswith("head.")}
    for k in head_sd:
        if k.endswith(BH.BUFFERS):
            head_sd[k] = run[-1]["student.head." + k]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        h = ns.DINOHead(student.num_features, MG.K, use_bn=True, **MG.HEAD)
    h.load_state_dict(head_sd)
    with torch.no_grad():
        ev = h.eval()(rows)
        o_ev = BH.dino_head_bn(rows, {"head." + k: v.clone() for k, v in head_sd.items()}, "head", train=False)
    _close(o_ev, ev, 1e-5, f"{kind} eval output")
    return dict(kind=kind, dense=dense, ncrops=ncrops, state_recipe=rec, weight_seed=WEIGHT_SEED, steps=steps,
                eval_rows=EVAL_ROWS, eval_seed=EVAL_SEED, eval_output=GD.sample(ev, 30))


def load(path: str = OUT) -> dict:
    """the fixture with each case's seeded weights, crops, architecture and eval rows rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    for C in G["cases"].values():
        C["state_dict"] = BH.seeded_state_dict(C["state_recipe"], C["weight_seed"])
        C["crops"] = crops(C["kind"], C["dense"])
        C["arch"] = arch(C["kind"], C["dense"])
        D = C["state_dict"]["head.mlp.0.weight"].shape[1]
        C["eval_input"] = torch.randn(C["eval_rows"], D, generator=torch.Generator().manual_seed(C["eval_seed"]))
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    out = dict(cases={name: case(kind, dense) for name, (kind, dense) in CASES.items()}, head=MG.HEAD, out_dim=MG.K,
               hp=MG.HP, nsteps=NSTEPS, vit_spec=MV.SPEC, swin_spec=MG.SMALL,
               generator="oracle/make_golden_bnhead.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB; losses",
          {n: [s["loss"] for s in c["steps"]] for n, c in out["cases"].items()})
