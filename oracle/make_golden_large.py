"""Generate tests/golden/esvit_large.pt by RUNNING THE UNMODIFIED REFERENCE at Swin-L widths.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout):

    python -m oracle.make_golden_large      # writes tests/golden/esvit_large.pt

The model is Swin-L (experiments/imagenet/swin/swin_large_patch4_window7_224.yaml: embed 192, heads 6/12/24/48, W7) at
reduced depth (2, 2, 2, 2), on 224^2 global and 96^2 local crops.  So every width of the real spec is exercised: the
patch embedding at E = 192, the stage 2 -> 3 PatchMerging LayerNorm over 4C = 3072, window attention at nH = 48, and
the DDINO region matching at P = num_features = 1536.  One training step of make_golden.py's loop runs through the
reference's own modules on CPU fp32, and the oracle is asserted against every stored value while the file is written.
Weights and crops are rebuilt from their seeds on load (oracle/golden.py); large tensors are stored as a seeded sample.
"""
from __future__ import annotations

import os
import sys

import torch

from . import golden as GD
from . import reference_import as R
from . import step as ST
from . import swin as S
from .make_golden import HEAD, HP, K, OUT, WEIGHT_SEED, build, reference_steps, stats

# MODEL.SPEC of experiments/imagenet/swin/swin_large_patch4_window7_224.yaml and swin_tiny_patch4_window14_224.yaml, in
# the form of oracle.swin's SWIN_T_W7 / SWIN_S_W14 / SWIN_B_W14
SWIN_L_W7 = dict(embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48), window_size=7)
SWIN_T_W14 = dict(embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24), window_size=14)
LARGE = dict(SWIN_L_W7, img_size=224, depths=(2, 2, 2, 2))
B, N_LOCAL, CROP_SEED, GLOBAL, LOCAL = 2, 2, 4321, 224, 96
FULL_GRADS = ("patch_embed.proj.weight", "patch_embed.proj.bias", "patch_embed.norm.weight", "patch_embed.norm.bias",
              "layers.0.blocks.1.attn.relative_position_bias_table", "layers.0.blocks.1.attn.qkv.weight",
              "layers.1.blocks.0.mlp.fc1.weight", "layers.2.downsample.reduction.weight",
              "layers.2.downsample.norm.weight", "layers.2.downsample.norm.bias",
              "layers.3.blocks.0.attn.relative_position_bias_table", "layers.3.blocks.1.attn.qkv.weight",
              "layers.3.blocks.1.mlp.fc2.weight", "norm.weight", "norm.bias", "head.mlp.0.weight",
              "head_dense.mlp.0.weight", "head_dense.last_layer.weight_v")


def make() -> dict:
    R.ensure_process_group()
    ns, spec, student = build(True, small=LARGE)
    _, _, teacher = build(True, small=LARGE)
    teacher.load_state_dict(student.state_dict())
    for p in teacher.parameters():
        p.requires_grad = False
    sd0 = {k: v.detach().clone() for k, v in student.state_dict().items()}
    ncrops = 2 + N_LOCAL
    crops = ST.synthetic_crops(B, N_LOCAL, seed=CROP_SEED, global_size=GLOBAL, local_size=LOCAL)
    loss_mod = ns.DDINOLoss(K, ncrops, 0.04, HP["teacher_temp"], 0, 10, HP["student_temp"], HP["center_momentum"])
    r0 = reference_steps(ns, student, teacher, loss_mod, crops, 1, True)[0]
    so, to = r0["student_output"], r0["teacher_output"]

    # ---- the oracle must reproduce all of it -------------------------------------------------
    orc = ST.OracleStep(sd0, spec, ncrops, K, **HP)
    lo = orc.step(crops, epoch=0, keep_grads=True)
    assert abs(lo - r0["loss"]) < 2e-5 * max(1, abs(r0["loss"])), (lo, r0["loss"])
    for k, g in r0["grads"].items():
        assert torch.allclose(orc.grads_step[k], g, atol=1e-7 + 1e-4 * float(g.abs().max()), rtol=1e-3), k
    assert torch.allclose(orc.center, loss_mod.center, atol=1e-6)
    assert torch.allclose(orc.center_grid, loss_mod.center_grid, atol=1e-6)

    # arg-max indices with the reference's own expression (main_esvit.py:735-736)
    N = to[3][0]
    split = [so[3][0]] * 2 + [so[3][1]] * (ncrops - 2)
    s_f = torch.split(so[2].detach(), [i * B for i in split], dim=0)
    t_f = to[2].detach().chunk(2)
    idx = {}
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            a = torch.nn.functional.normalize(s_f[v].view(B, split[v], -1), p=2, dim=-1)
            b = torch.nn.functional.normalize(t_f[iq].view(B, N, -1), p=2, dim=-1)
            idx[(iq, v)] = torch.matmul(a, b.permute(0, 2, 1)).max(dim=2)[1]
            assert torch.equal(idx[(iq, v)], orc.indices_step[(iq, v)])

    return dict(
        meta=dict(spec=dict(LARGE, use_dense_prediction=True), head=HEAD, out_dim=K, batch=B, n_local=N_LOCAL,
                  ncrops=ncrops, hp=HP, nsteps=1, crop_seed=CROP_SEED, global_size=GLOBAL, local_size=LOCAL,
                  weight_seed=WEIGHT_SEED,
                  generator="oracle/make_golden_large.py (reference run on CPU fp32, torch %s)" % torch.__version__),
        state_recipe=GD.recipe(sd0), initial_stats=stats({k: v for k, v in sd0.items() if v.dtype.is_floating_point}),
        losses=[r0["loss"]], center_after=loss_mod.center.clone(), center_grid_after=loss_mod.center_grid.clone(),
        s_cls=GD.sample(so[0]), s_region=GD.sample(so[1]), s_fea=GD.sample(so[2]), s_npatch=list(so[3]),
        t_cls=GD.sample(to[0]), t_region=GD.sample(to[1]), t_fea=GD.sample(to[2]), t_npatch=list(to[3]),
        indices=idx, grads_step0_stats=stats(r0["grads"]),
        grads_step0_full={k: GD.sample(r0["grads"][k]) for k in FULL_GRADS},
    )


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    D = make()
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "esvit_large.pt")
    torch.save(dict(dense=D), path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB; loss", D["losses"][0])
