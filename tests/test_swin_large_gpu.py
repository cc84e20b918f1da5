"""GPU: Swin-L (`swin_large_w7`: embed 192, heads 6/12/24/48) and Swin-T W14 (`swin_tiny_w14`).

Swin-L's widths take three kernels past the limits every other Swin spec stays within: the patch embedding at E = 192,
the stage 2 -> 3 PatchMerging LayerNorm over 4C = 3072 and the DDINO region matching at P = 1536 (where the teacher
view's 49 x 1536 rows stream through shared memory in several chunks).  Each is checked on its own against torch, then
the model against the executed reference at Swin-L widths (tests/golden/esvit_large.pt) and against the CPU oracle at
the true specs.  The true-spec Swin-L test runs the fp32 oracle at full depth on the CPU; its name contains `slow` so
`-k "not slow"` leaves it out."""
import os
from functools import partial

import pytest
import torch
import torch.nn as nn

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, assert_close, at_golden, load_golden, rel
from oracle import eval as E
from oracle import golden as GD
from oracle import make_golden_large as MGL
from oracle import swin as S

pytestmark = pytest.mark.gpu

GOLDEN_LARGE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_large.pt")


# ---- kernels -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S_", [224, 100, 36])
def test_patch_embed_e192(S_):
    """E = 192 forward and backward over two resolution groups (S and S - 8): token counts 2 * (S/4)^2 + ((S-8)/4)^2
    that are not multiples of the 64-token tile"""
    from test_ops_gpu import test_patch_embed_groups
    test_patch_embed_groups(192, S_)


@pytest.mark.parametrize("H", [7, 3, 14])
def test_patch_merge_ln_4c_3072(H):
    """C = 768, 4C = 3072: an odd map (zero-padded to even) and an even one in one call, forward and backward"""
    from test_ops_gpu import test_patch_merge_ln_groups
    test_patch_merge_ln_groups(H, 768)


_BUDGET = 220 * 1024  # esvit_region_match's shared-memory budget


def _chunk_rows(Tg, Tl, ncrops, P):
    """teacher rows per shared-memory chunk that esvit_region_match picks"""
    row, state = P * 4, (2 * Tg + (ncrops - 2) * Tl) * 8
    return Tg if Tg * row <= _BUDGET else (_BUDGET - state) // row


def _ncrops_for_chunk(Tg, Tl, P, tc):
    """the smallest crop count whose arg-max state leaves room for tc teacher rows per chunk"""
    n = 2
    while _chunk_rows(Tg, Tl, n, P) > tc:
        n += 1
    assert _chunk_rows(Tg, Tl, n, P) == tc
    return n


def _features(B, Tg, Tl, ncrops, P, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sn = torch.randn(B * (2 * Tg + (ncrops - 2) * Tl), P, device="cuda", generator=g)
    tn = torch.randn(2 * B * Tg, P, device="cuda", generator=g)
    return sn, tn


def _plant_ties(sn, tn, B, Tg):
    """teacher rows 5 and 40 of image 1 / view 0 are equal, and student row 3 of view 1 / image 1 is that row scaled:
    the first index (5) is the maximum, tied with 40, and the two sit in different chunks"""
    b, iq, v = 1, 0, 1
    t0 = (iq * B + b) * Tg
    tn[t0 + 40] = tn[t0 + 5]
    sn[(v * B + b) * Tg + 3] = 1.7 * tn[t0 + 5]
    return (iq, v, b, 3, 5)


def test_region_match_p1536_matches_torch_max():
    """P = 1536 (Swin-L num_features), Swin-L token counts (49 / 9), several chunks: indices bit-exact with torch.max
    over the fp32 cosine similarities of the same normalised features, first index on a planted tie"""
    from esvit_b200 import ops
    from test_vit_gpu import _region_ref
    B, ncrops, Tg, Tl, P = 2, 10, 49, 9, 1536
    assert 1 < _chunk_rows(Tg, Tl, ncrops, P) < Tg
    sn, tn = _features(B, Tg, Tl, ncrops, P, 17)
    iq, v, b, i, j = _plant_ties(sn, tn, B, Tg)
    idx, trow = ops.region_match(sn, tn, B, ncrops, Tg, Tl)
    assert int(idx[iq, v, b, i]) == j
    ref = _region_ref(sn.cpu(), tn.cpu(), B, ncrops, Tg, Tl).cuda()
    assert torch.equal(idx, ref)
    idx2, trow2 = ops.region_match(sn, tn, B, ncrops, Tg, Tl)
    assert torch.equal(idx, idx2) and torch.equal(trow, trow2)


@pytest.mark.parametrize("tc", [1, 2, 7])
def test_region_match_p1536_indices_do_not_depend_on_chunk_rows(tc):
    """The chunk size follows from the shared memory left beside the per-token arg-max state, so more local crops
    force smaller chunks.  The first ten crops of a many-crop call (tc teacher rows per chunk) get the indices and
    teacher rows of a ten-crop call (36 rows per chunk), ties included."""
    from esvit_b200 import ops
    B, Tg, Tl, P = 2, 49, 9, 1536
    n = _ncrops_for_chunk(Tg, Tl, P, tc)
    sn, tn = _features(B, Tg, Tl, n, P, 23 + tc)
    _plant_ties(sn, tn, B, Tg)
    idx, trow = ops.region_match(sn, tn, B, n, Tg, Tl)
    rows10 = B * (2 * Tg + 8 * Tl)
    idx10, trow10 = ops.region_match(sn[:rows10], tn, B, 10, Tg, Tl)
    assert _chunk_rows(Tg, Tl, 10, P) == 36
    assert torch.equal(idx[:, :10], idx10)
    assert torch.equal(trow[:rows10], trow10)
    assert int(idx[0, 1, 1, 3]) == 5


def tol_for(name):
    """the gradient gate of test_real_shapes_gpu.py's Swin-T test: 0.12 for the tensors whose gradient crosses the whole
    bf16 backward at its most sensitive point (the reference itself under bf16 autocast deviates from its fp32 run by
    0.11 - 0.18 on them), TOL_BF16_GRAD for every other parameter"""
    if "relative_position_bias_table" in name or name == "patch_embed.proj.weight" or \
            (name.startswith("layers.0.") and name.endswith("norm1.bias")):
        return 0.12
    return TOL_BF16_GRAD


# ---- the model against the executed reference at Swin-L widths ---------------------------------------------------
@pytest.fixture(scope="module")
def G():
    return load_golden(GOLDEN_LARGE)


def test_golden_large_forward_loss_gradients(G):
    """reduced-depth Swin-L (2, 2, 2, 2) with DDINO heads, 224^2 + 96^2 crops: forward outputs, loss and gradients
    against the reference's fp32 CPU run"""
    from esvit_b200 import engine
    D = G["dense"]
    M = D["meta"]
    sp, hp = dict(M["spec"]), M["hp"]
    spec = dict(embed_dim=sp["embed_dim"], depths=list(sp["depths"]), num_heads=list(sp["num_heads"]),
                window_size=sp["window_size"], drop_path_rate=0.0)
    step, student, teacher, loss = engine.make_step(
        out_dim=M["out_dim"], ncrops=M["ncrops"], dense=True, device="cuda:0", lr=hp["lr"],
        weight_decay=hp["weight_decay"], clip_grad=hp["clip_grad"], freeze_last_layer=hp["freeze_last_layer"],
        img_size=sp["img_size"], head_kwargs=M["head"], spec=spec, teacher_temp=hp["teacher_temp"])
    student.load_state_dict(D["state_dict"])
    teacher.load_state_dict(D["state_dict"])
    crops = [c.cuda() for c in D["crops"]]
    with torch.no_grad():
        t = teacher(crops[:2])
    s = student(crops)
    assert list(s[3]) == D["s_npatch"] == [49, 9] and list(t[3]) == D["t_npatch"]
    for a, k in zip(list(s[:3]) + list(t[:3]), ("s_cls", "s_region", "s_fea", "t_cls", "t_region", "t_fea")):
        assert_close(*at_golden(a, D[k]), TOL_BF16_ACT, k)
    l = loss(s, t, 0, None)
    l.backward()
    assert abs(float(l) - D["losses"][0]) < 5e-3 * abs(D["losses"][0]), (float(l), D["losses"][0])
    named = dict(student.named_parameters())
    bad = {}
    for k, g_ref in D["grads_step0_full"].items():
        r = rel(*at_golden(named[k].grad, g_ref))
        if r >= tol_for(k):
            bad[k] = r
    assert not bad, bad
    for k, (_, nrm) in D["grads_step0_stats"].items():
        g = named[k].grad
        assert g is not None, k
        if nrm > 1e-8:
            assert abs(float(g.double().norm()) - nrm) < 0.1 * nrm + 1e-7, (k, float(g.norm()), nrm)


# ---- true specs against the CPU oracle ---------------------------------------------------------------------------
def _perturb(student, seed=11):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in student.named_parameters():
            if n.endswith(".bias") or (p.dim() == 1 and "norm" in n) or "relative_position_bias_table" in n:
                p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.1)


def _true_spec_case(arch, ospec_d, K, ncrops, B, check_grads):
    """make_step(arch) against oracle.swin / oracle.losses on the same weights and crops: forward outputs, DDINO loss,
    region indices (bit-exact on the CUDA path's own features) and, with check_grads, every parameter gradient"""
    from esvit_b200 import engine
    from oracle import losses as L
    from oracle import step as ST
    step, student, teacher, loss = engine.make_step(arch=arch, out_dim=K, ncrops=ncrops, dense=True, device="cuda:0",
                                                    drop_path=0.0, seed=0)
    _perturb(student)
    teacher.load_state_dict(student.state_dict())
    crops = ST.synthetic_crops(B, ncrops - 2, seed=1234)
    sd = {k: v.detach().cpu().clone().requires_grad_(check_grads and v.dtype.is_floating_point
                                                     and not k.endswith("weight_g"))
          for k, v in student.state_dict().items()}
    ospec = S.SwinSpec(img_size=224, use_dense_prediction=True, **ospec_d)
    with torch.no_grad():
        t_ref = S.multicrop_forward(crops[:2], {k: v.detach() for k, v in sd.items()}, ospec)
    with torch.set_grad_enabled(check_grads):
        s_ref = S.multicrop_forward(crops, sd, ospec)
        l_ref = L.ddino_loss(s_ref, t_ref, torch.zeros(1, K), torch.zeros(1, K), ncrops, 0.04)
    if check_grads:
        l_ref.backward()

    cc = [c.cuda() for c in crops]
    with torch.no_grad():
        t = teacher(cc[:2])
    s = student(cc)
    l = loss(s, t, 0, None)
    if check_grads:
        l.backward()
    torch.cuda.synchronize()
    assert list(s[3]) == list(s_ref[3]) == [49, 9]
    for a, b, name in zip(list(s[:3]) + list(t[:3]), list(s_ref[:3]) + list(t_ref[:3]),
                          ("student cls", "student region", "student features", "teacher cls", "teacher region",
                           "teacher features")):
        assert_close(a, b, TOL_BF16_ACT, name)
    assert abs(float(l) - float(l_ref)) < 5e-3 * abs(float(l_ref)), (float(l), float(l_ref))
    s_fea, t_fea = s[2].detach().float().cpu(), t[2].detach().float().cpu()
    s_feas, t_feas = torch.split(s_fea, [49 * B] * 2 + [9 * B] * (ncrops - 2)), t_fea.chunk(2)
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            T = 49 if v < 2 else 9
            want = L.region_match(s_feas[v].view(B, T, -1), t_feas[iq].view(B, 49, -1))
            assert torch.equal(loss.last_indices[iq, v, :, :T].cpu(), want), (iq, v)
    if not check_grads:
        return

    bad = {}
    for n, p in student.named_parameters():
        if sd[n].grad is None:
            assert p.grad is None or n.endswith("weight_g"), n
            continue
        assert p.grad is not None, n
        if float(sd[n].grad.norm()) <= 1e-7:
            continue
        r = rel(p.grad, sd[n].grad)
        if r >= tol_for(n):
            bad[n] = r
    assert not bad, bad


def test_slow_swin_large_true_spec_k65536_matches_oracle():
    """swin_large_w7 at K = 65 536, 2 + 8 crops, B = 2: outputs, loss, indices and every parameter gradient"""
    _true_spec_case("swin_large_w7", MGL.SWIN_L_W7, 65536, 10, 2, check_grads=True)


def test_swin_tiny_w14_true_spec_k65536_matches_oracle():
    """swin_tiny_w14 (2x2 shifted windows of 14 in stage 0, one un-shifted 14x14 window in stage 1, ws clamped to 7 in
    stages 2-3) at K = 65 536, 2 + 8 crops, B = 2: outputs, loss, indices and every parameter gradient"""
    _true_spec_case("swin_tiny_w14", MGL.SWIN_T_W14, 65536, 10, 2, check_grads=True)


def test_swin_large_cuda_graph_step_equals_eager_step():
    """The gate of test_model_gpu.py's graph test: 2e-3 on losses and parameters after six optimiser steps, with
    non-trivial weights (biases, LN affine and bias tables perturbed) as there.

    One slice is held to a different bound: the key third of every qkv bias.  Adding a constant to a row's keys leaves
    its softmax unchanged, so the gradient of b_k is exactly zero and what any run computes for it is rounding noise
    (fp32 atomics make it differ from run to run, eager or replayed).  AdamW turns that noise into steps of about lr,
    so b_k may move by up to lr per step in either run, and the two may differ by up to twice the summed learning rates.
    At Swin-L's stage 3 that slice alone puts the whole qkv bias ~3e-3 apart between two eager runs."""
    from esvit_b200 import engine
    from oracle import step as ST
    K, ncrops, B = 4096, 4, 2
    crops = [c.cuda() for c in ST.synthetic_crops(B, ncrops - 2, seed=77)]
    runs = []
    for graph in (False, True):
        step, student, teacher, loss = engine.make_step(arch="swin_large_w7", out_dim=K, ncrops=ncrops, dense=True,
                                                        device="cuda:0", drop_path=0.0, seed=2)
        step.use_cuda_graph = graph
        _perturb(student)
        teacher.load_state_dict(student.state_dict())
        runs.append((step, student, loss))
    le, lg, lrs = [], [], []
    for it in range(6):  # 3 eager warm-up calls + capture + 2 replays on the graph side
        lrs.append(5e-4 * (1 + 0.1 * it))
        le.append(float(runs[0][0](crops, 1, lrs[-1], 0.04, 0.996)))
        lg.append(float(runs[1][0](crops, 1, lrs[-1], 0.04, 0.996)))
    assert len(runs[1][0]._graphs) == 1
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)
    for (n, a), g in zip(runs[0][1].named_parameters(), runs[1][1].parameters()):
        if n.endswith("attn.qkv.bias"):
            C = a.shape[0] // 3
            assert float((g[C:2 * C] - a[C:2 * C]).abs().max()) <= 2 * sum(lrs), n + " (k)"
            a, g = torch.cat([a[:C], a[2 * C:]]), torch.cat([g[:C], g[2 * C:]])
        assert_close(g, a, 2e-3, n)
    assert_close(runs[1][2].center, runs[0][2].center, 1e-3, "center")


# ---- evaluation entry points at Swin-L width ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def large_model():
    from esvit_b200.swin_transformer import SwinTransformer
    spec = dict(MGL.SWIN_L_W7)
    m = SwinTransformer(img_size=224, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                        **spec)
    sd = GD.seeded_state_dict(GD.recipe(m.state_dict()), 5)
    m.load_state_dict(sd)
    return m.cuda().eval(), sd, S.SwinSpec(img_size=224, **spec)


def test_large_n_last_blocks_matches_oracle(large_model):
    m, sd, ospec = large_model
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        out = m.forward_return_n_last_blocks(x.cuda(), 4, False, list(ospec.depths))
        out_pool = m.forward_return_n_last_blocks(x.cuda(), 4, True, list(ospec.depths))
        ref = E.n_last_blocks(x, sd, ospec, 4)
    widths = [768, 768, 1536, 1536]
    assert out.shape == (2, sum(widths)) and torch.equal(out, out_pool)
    c0 = 0
    for i, c in enumerate(widths):
        assert_close(out[:, c0:c0 + c], ref[:, c0:c0 + c], TOL_BF16_ACT, f"slice {i}")
        c0 += c


def test_large_selfattention_matches_oracle(large_model):
    """every block's probabilities (nH = 6, 12, 24, 48) and the last block's alone"""
    from oracle import attn as A
    m, sd, ospec = large_model
    x = E.probe_images(1, 224, 9)
    maps = m.forward_selfattention(x.cuda(), 2)
    with torch.no_grad():
        refs = A.selfattention(x, sd, ospec, 2)
    assert len(maps) == len(refs) == 24
    assert [t.shape[1] for t in maps] == [6] * 2 + [12] * 2 + [24] * 18 + [48] * 2
    for i, (a, r) in enumerate(zip(maps, refs)):
        assert a.shape == r.shape, (i, tuple(a.shape), tuple(r.shape))
        assert_close(a, r, TOL_BF16_ACT, f"block {i}")
    assert torch.equal(m.forward_selfattention(x.cuda(), 1), maps[-1])


def test_large_feature_maps_match_oracle(large_model):
    m, sd, ospec = large_model
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        pooled, region = m.forward_feature_maps(x.cuda())
        p_ref, r_ref = S.forward_features(x, sd, ospec)
    assert tuple(region.shape) == (2, 49, 1536) and tuple(pooled.shape) == (2, 1536)
    assert_close(pooled, p_ref, TOL_BF16_ACT, "pooled")
    assert_close(region, r_ref, TOL_BF16_ACT, "region")
