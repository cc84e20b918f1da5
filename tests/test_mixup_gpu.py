"""Mixup targets on the GPU: the mixing kernel against fp64, DINOLoss against the reference fixture and the oracle at
the real step shape, identity targets against the plain loss, DDINOLoss ignoring the targets, the packaged step
(eager vs CUDA graph) and the rejected inputs."""
import os

import pytest
import torch

from helpers import TOL_BF16_ACT, assert_close, at_golden, rel

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_mixup.pt")
BF16 = torch.bfloat16
# mixing kernel gate (DESIGN.md §4.12): the fp16 rounding of the stored row (half an ulp, 2^-11 relative; 2^-25 absolute
# in the subnormal range of the 2^12-scaled format) plus 2^-16 relative for the hi + lo weights and fp32 accumulation
MIX_REL, MIX_ABS = 2.0 ** -11 + 2.0 ** -16, 2.0 ** -24


def _targets(kind, B, ncrops, seed):
    from oracle import mixup as M
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(ncrops):
        if kind == "dense":  # per-row lambda and label smoothing: every entry non-zero, not symmetric
            out.append(M.timm_mixup_target(B, torch.rand(B, generator=g), 0.1))
        elif kind == "sparse":  # one lambda, no smoothing: two non-zeros per row
            out.append(M.timm_mixup_target(B, float(torch.rand((), generator=g)), 0.0))
        else:  # arbitrary non-negative, one all-zero column per view (C = 0)
            T = torch.rand(B, B, generator=g) * 3
            T[:, v % B] = 0
            out.append(T)
    return torch.stack(out)


def _mix_ref(q, T):
    """fp64 (q_hat, C) of esvit_mixup_q: q [2B, K] (any scale), T [ncrops, B, B]."""
    ncrops, B, _ = T.shape
    qd, Td = q.double(), T.double()
    rows, mass = [], []
    for v in range(ncrops):
        W = torch.cat([Td[v] * (iq != v) for iq in range(2)], 0)  # [(iq, j), b]
        C = W.sum(0)
        rows.append(torch.where(C[:, None] > 0, (W.t() @ qd) / C.clamp_min(1e-300)[:, None], torch.zeros_like(qd[:B])))
        mass.append(C)
    return torch.cat(rows), torch.cat(mass)


@pytest.mark.parametrize("kind", ["dense", "sparse", "zero_column"])
@pytest.mark.parametrize("K", [4096, 65536])
@pytest.mark.parametrize("B", [8, 64])
def test_mixing_kernel_matches_fp64(B, K, kind):
    from esvit_b200 import ops
    ncrops = 10
    g = torch.Generator().manual_seed(B * 7 + K)
    # stored teacher probabilities as esvit_row_softmax_q writes them: 2^12 * softmax, fp16, sharp rows
    q = (torch.softmax(torch.randn(2 * B, K, generator=g) * 4, -1) * 4096).half()
    T = _targets(kind, B, ncrops, seed=B + K)
    w_scale = 1.0 / ((2 * ncrops - 2) * B)
    q_hat, w = ops.mixup_q(q.cuda(), T.cuda(), w_scale)
    torch.cuda.synchronize()
    ref, C = _mix_ref(q, T)
    err = (q_hat.double().cpu() - ref).abs()
    bound = MIX_REL * ref.abs() + MIX_ABS
    print(f"\nmixup_q B={B} K={K} {kind}: max |err| / (2^-11 |ref| + 2^-24) = "
          f"{float((err / (2.0 ** -11 * ref.abs() + MIX_ABS)).max()):.3f}, max rel (|ref| > 1e-3) = "
          f"{float((err / ref.abs())[ref.abs() > 1e-3].max()):.3e}")
    assert bool((err <= bound).all()), float((err - bound).max())
    assert torch.allclose(w.double().cpu(), C * w_scale, rtol=1e-6, atol=0)
    if kind == "zero_column":
        zero = C == 0
        assert bool(zero.any()) and float(q_hat.cpu()[zero].abs().max()) == 0 and float(w.cpu()[zero].abs().max()) == 0


def _golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.mark.parametrize("name", ["small_batch", "batch_eps", "elem", "elem_eps", "arbitrary_zero_column"])
def test_dino_loss_mixup_matches_reference_fixture(name):
    from esvit_b200.losses import DINOLoss
    from oracle import make_golden_mixup as MG
    G = _golden()
    c = G["cases"][name]
    mod = DINOLoss(c["K"], c["ncrops"], *G["meta"]["schedule"]).cuda()
    targets = [t.cuda() for t in c["targets"]]
    for rec in c["steps"]:
        s, t = MG.case_inputs(c["B"], c["K"], c["ncrops"], c["seed"], rec["epoch"])
        sc = s.cuda().to(BF16).requires_grad_(True)
        loss = mod(sc, t.cuda().to(BF16), rec["epoch"], targets)
        loss.backward()
        lv = float(loss.detach())
        assert abs(lv - rec["loss"]) <= TOL_BF16_ACT * abs(rec["loss"]), (lv, rec["loss"])
        assert_close(*at_golden(sc.grad.float().cpu(), rec["grad"]), TOL_BF16_ACT, f"{name} dlogits")
        assert_close(mod.center.cpu(), rec["center"], 1e-5, f"{name} center")


def test_dino_loss_mixup_real_shape_matches_oracle():
    """Swin-T step shape: DINOLoss over 2 + 8 crops, K = 65536, B = 64, timm per-row targets with smoothing on the first
    six views and eye(B) on the rest."""
    from esvit_b200.losses import DINOLoss
    from oracle import losses as L
    from oracle import mixup as M
    B, K, ncrops = 64, 65536, 10
    g = torch.Generator(device="cuda").manual_seed(11)
    s = (torch.randn(ncrops * B, K, device="cuda", generator=g) * 2).to(BF16)
    t = (torch.randn(2 * B, K, device="cuda", generator=g) * 1.5).to(BF16)
    center = torch.randn(1, K, device="cuda", generator=g) * 0.1
    T = _targets("dense", B, ncrops, seed=5).cuda()
    T[6:] = torch.eye(B, device="cuda")
    targets = list(T)
    sr = s.float().requires_grad_(True)
    lr = M.dino_loss_mixup(sr, t.float(), center, ncrops, 0.04, targets, 0.1)
    lr.backward()
    mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).cuda()
    mod.center.copy_(center)
    sc = s.clone().requires_grad_(True)
    loss = mod(sc, t, 0, targets)
    (loss * 3.0).backward()  # upstream scale (GradScaler-style) read on the device
    print(f"\nreal shape: loss {float(loss):.6f} oracle {float(lr):.6f} rel {abs(float(loss) - float(lr)) / abs(float(lr)):.2e}, "
          f"dlogits rel l2 {rel(sc.grad, 3 * sr.grad):.2e}")
    assert abs(float(loss) - float(lr)) < 1e-4 * abs(float(lr)), (float(loss), float(lr))
    assert_close(sc.grad, 3 * sr.grad, 5e-3, "dlogits")
    assert_close(mod.center, L.center_update(center, t.float(), 0.9), 1e-5, "center")


@pytest.mark.parametrize("K", [384, 65536])
def test_identity_targets_equal_plain_dino_loss(K):
    from esvit_b200.losses import DINOLoss
    B, ncrops = 16, 10
    g = torch.Generator(device="cuda").manual_seed(K)
    s = (torch.randn(ncrops * B, K, device="cuda", generator=g) * 2).to(BF16)
    t = (torch.randn(2 * B, K, device="cuda", generator=g) * 1.5).to(BF16)
    out = []
    for targets in (None, [torch.eye(B, device="cuda")] * ncrops):
        mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).cuda()
        sc = s.clone().requires_grad_(True)
        loss = mod(sc, t, 0, targets)
        loss.backward()
        out.append((float(loss), sc.grad.float(), mod.center.clone()))
    (l0, g0, c0), (l1, g1, c1) = out
    print(f"\neye targets K={K}: loss rel {abs(l1 - l0) / abs(l0):.2e}, dlogits rel l2 {rel(g1, g0):.2e}")
    assert abs(l1 - l0) <= 1e-5 * abs(l0), (l0, l1)
    assert_close(g1, g0, 2e-3, "dlogits")
    assert torch.equal(c0, c1)


def test_ddino_loss_ignores_targets_bit_for_bit():
    from esvit_b200.losses import DDINOLoss
    B, ncrops, Tg, Tl, P, K = 2, 5, 49, 9, 128, 4096
    g = torch.Generator().manual_seed(3)
    Rs = B * (2 * Tg + (ncrops - 2) * Tl)
    s_cls, t_cls = torch.randn(ncrops * B, K, generator=g).to(BF16), torch.randn(2 * B, K, generator=g).to(BF16)
    s_reg, t_reg = torch.randn(Rs, K, generator=g).to(BF16), torch.randn(2 * B * Tg, K, generator=g).to(BF16)
    s_fea, t_fea = torch.randn(Rs, P, generator=g), torch.randn(2 * B * Tg, P, generator=g)
    targets = list(_targets("dense", B, ncrops, seed=1).cuda())
    out = []
    for tm in (None, targets):
        mod = DDINOLoss(K, ncrops, 0.04, 0.04, 0, 10).cuda()
        sc, sg = s_cls.cuda().requires_grad_(True), s_reg.cuda().requires_grad_(True)
        loss = mod((sc, sg, s_fea.cuda(), [Tg, Tl]), (t_cls.cuda(), t_reg.cuda(), t_fea.cuda(), [Tg]), 0, tm)
        loss.backward()
        out.append((loss.detach(), sc.grad, sg.grad, mod.center.clone(), mod.center_grid.clone()))
    for a, b in zip(*out):
        assert torch.equal(a, b)


def _bad_inputs(B, ncrops):
    good = [torch.eye(B, device="cuda") for _ in range(ncrops)]
    nan, neg, inf = [t.clone() for t in good], [t.clone() for t in good], [t.clone() for t in good]
    nan[3][1, 2] = float("nan")
    neg[2][0, 1] = -0.25
    inf[0][0, 0] = float("inf")
    return {
        "tensor_not_list": torch.stack(good),
        "too_few_views": good[:-1],
        "wrong_shape": good[:-1] + [torch.eye(B + 1, device="cuda")],
        "not_a_tensor": good[:-1] + [[[1.0] * B] * B],
        "integer": good[:-1] + [torch.eye(B, device="cuda").long()],
        "cpu": good[:-1] + [torch.eye(B)],
        "nan": nan, "inf": inf, "negative": neg,
    }


@pytest.mark.parametrize("case", ["tensor_not_list", "too_few_views", "wrong_shape", "not_a_tensor", "integer", "cpu",
                                  "nan", "inf", "negative"])
def test_malformed_targets_raise_value_error(case):
    from esvit_b200.losses import DINOLoss
    B, ncrops, K = 4, 4, 256
    mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).cuda()
    s = torch.randn(ncrops * B, K, device="cuda").to(BF16).requires_grad_(True)
    t = torch.randn(2 * B, K, device="cuda").to(BF16)
    with pytest.raises(ValueError):
        mod(s, t, 0, _bad_inputs(B, ncrops)[case])


def test_stored_probability_path_off_rejects_mixup_only(monkeypatch):
    from esvit_b200.losses import DINOLoss
    monkeypatch.setenv("ESVIT_CE_Q", "0")
    B, ncrops, K = 4, 4, 256
    mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).cuda()
    s = torch.randn(ncrops * B, K, device="cuda").to(BF16).requires_grad_(True)
    t = torch.randn(2 * B, K, device="cuda").to(BF16)
    assert torch.isfinite(mod(s, t, 0, None))
    assert torch.isfinite(mod(s, t, 0, []))  # falsy targets: the plain loss, as in the reference
    with pytest.raises(NotImplementedError):
        mod(s, t, 0, [torch.eye(B, device="cuda")] * ncrops)


def _mixup_step(graph: bool):
    from esvit_b200 import engine
    from helpers import load_golden
    G = load_golden()
    meta = G["dense"]["meta"]
    sp, hp = meta["spec"], meta["hp"]
    spec = dict(embed_dim=sp["embed_dim"], depths=list(sp["depths"]), num_heads=list(sp["num_heads"]),
                window_size=sp["window_size"], drop_path_rate=0.0)
    crops = [c.cuda() for c in G["dense"]["crops"]]
    step, student, teacher, loss = engine.make_step(
        out_dim=meta["out_dim"], ncrops=len(crops), dense=False, device="cuda:0", lr=hp["lr"],
        weight_decay=hp["weight_decay"], clip_grad=hp["clip_grad"], freeze_last_layer=hp["freeze_last_layer"],
        img_size=sp["img_size"], head_kwargs=meta["head"], spec=spec, teacher_temp=hp["teacher_temp"],
        cuda_graph=graph)
    sd = {k: v for k, v in G["dense"]["state_dict"].items() if not k.startswith("head_dense")}
    student.load_state_dict(sd)
    teacher.load_state_dict(sd)
    return step, student, loss, crops, hp


def test_packaged_mixup_step_graph_equals_eager_and_plain_step_unchanged():
    """Plain, mixup, then plain steps again: the graph side captures one graph of each kind and agrees with the eager
    side under the graph-vs-eager gate of test_model_gpu.py; a plain step also equals the plain step of a model that
    never ran a mixup step when both start from the same weights and center."""
    from oracle import mixup as M
    stepE, sE, lE, crops, hp = _mixup_step(False)
    stepG, sG, lG, _, _ = _mixup_step(True)
    B = crops[0].shape[0]
    lam = [0.7, 0.35, 0.9]
    mixed = [lam[v] * c + (1 - lam[v]) * c.flip(0) if v < 3 else c for v, c in enumerate(crops)]
    targets = [M.timm_mixup_target(B, lam[v], 0.1).cuda() if v < 3 else torch.eye(B, device="cuda")
               for v in range(len(crops))]
    le, lg = [], []
    # each graph needs 3 eager warm-up steps before its capture; they run at lr = 0 (the weights stay put) so that, as in
    # test_model_gpu.py, at most six optimiser steps amplify the atomic-order noise of the small-parameter gradients
    plan = ["plain"] * 4 + ["mixup"] * 5 + ["plain"]
    warm = {0, 1, 2, 4, 5, 6}
    for it, kind in enumerate(plan):
        lr = 0.0 if it in warm else hp["lr"] * (1 + 0.1 * it)
        kw = dict(student_images=mixed, targets_mixup=targets) if kind == "mixup" else {}
        le.append(float(stepE.step(crops, 1, lr, hp["weight_decay"], 0.996, **kw)))
        lg.append(float(stepG.step(crops, 1, lr, hp["weight_decay"], 0.996, **kw)))
    assert len(stepG._graphs) == 2
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)
    for (n, a), b in zip(sE.named_parameters(), sG.parameters()):
        assert_close(b, a, 2e-3, n)
    assert_close(lG.center, lE.center, 1e-3, "center")
    # the mixup step computes a different loss from the plain step at the same weights
    assert abs(le[4] - le[2]) > 1e-3 * abs(le[2])  # (steps 2 and 4 see the same weights: lr = 0 in between)

    # a plain step after a mixup step, against the same plain step of a model that only ran plain steps from there
    stepF, sF, lF, _, _ = _mixup_step(False)
    sF.load_state_dict(sE.state_dict())
    stepF.teacher.load_state_dict(stepE.teacher.state_dict())
    lF.center.copy_(lE.center)
    a = float(stepE.step(crops, 1, hp["lr"], hp["weight_decay"], 0.996))
    b = float(stepF.step(crops, 1, hp["lr"], hp["weight_decay"], 0.996))
    assert abs(a - b) <= 1e-6 * abs(b), (a, b)
