"""GPU parity at the TRUE dimensions of BASELINE.json configs[1] (Swin-T W7, 2 global + 8 local crops, out_dim 65536)
and at the head counts / widths of every BASELINE config - the miniature fixtures of test_model_gpu.py / test_ops_gpu.py
never exercise K = 65536, nH in {3, 6, 24, 32}, C in {96, 128, 192, 768, 1024} or the real depth.

The checker is the CPU oracle (oracle/, pinned against the executed reference by tests/test_oracle_golden.py) run in the
same process on the same seeded crops and the same random-init weights."""
import pytest
import torch

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, assert_close, rel

pytestmark = pytest.mark.gpu


def _perturb(student, seed=11):
    """non-trivial biases / LN affine / rel-pos tables (the reference initialises them to 0 / 1 / ~0.02)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in student.named_parameters():
            if n.endswith(".bias") or (p.dim() == 1 and "norm" in n) or "relative_position_bias_table" in n:
                p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.1)


def test_swin_tiny_k65536_forward_loss_indices_gradients_match_oracle():
    """configs[1] at B = 2: forward outputs, DDINO loss, region arg-max indices (bit-exact on shared features) and every
    parameter gradient of the CUDA path against oracle.swin / oracle.losses."""
    from esvit_b200 import engine
    from oracle import losses as L
    from oracle import step as ST
    from oracle import swin as S
    K, ncrops, B = 65536, 10, 2
    step, student, teacher, loss = engine.make_step(arch="swin_tiny_w7", out_dim=K, ncrops=ncrops, dense=True,
                                                    device="cuda:0", drop_path=0.0, seed=0)
    _perturb(student)
    teacher.load_state_dict(student.state_dict())
    crops = ST.synthetic_crops(B, ncrops - 2, seed=1234)
    sd = {k: v.detach().cpu().clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g"))
          for k, v in student.state_dict().items()}
    ospec = S.SwinSpec(img_size=224, use_dense_prediction=True, **S.SWIN_T_W7)
    with torch.no_grad():
        t_ref = S.multicrop_forward(crops[:2], {k: v.detach() for k, v in sd.items()}, ospec)
    s_ref = S.multicrop_forward(crops, sd, ospec)
    l_ref, idx_ref = L.ddino_loss(s_ref, t_ref, torch.zeros(1, K), torch.zeros(1, K), ncrops, 0.04, return_indices=True)
    l_ref.backward()

    cc = [c.cuda() for c in crops]
    with torch.no_grad():
        t = teacher(cc[:2])
    s = student(cc)
    l = loss(s, t, 0, None)
    l.backward()
    torch.cuda.synchronize()
    assert list(s[3]) == list(s_ref[3]) == [49, 9]
    assert s[0].shape == (ncrops * B, K) and s[1].shape == (B * (2 * 49 + 8 * 9), K) and t[1].shape == (B * 2 * 49, K)
    for a, b, name in zip(s[:3], s_ref[:3], ("student cls logits", "student region logits", "student features")):
        assert_close(a, b, TOL_BF16_ACT, name)
    for a, b, name in zip(t[:3], t_ref[:3], ("teacher cls logits", "teacher region logits", "teacher features")):
        assert_close(a, b, TOL_BF16_ACT, name)
    assert abs(float(l) - float(l_ref)) < 5e-3 * abs(float(l_ref)), (float(l), float(l_ref))

    # arg-max indices: bit-exact when the oracle's matcher is fed OUR features (the op boundary of BASELINE.md section 3)
    s_fea, t_fea = s[2].detach().float().cpu(), t[2].detach().float().cpu()
    split = [49 * B] * 2 + [9 * B] * (ncrops - 2)
    s_feas, t_feas = torch.split(s_fea, split), t_fea.chunk(2)
    same_as_oracle_run = 0
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            T = 49 if v < 2 else 9
            want = L.region_match(s_feas[v].view(B, T, -1), t_feas[iq].view(B, 49, -1))
            got = loss.last_indices[iq, v, :, :T].cpu()
            assert torch.equal(got, want), (iq, v)
            same_as_oracle_run += int((got == idx_ref[(iq, v)]).sum())
    total = sum(B * (49 if v < 2 else 9) for iq in range(2) for v in range(ncrops) if v != iq)
    # against the oracle's OWN fp32 features the pairing may flip only where two cosines are closer than the bf16 noise
    assert same_as_oracle_run >= 0.9 * total, (same_as_oracle_run, total)

    # Gradient gate.  TOL_BF16_GRAD (6e-2 rel-L2) for every parameter, except the three parameter classes whose gradient
    # passes through the WHOLE 12-block bf16 backward and a softmax / LayerNorm at its most sensitive point: for those the
    # reference ALGORITHM itself, run under bf16 autocast, deviates from its own fp32 run by 0.11 - 0.35 rel-L2 on these
    # very inputs (stage-0 norm1.bias 0.35, rel-pos bias tables 0.11 - 0.18, patch_embed.proj.weight 0.18; median over all 187
    # tensors 0.03) - the gate for them is 0.12, i.e. tighter than the reference's own mixed-precision noise.
    def tol_for(name: str) -> float:
        if "relative_position_bias_table" in name or name == "patch_embed.proj.weight" or \
                (name.startswith("layers.0.") and name.endswith("norm1.bias")):
            return 0.12
        return TOL_BF16_GRAD

    bad, worst = {}, 0.0
    for n, p in student.named_parameters():
        if sd[n].grad is None:
            assert p.grad is None or n.endswith("weight_g"), n
            continue
        assert p.grad is not None, n
        if float(sd[n].grad.norm()) <= 1e-7:
            continue
        r = rel(p.grad, sd[n].grad)
        worst = max(worst, r)
        if r >= tol_for(n):
            bad[n] = r
    assert not bad, bad


@pytest.mark.parametrize("K", [65536])
def test_dino_and_ddino_loss_k65536(K):
    """the CE / LSE / column-sum kernels at the real out_dim against oracle.losses (test_ops_gpu stops at 4096)"""
    from esvit_b200.losses import DDINOLoss, DINOLoss
    from oracle import losses as L
    from test_ops_gpu import _loss_inputs
    d = torch.device("cuda:0")
    B, ncrops, Tg, Tl, P = 2, 10, 49, 9, 768
    s_cls, t_cls, s_reg, t_reg, s_fea, t_fea, center, center_grid = _loss_inputs(B, ncrops, K, Tg, Tl, P, seed=5)
    # view-level
    sr = s_cls.float().requires_grad_(True)
    l_r = L.dino_loss(sr, t_cls.float(), center, ncrops, 0.04, 0.1)
    l_r.backward()
    mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).to(d)
    mod.center.copy_(center)
    sc = s_cls.to(d).requires_grad_(True)
    l = mod(sc, t_cls.to(d), 0, None)
    l.backward()
    assert abs(float(l) - float(l_r)) < 1e-4 * abs(float(l_r)), (float(l), float(l_r))
    assert_close(sc.grad, sr.grad, 5e-3, "dlogits (view)")
    assert_close(mod.center, L.center_update(center, t_cls.float(), 0.9), 1e-5, "center")
    # view + region
    scr, srr = s_cls.float().requires_grad_(True), s_reg.float().requires_grad_(True)
    l_r, idx_r = L.ddino_loss((scr, srr, s_fea, [Tg, Tl]), (t_cls.float(), t_reg.float(), t_fea, [Tg]), center,
                              center_grid, ncrops, 0.04, 0.1, return_indices=True)
    l_r.backward()
    mod = DDINOLoss(K, ncrops, 0.04, 0.04, 0, 10).to(d)
    mod.center.copy_(center)
    mod.center_grid.copy_(center_grid)
    sc, sg = s_cls.to(d).requires_grad_(True), s_reg.to(d).requires_grad_(True)
    l = mod((sc, sg, s_fea.to(d), [Tg, Tl]), (t_cls.to(d), t_reg.to(d), t_fea.to(d), [Tg]), 0, None)
    l.backward()
    assert abs(float(l) - float(l_r)) < 1e-4 * abs(float(l_r)), (float(l), float(l_r))
    for (iq, v), ref in idx_r.items():
        T = Tg if v < 2 else Tl
        assert torch.equal(mod.last_indices[iq, v, :, :T].cpu(), ref)
    assert_close(sc.grad, scr.grad, 5e-3, "dcls")
    assert_close(sg.grad, srr.grad, 5e-3, "dregion")
    assert_close(mod.center, L.center_update(center, t_cls.float(), 0.9), 1e-5, "center")
    assert_close(mod.center_grid, L.center_update(center_grid, t_reg.float(), 0.9), 1e-5, "center_grid")


@pytest.mark.parametrize("C,nH,H,shift,res", [
    (96, 3, 28, 3, 56),     # Swin-T/S stage 0 (head-fastest grid with nH = 3), shifted 4x4 windows
    (96, 3, 24, 3, 56),     # ... local crop: padded 24 -> 28
    (192, 6, 14, 3, 28),    # stage 1
    (192, 6, 12, 3, 28),    # stage 1 local crop: padded 12 -> 14
    (768, 24, 7, 0, 7),     # stage 3: one window, nH = 24
    (768, 24, 3, 0, 7),     # stage 3 local crop: padded 3 -> 7
    (128, 4, 14, 3, 56),    # Swin-B stage 0 width
    (1024, 32, 7, 0, 7),    # Swin-B stage 3
])
def test_swin_block_w7_real_heads(C, nH, H, shift, res):
    from test_ops_gpu import _block_case
    _block_case(H, 7, shift, C, nH, res, seed=C + H + shift)


@pytest.mark.parametrize("C,nH,H,shift,res", [
    (96, 3, 28, 7, 56),     # Swin-S W14 stage 0: 2x2 windows of 14, shifted
    (96, 3, 24, 7, 56),     # local crop 24 -> 28
    (128, 4, 28, 0, 56),    # Swin-B W14 stage 0
    (384, 12, 14, 0, 14),   # stage 2: the single un-shifted 14x14 window (models/swin_transformer.py:206-209)
    (384, 12, 6, 0, 14),    # stage 2 local crop: 6 -> 14 (36 real tokens of 196)
    (1024, 32, 7, 0, 7),    # Swin-B stage 3 (ws clamps to 7)
])
def test_swin_block_w14_real_heads(C, nH, H, shift, res):
    from test_ops_gpu import _block_case
    _block_case(H, 14, shift, C, nH, res, seed=C + H + shift + 1)
