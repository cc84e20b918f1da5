"""GPU parity of every esvit_b200 kernel against the CPU oracle / plain fp32 torch on the same seeded inputs."""
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, TOL_FP32_KERNEL, assert_close, load_golden, rel

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


def _dev():
    return torch.device("cuda:0")


@pytest.mark.parametrize("C", [32, 96, 192, 384, 768, 1536, 2048])
@pytest.mark.parametrize("out_bf16", [True, False])
def test_add_layer_norm(C, out_bf16):
    from esvit_b200 import ops
    torch.manual_seed(C)
    B, L = 3, 37
    x = torch.randn(B, L, C) * 2 + 0.3
    delta = (torch.randn(B, L, C) * 0.5).to(BF16)
    keep = torch.tensor([0.0, 1 / 0.9, 1 / 0.9])
    g, b = 1 + 0.1 * torch.randn(C), 0.1 * torch.randn(C)
    gy = torch.randn(B, L, C)
    gx = torch.randn(B, L, C)
    if out_bf16:
        gy = gy.to(BF16).float()

    def ref(x, delta, g, b):
        xo = x + keep.view(B, 1, 1) * delta
        return xo, F.layer_norm(xo, (C,), g, b, 1e-6)

    xr, dr, gr, br = [t.clone().requires_grad_(True) for t in (x, delta.float(), g, b)]
    xo_r, y_r = ref(xr, dr, gr, br)
    (xo_r * gx).sum().backward(retain_graph=True)
    (y_r * gy).sum().backward()

    d = _dev()
    xc, dc, gc, bc = [t.to(d).requires_grad_(True) for t in (x, delta, g, b)]
    xo, y = ops.add_layer_norm(xc, dc, keep.to(d), gc, bc, 1e-6, y_bf16=out_bf16)
    assert y.dtype == (BF16 if out_bf16 else torch.float32)
    torch.autograd.backward([xo, y], [gx.to(d), gy.to(d).to(y.dtype)])
    assert_close(xo, xo_r, 1e-6, "xout")
    assert_close(y, y_r, 5e-3 if out_bf16 else TOL_FP32_KERNEL, "y")
    assert_close(xc.grad, xr.grad, 1e-4, "dx")
    assert_close(dc.grad, dr.grad, 5e-3, "ddelta")
    assert_close(gc.grad, gr.grad, 1e-4, "dgamma")
    assert_close(bc.grad, br.grad, 1e-4, "dbeta")
    # plain LN (no delta) and plain residual add
    x2 = x.to(d).requires_grad_(True)
    _, y2 = ops.add_layer_norm(x2, None, None, gc.detach(), bc.detach(), 1e-6, y_bf16=False)
    assert_close(y2, F.layer_norm(x, (C,), g, b, 1e-6), TOL_FP32_KERNEL, "ln")
    x3, d3 = x.to(d).requires_grad_(True), delta.to(d).requires_grad_(True)
    xo3 = ops.residual_add(x3, d3, None)
    xo3.backward(gx.to(d))
    assert_close(xo3, x + delta.float(), 1e-6, "add")
    assert_close(x3.grad, gx, 1e-6, "add dx")
    assert_close(d3.grad, gx, 5e-3, "add ddelta")


@pytest.mark.parametrize("H,C", [(8, 32), (6, 96), (7, 64), (14, 192), (4, 512)])
def test_patch_merge_ln_groups(H, C):
    """two resolution groups back to back (B = 2 maps of H x H, then 1 map of (H+1) x (H+1)), so the row offsets of
    the second group and the odd / even padding are covered in one call"""
    from esvit_b200 import ops
    from oracle import swin as O
    torch.manual_seed(H * C)
    sizes = ((2, H), (1, H + 1))
    xs = [torch.randn(B, S * S, C) for B, S in sizes]
    g, b = 1 + 0.1 * torch.randn(4 * C), 0.1 * torch.randn(4 * C)
    W = torch.eye(4 * C)  # identity "reduction" so the oracle's gather+LN is observable
    sd = {"m.norm.weight": g.clone().requires_grad_(True), "m.norm.bias": b.clone().requires_grad_(True),
          "m.reduction.weight": W}
    xr = [x.clone().requires_grad_(True) for x in xs]
    y_r = torch.cat([O.patch_merging(x, sd, "m").reshape(-1, 4 * C) for x in xr])
    gy = torch.randn_like(y_r).to(BF16).float()
    (y_r * gy).sum().backward()
    dx_r = torch.cat([x.grad.reshape(-1, C) for x in xr])
    grp, r0 = [], 0
    for B, S in sizes:
        grp.append((B, S, S, r0))
        r0 += B * S * S
    d = _dev()
    xc = torch.cat([x.reshape(-1, C) for x in xs]).to(d).requires_grad_(True)
    gc, bc = g.to(d).requires_grad_(True), b.to(d).requires_grad_(True)
    y = ops.PatchMergeLNGroupsFn.apply(xc, gc, bc, 1e-6, tuple(grp))
    y.backward(gy.to(d).to(BF16))
    assert_close(y, y_r, 5e-3, "y")
    assert_close(xc.grad, dx_r, 1e-4, "dx")
    assert_close(gc.grad, sd["m.norm.weight"].grad, 1e-4, "dgamma")
    assert_close(bc.grad, sd["m.norm.bias"].grad, 1e-4, "dbeta")


@pytest.mark.parametrize("E,S", [(32, 48), (96, 96), (96, 224), (128, 112), (64, 40)])
def test_patch_embed_groups(E, S):
    """two resolution groups written back to back (B = 2 images of S x S, then 1 of (S-8) x (S-8)): the second group's
    row offset, and the weight / bias / LN gradients accumulated over both"""
    from esvit_b200 import ops
    from oracle import swin as O
    torch.manual_seed(E + S)
    imgs = [torch.randn(2, 3, S, S), torch.randn(1, 3, S - 8, S - 8)]
    sd = {"p.proj.weight": (torch.randn(E, 3, 4, 4) * 0.1), "p.proj.bias": torch.randn(E) * 0.1,
          "p.norm.weight": 1 + 0.1 * torch.randn(E), "p.norm.bias": 0.1 * torch.randn(E)}
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    y_r = torch.cat([O.patch_embed(img, sdr, "p", 4).reshape(-1, E) for img in imgs])
    gy = torch.randn_like(y_r)
    (y_r * gy).sum().backward()
    d = _dev()
    ps = {k: v.to(d).requires_grad_(True) for k, v in sd.items()}
    y = ops.PatchEmbedGroupsFn.apply(ps["p.proj.weight"], ps["p.proj.bias"], ps["p.norm.weight"], ps["p.norm.bias"],
                                     1e-6, *[img.to(d) for img in imgs])
    y.backward(gy.to(d))
    assert_close(y, y_r, TOL_FP32_KERNEL, "y")
    for k in sd:
        assert_close(ps[k].grad, sdr[k].grad, 2e-4, k)


@pytest.mark.parametrize("C", [96, 384])
def test_add_layer_norm_with_fused_branch_bias(C):
    """delta already holds the proj / fc2 bias (GEMM epilogue); the add+LN backward also returns that bias'
    gradient (column sums of ddelta), so no separate reduction kernel is needed."""
    from esvit_b200 import ops
    torch.manual_seed(C + 1)
    B, L = 4, 29
    x = torch.randn(B, L, C)
    delta = (torch.randn(B, L, C) * 0.5).to(BF16)
    bias = torch.randn(C) * 0.3
    keep = torch.tensor([0.0, 1 / 0.8, 1 / 0.8, 0.0])
    g, b = 1 + 0.1 * torch.randn(C), 0.1 * torch.randn(C)
    gy, gx = torch.randn(B, L, C).to(BF16).float(), torch.randn(B, L, C)
    xr, dr, br_, gr, ber = [t.clone().requires_grad_(True) for t in (x, delta.float(), bias, g, b)]
    xo_r = xr + keep.view(B, 1, 1) * (dr + (br_ - br_.detach()))
    y_r = F.layer_norm(xo_r, (C,), gr, ber, 1e-6)
    torch.autograd.backward([xo_r, y_r], [gx, gy])
    d = _dev()
    xc, dc, bc_, gc, bec = [t.to(d).requires_grad_(True) for t in (x, delta, bias, g, b)]
    xo, y = ops.add_layer_norm(xc, dc, keep.to(d), gc, bec, 1e-6, y_bf16=True, delta_bias=bc_)
    torch.autograd.backward([xo, y], [gx.to(d), gy.to(d).to(BF16)])
    assert_close(xo, xo_r, 1e-6, "xout")
    assert_close(y, y_r, 5e-3, "y")
    assert_close(xc.grad, xr.grad, 1e-4, "dx")
    assert_close(dc.grad, dr.grad, 5e-3, "ddelta")
    assert_close(bc_.grad, br_.grad, 1e-4, "dbias")
    assert_close(gc.grad, gr.grad, 1e-4, "dgamma")
    # residual add only
    x3, d3, b3 = x.to(d).requires_grad_(True), delta.to(d).requires_grad_(True), bias.to(d).requires_grad_(True)
    xo3 = ops.residual_add(x3, d3, keep.to(d), b3)
    xo3.backward(gx.to(d))
    assert_close(xo3, xo_r, 1e-6, "add")
    assert_close(d3.grad, keep.view(B, 1, 1) * gx, 5e-3, "add ddelta")
    assert_close(b3.grad, (keep.view(B, 1, 1) * gx).sum((0, 1)), 1e-4, "add dbias")


def test_token_mean_groups():
    """two resolution groups back to back: 5 maps of 7 x 7, then 3 maps of 3 x 3"""
    from esvit_b200 import ops
    torch.manual_seed(0)
    xs = [torch.randn(5, 49, 128), torch.randn(3, 9, 128)]
    d = _dev()
    xc = torch.cat([x.reshape(-1, 128) for x in xs]).to(d).requires_grad_(True)
    p = ops.TokenMeanGroupsFn.apply(xc, ((5, 7, 7, 0), (3, 3, 3, 5 * 49)))
    g = torch.randn(8, 128)
    p.backward(g.to(d))
    assert_close(p, torch.cat([x.mean(1) for x in xs]), 1e-6)
    assert_close(xc.grad, torch.cat([(g[:5] / 49).repeat_interleave(49, 0), (g[5:] / 9).repeat_interleave(9, 0)]),
                 1e-6)


def test_gelu_l2norm_weightnorm():
    from esvit_b200 import ops
    torch.manual_seed(1)
    d = _dev()
    x = (torch.randn(64, 256) * 2).to(BF16)
    xr = x.float().requires_grad_(True)
    g = torch.randn(64, 256).to(BF16)
    yr = F.normalize(xr, dim=-1, p=2)
    yr.backward(g.float())
    xc = x.to(d).requires_grad_(True)
    y = ops.L2NormFn.apply(xc, 1e-12)
    y.backward(g.to(d))
    assert_close(y, yr, 4e-3, "l2norm")
    assert_close(xc.grad, xr.grad, 6e-3, "l2norm grad")

    v = torch.randn(512, 64) * 0.05
    gg = 1 + 0.1 * torch.randn(512, 1)
    vr, gr = v.clone().requires_grad_(True), gg.clone().requires_grad_(True)
    wr = vr * (gr / vr.norm(2, dim=1, keepdim=True))
    gw = torch.randn(512, 64).to(BF16)
    wr.backward(gw.float())
    vc, gc = v.to(d).requires_grad_(True), gg.to(d).requires_grad_(True)
    w = ops.WeightNormFn.apply(vc, gc)
    w.backward(gw.to(d))
    assert_close(w, wr, 4e-3, "weight_norm")
    assert_close(vc.grad, vr.grad, 1e-4, "dv")
    assert_close(gc.grad, gr.grad, 1e-4, "dg")


def _block_case(H, ws_cfg, shift_blk, C, nH, res_nominal, seed):
    """my SwinTransformerBlock vs oracle swin_block on one (resolution, window, shift) case, fwd + bwd."""
    from functools import partial

    import torch.nn as nn

    from esvit_b200.swin_transformer import SwinTransformerBlock
    from oracle import swin as O
    torch.manual_seed(seed)
    B = 2
    blk = SwinTransformerBlock(C, (res_nominal, res_nominal), nH, window_size=ws_cfg, shift_size=shift_blk,
                               norm_layer=partial(nn.LayerNorm, eps=1e-6))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in blk.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif p.dim() == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
            elif "relative_position_bias_table" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            else:
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 / math.sqrt(p.shape[1])))
    ws, shift = blk.window_size, blk.shift_size
    sd = {"b." + k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in blk.state_dict().items()}
    x = torch.randn(B, H * H, C, generator=g)
    xr = x.clone().requires_grad_(True)
    y_r = O.swin_block(xr, sd, "b", nH, ws, shift)
    gy = torch.randn(y_r.shape, generator=g)
    (y_r * gy).sum().backward()
    d = _dev()
    blk = blk.to(d)
    xc = x.to(d).requires_grad_(True)
    y, _ = blk(xc)
    y.backward(gy.to(d))
    torch.cuda.synchronize()
    assert_close(y, y_r, TOL_BF16_ACT, f"block out H={H} ws={ws} shift={shift}")
    assert_close(xc.grad, xr.grad, TOL_BF16_GRAD, "dx")
    for n, p in blk.named_parameters():
        assert p.grad is not None, n
        assert_close(p.grad, sd["b." + n].grad, TOL_BF16_GRAD, n)


@pytest.mark.parametrize("H,ws,shift,res", [
    (14, 7, 0, 14), (14, 7, 3, 14),   # 2x2 windows, plain and shifted
    (28, 7, 3, 56),                   # 4x4 windows shifted
    (12, 7, 3, 28),                   # padded 12 -> 14, shifted (96^2 crop, stage 1)
    (6, 7, 3, 14),                    # padded 6 -> 7: single window that STILL gets a shift mask
    (3, 7, 0, 7),                     # padded 3 -> 7, window == nominal resolution (stage 3 local crop)
    (7, 7, 3, 7),                     # nominal res <= window: shift disabled at construction
    (24, 7, 0, 56), (24, 7, 3, 56),   # padded 24 -> 28 (96^2 crop, stage 0)
])
def test_swin_block_w7(H, ws, shift, res):
    _block_case(H, ws, shift, 64, 2, res, seed=H * 10 + shift)


@pytest.mark.parametrize("H,ws,shift,res", [
    (14, 14, 0, 14), (28, 14, 7, 28), (24, 14, 7, 56), (6, 14, 7, 28), (12, 14, 0, 28), (3, 14, 0, 7),
])
def test_swin_block_w14(H, ws, shift, res):
    _block_case(H, ws, shift, 64, 2, res, seed=H * 10 + shift + 1)


def test_swin_block_many_heads():
    _block_case(14, 7, 3, 384, 12, 14, seed=5)


def test_swin_block_w14_many_heads():
    _block_case(28, 14, 7, 256, 8, 28, seed=6)


@pytest.mark.parametrize("gy", [1, 3])
@pytest.mark.parametrize("H,ws,shift,res", [(28, 14, 7, 28), (24, 14, 0, 56), (28, 7, 3, 56), (24, 7, 3, 56)])
def test_swin_block_persistent_loops(monkeypatch, gy, H, ws, shift, res):
    """a forced small grid (ESVIT_ATTN_GY) makes every CTA walk several windows: pipeline stages wrap, per-CTA
    accumulators (bias / qkv-bias gradients) span windows."""
    monkeypatch.setenv("ESVIT_ATTN_GY", str(gy))
    _block_case(H, ws, shift, 64, 2, res, seed=H + ws + shift + gy)


def test_region_match_bit_exact_on_golden_features():
    """argmax indices bit-exact on identical feature inputs (BASELINE.md §3) - features and expected indices are
    the reference's own (tests/golden)."""
    from esvit_b200 import ops
    G = load_golden()["dense"]
    B, ncrops = G["meta"]["batch"], G["meta"]["ncrops"]
    Tg, Tl = G["s_npatch"]
    d = _dev()
    idx, trow = ops.region_match(G["s_fea"].to(d), G["t_fea"].to(d), B, ncrops, Tg, Tl)
    idx = idx.cpu()
    for (iq, v), ref in G["indices"].items():
        T = Tg if v < 2 else Tl
        assert torch.equal(idx[iq, v, :, :T], ref), (iq, v)
    # teacher-row table consistent with the indices
    trow = trow.cpu()
    r = 0
    for v in range(ncrops):
        T = Tg if v < 2 else Tl
        for b in range(B):
            for i in range(T):
                for iq in range(2):
                    exp = -1 if v == iq else (iq * B + b) * Tg + int(G["indices"][(iq, v)][b, i])
                    assert int(trow[r, iq]) == exp
                r += 1


@pytest.mark.parametrize("P", [128, 768, 1024])
def test_region_match_random(P):
    from esvit_b200 import ops
    from oracle import losses as L
    torch.manual_seed(P)
    B, ncrops, Tg, Tl = 3, 4, 49, 9
    s = torch.randn(B * (2 * Tg + 2 * Tl), P)
    t = torch.randn(2 * B * Tg, P)
    idx, _ = ops.region_match(s.to(_dev()), t.to(_dev()), B, ncrops, Tg, Tl)
    idx = idx.cpu()
    split = [Tg * B, Tg * B, Tl * B, Tl * B]
    sf = torch.split(s, split)
    tf = t.chunk(2)
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                assert (idx[iq, v] == -1).all()
                continue
            T = Tg if v < 2 else Tl
            ref = L.region_match(sf[v].view(B, T, P), tf[iq].view(B, Tg, P))
            assert torch.equal(idx[iq, v, :, :T], ref)


def _loss_inputs(B, ncrops, K, Tg, Tl, P, seed):
    g = torch.Generator().manual_seed(seed)
    s_cls = (torch.randn(ncrops * B, K, generator=g) * 0.5).to(BF16)
    t_cls = (torch.randn(2 * B, K, generator=g) * 0.5).to(BF16)
    Rs = B * (2 * Tg + (ncrops - 2) * Tl)
    s_reg = (torch.randn(Rs, K, generator=g) * 0.5).to(BF16)
    t_reg = (torch.randn(2 * B * Tg, K, generator=g) * 0.5).to(BF16)
    s_fea = torch.randn(Rs, P, generator=g)
    t_fea = torch.randn(2 * B * Tg, P, generator=g)
    center = torch.randn(1, K, generator=g) * 0.1
    center_grid = torch.randn(1, K, generator=g) * 0.1
    return s_cls, t_cls, s_reg, t_reg, s_fea, t_fea, center, center_grid


@pytest.mark.parametrize("ce_q", ["1", "0"])  # teacher probabilities stored once per row (default) / recomputed per pairing
@pytest.mark.parametrize("K", [384, 4096])
def test_dino_loss(K, ce_q, monkeypatch):
    monkeypatch.setenv("ESVIT_CE_Q", ce_q)
    from esvit_b200.losses import DINOLoss
    from oracle import losses as L
    B, ncrops = 3, 5
    s_cls, t_cls, *_, center, _ = _loss_inputs(B, ncrops, K, 4, 2, 32, seed=K)
    sr = s_cls.float().requires_grad_(True)
    l_r = L.dino_loss(sr, t_cls.float(), center, ncrops, 0.04, 0.1)
    l_r.backward()
    c_r = L.center_update(center, t_cls.float(), 0.9)
    d = _dev()
    mod = DINOLoss(K, ncrops, 0.04, 0.04, 0, 10).to(d)
    mod.center.copy_(center)
    sc = s_cls.to(d).requires_grad_(True)
    l = mod(sc, t_cls.to(d), 0, None)
    (l * 1.0).backward()
    assert abs(float(l) - float(l_r)) < 1e-4 * abs(float(l_r)), (float(l), float(l_r))
    assert_close(sc.grad, sr.grad, 5e-3, "dlogits")
    assert_close(mod.center, c_r, 1e-5, "center")


@pytest.mark.parametrize("ce_q", ["1", "0"])
@pytest.mark.parametrize("K", [384, 4096])
def test_ddino_loss(K, ce_q, monkeypatch):
    monkeypatch.setenv("ESVIT_CE_Q", ce_q)
    from esvit_b200.losses import DDINOLoss
    from oracle import losses as L
    B, ncrops, Tg, Tl, P = 2, 5, 49, 9, 128
    s_cls, t_cls, s_reg, t_reg, s_fea, t_fea, center, center_grid = _loss_inputs(B, ncrops, K, Tg, Tl, P, seed=K + 1)
    scr, srr = s_cls.float().requires_grad_(True), s_reg.float().requires_grad_(True)
    l_r, idx_r = L.ddino_loss((scr, srr, s_fea, [Tg, Tl]), (t_cls.float(), t_reg.float(), t_fea, [Tg]), center,
                              center_grid, ncrops, 0.04, 0.1, return_indices=True)
    l_r.backward()
    d = _dev()
    mod = DDINOLoss(K, ncrops, 0.04, 0.04, 0, 10).to(d)
    mod.center.copy_(center)
    mod.center_grid.copy_(center_grid)
    sc, sg = s_cls.to(d).requires_grad_(True), s_reg.to(d).requires_grad_(True)
    l = mod((sc, sg, s_fea.to(d), [Tg, Tl]), (t_cls.to(d), t_reg.to(d), t_fea.to(d), [Tg]), 0, None)
    (l * 2.0).backward()  # upstream scale (GradScaler-style) must flow through the device scalar
    assert abs(float(l) - float(l_r)) < 1e-4 * abs(float(l_r)), (float(l), float(l_r))
    for (iq, v), ref in idx_r.items():
        T = Tg if v < 2 else Tl
        assert torch.equal(mod.last_indices[iq, v, :, :T].cpu(), ref)
    assert_close(sc.grad, 2 * scr.grad, 5e-3, "dcls")
    assert_close(sg.grad, 2 * srr.grad, 5e-3, "dregion")
    assert_close(mod.center, L.center_update(center, t_cls.float(), 0.9), 1e-5, "center")
    assert_close(mod.center_grid, L.center_update(center_grid, t_reg.float(), 0.9), 1e-5, "center_grid")


def test_colsum_matches_fp32_sum():
    from esvit_b200 import ops
    torch.manual_seed(3)
    t = torch.randn(777, 4096).to(BF16)
    out = ops.colsum(t.to(_dev()))
    assert_close(out, t.float().sum(0), 1e-5)
    out2 = ops.colsum(t.to(_dev()))
    assert torch.equal(out, out2), "colsum must be deterministic"


def test_ema_bit_exact():
    """teacher EMA copies bit-exact: fl(fl(k*m) + fl(q*(1-m))) like param_k.mul_(m).add_((1-m)*param_q)."""
    from esvit_b200 import ops
    torch.manual_seed(4)
    shapes = [(96,), (288, 96), (169, 3), (7,), (1,), (65536, 16), (33, 5)] + [(17 + i,) for i in range(70)]
    m = 0.996
    ks = [torch.randn(s) for s in shapes]
    qs = [torch.randn(s) for s in shapes]
    ref = [k.clone().mul_(m).add_((1 - m) * q) for k, q in zip(ks, qs)]
    d = _dev()
    kc, qc = [k.to(d) for k in ks], [q.to(d) for q in qs]
    ops.ema_update_(kc, qc, m)
    for a, b in zip(kc, ref):
        assert torch.equal(a.cpu(), b)
    # and against the same two ATen ops executed on the GPU
    kg = [k.to(d).mul_(m).add_((1 - m) * q.to(d)) for k, q in zip(ks, qs)]
    for a, b in zip(kc, kg):
        assert torch.equal(a, b)


def test_clip_gradients_per_tensor():
    from esvit_b200 import ops
    from oracle import losses as L
    torch.manual_seed(5)
    shapes = [(96,), (288, 96), (169, 3), (7,), (4096, 64), (3, 3)] + [(5 + i, 3) for i in range(70)]
    gs = [torch.randn(s) * (10.0 if i % 2 == 0 else 0.01) for i, s in enumerate(shapes)]
    ref = [g.clone() for g in gs]
    norms_r = L.clip_gradients(ref, 3.0)
    d = _dev()
    gc = [g.to(d) for g in gs]
    norms = ops.clip_grads_(gc, 3.0)
    assert_close(norms, torch.tensor(norms_r), 1e-5, "norms")
    for a, b in zip(gc, ref):
        assert_close(a, b, 1e-5, "clipped grad")


@pytest.mark.parametrize("misaligned", [False, True])
def test_fused_adamw_clip_ema_matches_reference_sequence(misaligned):
    """esvit_adamw_ema_multi == utils.clip_gradients -> cancel last_layer grads -> torch.optim.AdamW.step -> EMA loop
    (main_esvit.py:579-590) on a toy module, over 3 steps with changing lr / wd / momentum.  misaligned: the gradients
    are views of ONE flat bucket at odd element offsets (DDP gradient_as_bucket_view style) -> the kernel's scalar path
    must still update every element."""
    import torch.nn as nn

    from esvit_b200.optim import FusedAdamWEMA
    from oracle import losses as L

    class Toy(nn.Module):
        def __init__(self):
            super().__init__()
            self.a = nn.Linear(33, 65)
            self.norm = nn.LayerNorm(65)
            self.last_layer = nn.Linear(65, 130, bias=False)
            self.g = nn.Parameter(torch.ones(130, 1), requires_grad=False)

    torch.manual_seed(7)
    ref_s, ref_t = Toy(), Toy()
    ref_t.load_state_dict(ref_s.state_dict())
    d = _dev()
    s, t = Toy().to(d), Toy().to(d)
    s.load_state_dict(ref_s.state_dict())
    t.load_state_dict(ref_s.state_dict())
    for p_ in list(ref_t.parameters()) + list(t.parameters()):
        p_.requires_grad = False
    reg = [p_ for n, p_ in ref_s.named_parameters() if p_.requires_grad and not (n.endswith(".bias") or p_.dim() == 1)]
    noreg = [p_ for n, p_ in ref_s.named_parameters() if p_.requires_grad and (n.endswith(".bias") or p_.dim() == 1)]
    ropt = torch.optim.AdamW([{"params": reg}, {"params": noreg, "weight_decay": 0.0}])
    fopt = FusedAdamWEMA(s, t, clip_grad=3.0)
    g = torch.Generator().manual_seed(8)
    for it, (lr, wd, mom, skip) in enumerate([(1e-3, 0.04, 0.996, True), (2e-3, 0.05, 0.997, True), (5e-4, 0.1, 0.99, False)]):
        grads = {n: torch.randn(p_.shape, generator=g) * (20.0 if it % 2 == 0 else 0.05)
                 for n, p_ in ref_s.named_parameters() if p_.requires_grad}
        for n, p_ in ref_s.named_parameters():
            p_.grad = grads[n].clone() if n in grads else None
        if misaligned:
            flat = torch.zeros(sum(g_.numel() + 8 for g_ in grads.values()) + 8, device=d)
            off = 1
            for n, p_ in s.named_parameters():
                if n in grads:
                    view = flat[off:off + p_.numel()].view(p_.shape)
                    view.copy_(grads[n])
                    assert view.data_ptr() % 16 != 0
                    p_.grad = view
                    off = ((off + p_.numel() + 3) // 4) * 4 + 1  # every view starts 4 bytes past a 16-byte boundary
                else:
                    p_.grad = None
        else:
            for n, p_ in s.named_parameters():
                p_.grad = grads[n].clone().to(d) if n in grads else None
        # reference sequence
        for i, pg in enumerate(ropt.param_groups):
            pg["lr"] = lr
            if i == 0:
                pg["weight_decay"] = wd
        L.clip_gradients([p_.grad for p_ in ref_s.parameters()], 3.0)
        if skip:
            for n, p_ in ref_s.named_parameters():
                if "last_layer" in n:
                    p_.grad = None
        ropt.step()
        L.ema_update(list(ref_t.parameters()), list(ref_s.parameters()), mom)
        # fused
        fopt.set_hyper(lr, wd, mom)
        fopt.set_skip_last_layer(skip)
        t_before = [p_.detach().clone() for p_ in t.parameters()]
        fopt.step()
        for (n, a), b in zip(s.named_parameters(), ref_s.parameters()):
            assert_close(a, b, 2e-6, f"param {n} step {it}")
        for (n, a), b in zip(t.named_parameters(), ref_t.parameters()):
            assert_close(a, b, 2e-6, f"teacher {n} step {it}")
        for k0, k1, q in zip(t_before, t.parameters(), s.parameters()):  # EMA bit-exact w.r.t. OUR updated student
            assert torch.equal(k1, k0.mul_(mom).add_((1 - mom) * q.detach()))


def test_fused_optimizer_state_dict_interchanges_with_torch_adamw():
    """FusedAdamWEMA.state_dict() uses torch.optim.AdamW's layout over utils.get_params_groups (what the reference saves as
    `optimizer` in its checkpoints, main_esvit.py:476-488): a torch AdamW loads it, and it loads a torch AdamW's."""
    import torch.nn as nn

    from esvit_b200 import utils
    from esvit_b200.optim import FusedAdamWEMA

    class Toy(nn.Module):
        def __init__(self):
            super().__init__()
            self.a = nn.Linear(16, 24)
            self.norm = nn.LayerNorm(24)
            self.last_layer = nn.Linear(24, 40, bias=False)
            self.g = nn.Parameter(torch.ones(40, 1), requires_grad=False)

    torch.manual_seed(3)
    d = _dev()
    s, t = Toy().to(d), Toy().to(d)
    fopt = FusedAdamWEMA(s, t, clip_grad=3.0)
    fopt.set_hyper(1e-3, 0.04, 0.996)
    fopt.set_skip_last_layer(False)
    for p_ in s.parameters():
        p_.grad = torch.randn_like(p_) if p_.requires_grad else None
    fopt.step()
    sd = fopt.state_dict()
    topt = torch.optim.AdamW(utils.get_params_groups(s))
    topt.load_state_dict(sd)  # the reference's restart_from_checkpoint does exactly this
    tparams = [p_ for g_ in topt.param_groups for p_ in g_["params"]]
    reg, noreg = fopt._torch_order()
    for k, i in enumerate(reg + noreg):
        assert tparams[k] is fopt.params[i]
        assert torch.equal(topt.state[tparams[k]]["exp_avg"], fopt.exp_avg[i])
        assert float(topt.state[tparams[k]]["step"]) == 1.0
    # and back: a fresh fused optimiser resumes from the torch optimiser's state
    f2 = FusedAdamWEMA(s, t, clip_grad=3.0)
    f2.load_state_dict(topt.state_dict())
    for a, b in zip(f2.exp_avg_sq, fopt.exp_avg_sq):
        assert torch.equal(a, b)
    assert torch.equal(f2.state[:, 0], fopt.state[:, 0])
