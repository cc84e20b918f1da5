"""GPU: the ViT backbone - esvit_mhsa_fwd / _bwd against fp64 attention of the same bf16 qkv, the token-embedding and
split kernels against fp32 torch, region_match with streamed teacher chunks, and VisionTransformer against the pinned
reference fixture (tests/golden/esvit_vit.pt) and the fp32 oracle (oracle/vit.py)."""
import pytest
import torch
import torch.nn.functional as F

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, TOL_FP32_KERNEL, assert_close, at_golden, rel
from oracle import make_golden_vit as MG
from oracle import vit as V

pytestmark = pytest.mark.gpu

TOL_OUT = 1e-2     # attention output: bf16 store of O and bf16 P in PV
TOL_GRAD = 2e-2    # dq / dk / dv (bf16 dS and stores)
LSE_ABS = 2e-4     # natural-log LSE through ex2 / lg2.approx
# patch_embed.proj.weight: its gradient is the contraction of the bf16 patch rows with the bf16 gradient of the whole
# backbone over every token, and the reference ALGORITHM itself under bf16 autocast deviates from its own fp32 run on
# exactly this tensor by 0.135 (fixture ddino_p16), 0.116 (ddino_p8), 0.017 (dino_p16) and 0.073 (deit_small, K = 65536,
# the inputs of the real-shape test) rel-L2 - in every case the largest deviation of all parameters (median 0.008 -
# 0.020).  Gates for this one tensor: 0.15 on the fixture, 0.12 at the real shape (the Swin real-shape gate of the same
# tensor); every other parameter keeps TOL_BF16_GRAD.
PATCH_W_TOL = {"fixture": 0.15, "real": 0.12}


def _qkv(B, L, nH, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, L, 3 * nH * 64, generator=g, device="cuda") * 1.5).to(torch.bfloat16)


def _ref_attn(qkv, nH):
    """fp64 attention of the bf16 qkv [B, L, 3C] -> (out [B, L, C], lse [B, nH, L]); differentiable w.r.t. qkv64"""
    B, L, C3 = qkv.shape
    t = qkv.reshape(B, L, 3, nH, 64).permute(2, 0, 3, 1, 4)
    s = (t[0] @ t[1].transpose(-2, -1)) * 64 ** -0.5
    lse = torch.logsumexp(s, dim=-1)
    return (s.softmax(-1) @ t[2]).transpose(1, 2).reshape(B, L, C3 // 3), lse


def _run(qkv, groups, nH, g):
    from esvit_b200 import ops
    q = qkv.detach().reshape(-1, qkv.shape[-1]).requires_grad_(True)
    out = ops.MhsaGroupsFn.apply(q, None, groups, nH, 64 ** -0.5)
    out.backward(g)
    return out, q.grad


@pytest.mark.parametrize("L", [37, 50, 145, 197, 785])
@pytest.mark.parametrize("nH", [3, 6, 12])
def test_mhsa_against_fp64(L, nH):
    from esvit_b200 import ops
    qkv = _qkv(1, L, nH, L * 31 + nH)
    g = (torch.randn(L, nH * 64, device="cuda")).to(torch.bfloat16)
    out, dq = _run(qkv, ((1, L, 0),), nH, g)
    _, lse = ops.mhsa(qkv, nH, 64 ** -0.5)
    q64 = qkv.double().requires_grad_(True)
    ref, ref_lse = _ref_attn(q64, nH)
    ref.backward(g.double().view(1, L, -1))
    assert_close(out, ref.view(L, -1), TOL_OUT, "out")
    assert float((lse.double() - ref_lse.detach()).abs().max()) < LSE_ABS
    for part, name in enumerate("qkv"):
        c = nH * 64
        assert_close(dq[:, part * c:(part + 1) * c], q64.grad.view(L, -1)[:, part * c:(part + 1) * c], TOL_GRAD, "d" + name)


def test_mhsa_grouped_buffer_and_reproducible():
    """one buffer of 2 x 197- and 3 x 37-token sequences (global / local crops of p16) == each sequence on its own;
    two runs are bit-identical"""
    nH = 6
    a, b = _qkv(2, 197, nH, 1), _qkv(3, 37, nH, 2)
    qkv = torch.cat([a.reshape(-1, 3 * nH * 64), b.reshape(-1, 3 * nH * 64)])
    T = qkv.shape[0]
    g = torch.randn(T, nH * 64, device="cuda").to(torch.bfloat16)
    groups = ((2, 197, 0), (3, 37, 394))
    out, dq = _run(qkv, groups, nH, g)
    out2, dq2 = _run(qkv, groups, nH, g)
    assert torch.equal(out, out2) and torch.equal(dq, dq2)
    r0 = 0
    for B, L, _ in groups:
        q64 = qkv[r0:r0 + B * L].view(B, L, -1).double().requires_grad_(True)
        ref, _ = _ref_attn(q64, nH)
        ref.backward(g[r0:r0 + B * L].double().view(B, L, -1))
        assert_close(out[r0:r0 + B * L], ref.reshape(B * L, -1), TOL_OUT, f"out L={L}")
        assert_close(dq[r0:r0 + B * L], q64.grad.reshape(B * L, -1), TOL_GRAD, f"dqkv L={L}")
        r0 += B * L


def test_mhsa_rejects_other_head_dims():
    from esvit_b200 import ops
    qkv = torch.zeros(1, 10, 3 * 96, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError):
        ops.mhsa(qkv, 3, 0.1)  # head dim 32


def test_embedding_kernels_against_torch():
    from esvit_b200 import ops
    D, p = 384, 16
    imgs = [torch.randn(2, 3, 224, 224, device="cuda"), torch.randn(3, 3, 96, 96, device="cuda")]
    w = torch.randn(D, 3, p, p, device="cuda") * 0.02
    patches = ops.vit_patches(imgs, p)
    ref_rows = torch.cat([F.unfold(im, p, stride=p).transpose(1, 2).reshape(-1, 3 * p * p) for im in imgs])
    assert torch.equal(patches, ref_rows.to(torch.bfloat16))
    tg = ((2, 196), (3, 36))
    pe = (ref_rows @ w.view(D, -1).t()).to(torch.bfloat16)
    bias = torch.randn(D, device="cuda", requires_grad=True)
    cls = torch.randn(1, 1, D, device="cuda", requires_grad=True)
    pos = [torch.randn(1, 197, D, device="cuda", requires_grad=True), torch.randn(1, 37, D, device="cuda", requires_grad=True)]
    pe_g = pe.detach().requires_grad_(True)
    x = ops.VitTokensGroupsFn.apply(pe_g, bias, cls, tg, *pos)
    c, r = ops.VitSplitGroupsFn.apply(x, tg)
    gc, gr = torch.randn_like(c), torch.randn_like(r)
    (c * gc).sum().add_((r * gr).sum()).backward()
    refs, p0 = [], 0
    cls_r = cls.detach().clone().requires_grad_(True)
    pos_r = [q.detach().clone().requires_grad_(True) for q in pos]
    pe_r = pe.detach().float().requires_grad_(True)
    cl, rg = [], []
    for (B, N), q in zip(tg, pos_r):
        t = torch.cat((cls_r.expand(B, -1, -1), pe_r[p0:p0 + B * N].view(B, N, D)), 1) + q
        cl.append(t[:, 0])
        rg.append(t[:, 1:].reshape(B * N, D))
        p0 += B * N
    cr, rr = torch.cat(cl), torch.cat(rg)
    assert torch.equal(c, cr) and torch.equal(r, rr)
    (cr * gc).sum().add_((rr * gr).sum()).backward()
    assert_close(pe_g.grad, pe_r.grad, 4e-3, "dpe")  # bf16 store of the gradient
    assert_close(bias.grad, pe_r.grad.sum(0), TOL_FP32_KERNEL, "dbias")  # bias is in pe: it only gets the gradient
    assert_close(cls.grad, cls_r.grad, TOL_FP32_KERNEL, "dcls")
    for q, qr in zip(pos, pos_r):
        assert_close(q.grad, qr.grad, TOL_FP32_KERNEL, "dpos")


def _region_ref(sn, tn, B, ncrops, Tg, Tl):
    """oracle.losses.region_match (torch.max over the fp32 cosine similarities, main_esvit.py:735-736) per crop pair"""
    from oracle import losses as LO
    idx = torch.full((2, ncrops, B, Tg), -1, dtype=torch.int64, device=sn.device)
    rows = [(v, b, ((v * B + b) * Tg if v < 2 else 2 * B * Tg + ((v - 2) * B + b) * Tl), Tg if v < 2 else Tl)
            for v in range(ncrops) for b in range(B)]
    for iq in range(2):
        for v, b, r0, T in rows:
            if v == iq:
                continue
            t = tn[(iq * B + b) * Tg:(iq * B + b + 1) * Tg]
            idx[iq, v, b, :T] = LO.region_match(sn[r0:r0 + T][None], t[None])[0]
    return idx


@pytest.mark.parametrize("Tg,Tl,P", [(196, 36, 384), (196, 36, 768), (49, 9, 768), (49, 9, 256)])
def test_region_match_streamed_chunks(Tg, Tl, P):
    """ViT token counts stream the teacher tokens through shared memory (Tg*P*4 > 220 KB); Swin shapes stay one chunk.
    Indices against the oracle's fp32 matcher on the same features, and run to run."""
    from esvit_b200 import ops
    B, ncrops = 2, 10
    g = torch.Generator(device="cuda").manual_seed(Tg + P)
    sn = torch.randn(B * (2 * Tg + (ncrops - 2) * Tl), P, device="cuda", generator=g)
    tn = torch.randn(2 * B * Tg, P, device="cuda", generator=g)
    idx, trow = ops.region_match(sn, tn, B, ncrops, Tg, Tl)
    idx2, trow2 = ops.region_match(sn, tn, B, ncrops, Tg, Tl)
    assert torch.equal(idx, idx2) and torch.equal(trow, trow2)
    ref = _region_ref(sn.cpu(), tn.cpu(), B, ncrops, Tg, Tl).cuda()
    assert torch.equal(idx, ref)


# ---- the module --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def G():
    return MG.load()


def _model(C, spec, dense=True):
    from esvit_b200 import vision_transformer as VT
    import torch.nn as nn
    from functools import partial
    m = VT.VisionTransformer(patch_size=C["patch"], mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                             use_dense_prediction=dense, **spec)
    m.load_state_dict(C["state_dict"], strict=True)
    if dense:
        m.head, m.head_dense = nn.Identity(), nn.Identity()
    return m.cuda()


@pytest.mark.parametrize("name", ["p16", "p8"])
def test_model_against_reference_fixture(G, name):
    C = G["cases"][name]
    m = _model(C, G["spec"]).eval()
    crops = [c.cuda() for c in C["crops"]]
    with torch.no_grad():
        cls, region, _, npatch = m(crops)
        nlast = m.forward_return_n_last_blocks(torch.cat(crops[:2]), 2, True)
    assert npatch == C["npatch"]
    for key, a in (("cls", cls), ("region", region), ("n_last", nlast)):
        a, r = at_golden(a.cpu(), C[key])
        assert_close(a, r, TOL_BF16_ACT, key)


@pytest.mark.parametrize("name", ["p16", "p8"])
def test_model_gradients_against_oracle(G, name):
    C = G["cases"][name]
    nH = G["spec"]["num_heads"]
    m = _model(C, G["spec"]).train()  # drop_path_rate 0: nothing random
    crops = [c.cuda() for c in C["crops"]]
    cls, region, _, _ = m(crops)
    gen = torch.Generator().manual_seed(5)
    gc, gr = torch.randn(cls.shape, generator=gen), torch.randn(region.shape, generator=gen)
    ((cls * gc.cuda()).sum() + (region * gr.cuda()).sum()).backward()
    sd = {k: v.clone().double().requires_grad_(True) for k, v in C["state_dict"].items()}
    oc, orr, _ = V.forward_dense(sd, [c.double() for c in C["crops"]], C["patch"], nH)
    ((oc * gc.double()).sum() + (orr * gr.double()).sum()).backward()
    for k, p in m.named_parameters():
        assert p.grad is not None, k
        assert_close(p.grad.cpu(), sd[k].grad, TOL_BF16_GRAD, k)


def test_n_last_blocks_consistent_with_forward(G):
    C = G["cases"]["p16"]
    m = _model(C, G["spec"], dense=False).eval()
    x = C["crops"][0].cuda()
    with torch.no_grad():
        a = m.forward_return_n_last_blocks(x, 1, False)
        b = m(x)
        maps = m.forward_feature_maps(x)
    assert_close(a, b, 1e-5, "n=1 vs forward")
    assert torch.equal(maps[:, 0], b)


def test_invalid_input_is_rejected(G):
    C = G["cases"]["p16"]
    m = _model(C, G["spec"], dense=False).eval()
    with pytest.raises(ValueError):
        m(torch.randn(1, 3, 224, 192, device="cuda"))
    with pytest.raises(ValueError):
        m(torch.randn(1, 3, 100, 100, device="cuda"))
    with pytest.raises(ValueError):
        m.forward_return_n_last_blocks(torch.randn(1, 3, 224, 224, device="cuda"), 0)
    with pytest.raises(ValueError):
        m.forward_return_n_last_blocks(torch.randn(1, 3, 224, 224, device="cuda"), len(m.blocks) + 1)
    with pytest.raises(NotImplementedError):
        m.forward_selfattention(torch.randn(1, 3, 224, 224, device="cuda"))


def _perturb(student, seed=11):
    """non-trivial biases / LN affine (the reference initialises them to 0 / 1)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in student.named_parameters():
            if n.endswith(".bias") or (p.dim() == 1 and "norm" in n):
                p.add_(torch.randn(p.shape, generator=g).to(p.device) * 0.1)


def test_deit_small_k65536_forward_loss_indices_gradients_match_oracle():
    """deit_small_p16 with its true spec (12 blocks, 6 heads, D 384), DINOHead heads at K = 65536, 2 x 224^2 + 8 x 96^2
    crops at B = 2, DDINO loss: forward outputs, loss, region arg-max indices (bit-exact on shared features) and every
    parameter gradient of the CUDA path against oracle.vit / oracle.losses in fp32 on the CPU."""
    from esvit_b200 import engine
    from oracle import losses as LO
    K, ncrops, B = 65536, 10, 2
    step, student, teacher, loss = engine.make_step(arch="deit_small_p16", out_dim=K, ncrops=ncrops, dense=True,
                                                    device="cuda:0", drop_path=0.0, seed=0)
    _perturb(student)
    teacher.load_state_dict(student.state_dict())
    gen = torch.Generator().manual_seed(1234)
    crops = [torch.randn(B, 3, 224, 224, generator=gen) for _ in range(2)] + \
            [torch.randn(B, 3, 96, 96, generator=gen) for _ in range(ncrops - 2)]
    sd = {k: v.detach().cpu().clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g"))
          for k, v in student.state_dict().items()}
    with torch.no_grad():
        t_ref = V.multicrop_forward({k: v.detach() for k, v in sd.items()}, crops[:2], 16, 6, True)
    s_ref = V.multicrop_forward(sd, crops, 16, 6, True)
    l_ref, idx_ref = LO.ddino_loss(s_ref, t_ref, torch.zeros(1, K), torch.zeros(1, K), ncrops, 0.04, return_indices=True)
    l_ref.backward()

    cc = [c.cuda() for c in crops]
    with torch.no_grad():
        t = teacher(cc[:2])
    s = student(cc)
    l = loss(s, t, 0, None)
    l.backward()
    torch.cuda.synchronize()
    assert list(s[3]) == list(s_ref[3]) == [196, 36]
    assert s[1].shape == (B * (2 * 196 + 8 * 36), K) and t[1].shape == (B * 2 * 196, K)
    for a, b, name in zip(s[:3], s_ref[:3], ("student cls logits", "student region logits", "student features")):
        assert_close(a, b, TOL_BF16_ACT, name)
    for a, b, name in zip(t[:3], t_ref[:3], ("teacher cls logits", "teacher region logits", "teacher features")):
        assert_close(a, b, TOL_BF16_ACT, name)
    assert abs(float(l) - float(l_ref)) < 5e-3 * abs(float(l_ref)), (float(l), float(l_ref))

    # arg-max indices: bit-exact when the oracle's matcher is fed the CUDA path's features (streamed teacher chunks)
    s_feas = torch.split(s[2].detach().float().cpu(), [196 * B] * 2 + [36 * B] * (ncrops - 2))
    t_feas = t[2].detach().float().cpu().chunk(2)
    for iq in range(2):
        for v in range(ncrops):
            if v == iq:
                continue
            T = 196 if v < 2 else 36
            want = LO.region_match(s_feas[v].view(B, T, -1), t_feas[iq].view(B, 196, -1))
            assert torch.equal(loss.last_indices[iq, v, :, :T].cpu(), want), (iq, v)

    bad, worst = {}, (0.0, "")
    for n, p in student.named_parameters():
        if sd[n].grad is None:
            assert p.grad is None or n.endswith("weight_g"), n
            continue
        assert p.grad is not None, n
        if float(sd[n].grad.norm()) <= 1e-7:
            continue
        r = rel(p.grad, sd[n].grad)
        worst = max(worst, (r, n))
        if r >= (PATCH_W_TOL["real"] if n == "patch_embed.proj.weight" else TOL_BF16_GRAD):
            bad[n] = r
    print("deit_small K=65536 worst gradient rel-L2", worst)
    assert not bad, bad


@pytest.mark.parametrize("name", ["ddino_p16", "dino_p16", "ddino_p8"])
def test_training_step_against_reference_fixture(G, name):
    """DINOHead heads at K = 4096, the CUDA DDINOLoss / DINOLoss: head outputs, loss and every parameter gradient against
    what the reference computed (tests/golden/esvit_vit.pt)"""
    from functools import partial
    import torch.nn as nn
    from esvit_b200 import vision_transformer as VT
    from esvit_b200.losses import DDINOLoss, DINOLoss
    C = G["train"][name]
    K = G["K"]
    temp, stemp = G["temps"]
    m = VT.VisionTransformer(patch_size=C["patch"], mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                             use_dense_prediction=C["dense"], **G["spec"])
    m.head = VT.DINOHead(G["spec"]["embed_dim"], K)
    if C["dense"]:
        m.head_dense = VT.DINOHead(G["spec"]["embed_dim"], K)
    m.load_state_dict(C["state_dict"], strict=True)
    m = m.cuda().train()
    x = [c.cuda() for c in C["crops"]]
    loss_mod = (DDINOLoss if C["dense"] else DINOLoss)(K, len(x), temp, temp, 0, 10, stemp, 0.9).cuda()
    with torch.no_grad():
        t = m(x[:2])
    s = m(x)
    l = loss_mod(s, t, 1, None)
    l.backward()
    assert abs(float(l) - C["loss"]) < 5e-3 * abs(C["loss"]), (float(l), C["loss"])
    for i, o in enumerate(list(s[:3]) if C["dense"] else [s]):
        a, r = at_golden(o.detach().float().cpu(), C["outputs"][i])
        assert_close(a, r, TOL_BF16_ACT, f"output {i}")
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == sorted(C["grads"])
    for k, ref in C["grads"].items():
        a, r = at_golden(grads[k].cpu(), ref)
        assert_close(a, r, PATCH_W_TOL["fixture"] if k == "patch_embed.proj.weight" else TOL_BF16_GRAD, k)


def test_drop_path_rows_of_a_forward_match_oracle(G, monkeypatch):
    """student DropPath (linspace(0, 0.1, depth)): the per-(block, branch, image) scales the model draws, broadcast to
    the rows of every resolution group, give the oracle's forward and gradients with the same per-image scales"""
    from functools import partial
    import torch.nn as nn
    from esvit_b200 import backbone, vision_transformer as VT
    C = G["cases"]["p16"]
    nH = G["spec"]["num_heads"]
    m = VT.VisionTransformer(patch_size=16, mlp_ratio=4, qkv_bias=True, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                             use_dense_prediction=True, drop_path_rate=0.5, **G["spec"])
    m.load_state_dict(C["state_dict"], strict=True)
    m.head, m.head_dense = nn.Identity(), nn.Identity()
    m = m.cuda().train()
    drawn = []
    orig = backbone.drop_path_rows
    monkeypatch.setattr(backbone, "drop_path_rows",
                        lambda m_, s, counts, dev: drawn.append((counts, orig(m_, s, counts, dev))) or drawn[-1][1])
    torch.manual_seed(3)
    crops = [c.cuda() for c in C["crops"]]
    cls, region, _, _ = m(crops)
    (counts, keeps), = drawn
    assert keeps is not None and float((keeps == 0).float().mean()) > 0  # something was dropped
    okeeps, r0 = [], 0
    for B, L in counts:
        rows = keeps[:, r0:r0 + B * L].view(keeps.shape[0], B, L)
        assert torch.equal(rows, rows[:, :, :1].expand_as(rows))  # one scale per image
        per = rows[:, :, 0].cpu().double()
        okeeps.append([(per[2 * i], per[2 * i + 1]) for i in range(len(m.blocks))])
        r0 += B * L
    assert r0 == keeps.shape[1]
    assert torch.equal(keeps[0], torch.ones_like(keeps[0]))  # block 0 has drop probability 0
    gen = torch.Generator().manual_seed(5)
    gc, gr = torch.randn(cls.shape, generator=gen), torch.randn(region.shape, generator=gen)
    ((cls * gc.cuda()).sum() + (region * gr.cuda()).sum()).backward()
    sd = {k: v.clone().double().requires_grad_(True) for k, v in C["state_dict"].items()}
    oc, orr, _ = V.forward_dense(sd, [c.double() for c in C["crops"]], 16, nH, okeeps)
    ((oc * gc.double()).sum() + (orr * gr.double()).sum()).backward()
    assert_close(cls.cpu(), oc, TOL_BF16_ACT, "cls")
    assert_close(region.cpu(), orr, TOL_BF16_ACT, "region")
    for k, p in m.named_parameters():
        assert_close(p.grad.cpu(), sd[k].grad, TOL_BF16_GRAD, k)


def test_head_and_loss_kernels_past_2_pow_31_elements():
    """The head and loss path at ViT row counts holds more than 2^31 elements per tensor (deit_small, B = 64: 43 520
    region rows x 65 536).  Rows past element 2^31 are copies of the first rows, so every row-wise result there must
    equal the first rows' bit for bit: the GEMM (forward and input gradient), row LSE and the CE forward / backward; the
    last layer's fp32 weight gradient over all rows matches fp32 torch (the teacher's 25 088 rows stay below 2^31)."""
    from esvit_b200 import ops
    K, D = 65536, 256
    R = (1 << 31) // K + 256                    # 33024 rows: the last 256 start past element 2^31
    base, tail = R - 256, 256
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(tail, D, device="cuda", generator=g).to(torch.bfloat16)
    a = torch.cat([x, torch.randn(base - tail, D, device="cuda", generator=g).to(torch.bfloat16), x])
    w = (torch.randn(K, D, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    s = ops.gemm(a, w)                          # [R, K] bf16
    assert s.numel() > 1 << 31
    assert torch.equal(s[base:], s[:tail])
    dx = ops.gemm(s, w, None, b_mn=True)        # input gradient through the 65536-wide last layer
    assert torch.equal(dx[base:], dx[:tail])
    center = torch.zeros(K, device="cuda")
    lse = ops.row_lse(s, center, 10.0)
    assert torch.equal(lse[base:], lse[:tail])
    t = s[:2].contiguous()
    trow = torch.tensor([[0, 1]], dtype=torch.int32, device="cuda").expand(R, 2).contiguous()
    wgt = torch.ones(R, device="cuda")
    s_g = s.detach().requires_grad_(True)
    loss = ops.DinoCEFn.apply(s_g, t, center, None, trow, wgt, 25.0, 10.0, None)
    loss.backward()
    assert torch.isfinite(loss)
    assert torch.equal(s_g.grad[base:], s_g.grad[:tail])
    dw = ops.gemm_wgrad(s_g.grad, a)           # [K, D] fp32 = dlogits^T a, reads dlogits past element 2^31
    ref = torch.zeros(K, D, device="cuda")
    for r0 in range(0, R, 4096):
        ref += s_g.grad[r0:r0 + 4096].float().t() @ a[r0:r0 + 4096].float()
    assert_close(dw, ref, 1e-4, "last-layer weight gradient")


def test_cuda_graph_step_equals_eager_step():
    """deit_tiny p16, 2 + 2 crops: the captured-and-replayed step computes what the eager step computes.  Not bit-equal,
    for the reason tests/test_model_gpu.py gives (LayerNorm / bias gradients reduced with fp32 atomics, and here also
    torch's bicubic-interpolation backward of the local crops' positional embedding); same 2e-3 gate."""
    from esvit_b200 import engine
    spec = dict(vit_arch="deit_tiny", patch_size=16, drop_path_rate=0.0)
    gen = torch.Generator().manual_seed(1)
    imgs = [torch.randn(2, 3, 224, 224, generator=gen).cuda() for _ in range(2)] + \
           [torch.randn(2, 3, 96, 96, generator=gen).cuda() for _ in range(2)]
    runs = []
    for graph in (False, True):
        step, student, _, _ = engine.make_step(spec=spec, out_dim=1024, ncrops=4, seed=0, cuda_graph=graph)
        ls = [float(step(imgs, 1, 1e-4, 0.04, 0.996)) for _ in range(6)]  # graph side: 3 warm-up, capture, 2 replays
        runs.append((ls, [p.detach().clone() for p in student.parameters()], len(step._graphs)))
    (le, pe, _), (lg, pg, ng) = runs
    assert ng == 1
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)
    # the whole parameter vector: biases start at 0 here, so a single bias is all update and its relative noise is large
    assert_close(torch.cat([p.reshape(-1) for p in pg]), torch.cat([p.reshape(-1) for p in pe]), 2e-3, "parameters")
