"""GPU: the Vision Longformer backbone (esvit_b200.vision_longformer) and its new kernels (csrc/vil_dense.cu).

Dense biased attention at every dense-stage geometry of vil_2262 against fp64 attention; the stream patch embedding and
global-token assembly against Conv2d + LN + cat; the relative-position bias assembly against autograd of the
reference's gather + bicubic interpolate in fp64; the sliding-chunk groups wrapper against per-group
SlidingChunkAttnFn; the module against the reference fixture tests/golden/esvit_vil.pt (forward, n-last taps, both
training steps under the reference's drawn modes) and vil_2262 at real shape against the fp32 oracle (oracle/vil.py);
the vil_2262 training step eager vs CUDA graph, fresh mode draws on replay and per-image DropPath keeps."""
import pytest
import torch
import torch.nn.functional as F

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, assert_close, at_golden, rel

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _dense_ref(qkv, bias, B, L, nH, scale):
    C = 32 * nH
    t = qkv.view(B, L, 3, nH, 32).permute(2, 0, 3, 1, 4)
    s = scale * t[0] @ t[1].transpose(-1, -2) + bias[None]
    return (s.softmax(-1) @ t[2]).transpose(1, 2).reshape(B * L, C)


@pytest.mark.parametrize("L,nH,B", [(197, 12, 3), (37, 12, 3), (49, 24, 3), (9, 24, 3), (197, 12, 33), (9, 24, 40)])
def test_dense_bias_attention_matches_fp64(L, nH, B):
    """B > 16: several images per bias-gradient part (the dq kernel's image loop)"""
    from esvit_b200 import ops
    C, scale = 32 * nH, 32 ** -0.5
    g = torch.Generator(device="cuda").manual_seed(L * 100 + nH)
    qkv = torch.randn(B * L, 3 * C, generator=g, device="cuda").to(BF16)
    bias = torch.randn(nH, L, L, generator=g, device="cuda")
    dout = torch.randn(B * L, C, generator=g, device="cuda").to(BF16)

    def run():
        a = qkv.clone().requires_grad_(True)
        b = bias.clone().requires_grad_(True)
        out = ops.DenseBiasAttnGroupsFn.apply(a, None, b.view(-1), ((B, L, 0, 0),), nH, scale)
        da, db = torch.autograd.grad(out, (a, b), dout)
        return out.detach(), da, db

    got = run()
    a, b = qkv.double().requires_grad_(True), bias.double().requires_grad_(True)
    want = _dense_ref(a, b, B, L, nH, scale)
    da, db = torch.autograd.grad(want, (a, b), dout.double())
    assert_close(got[0], want, TOL_BF16_ACT, "out")
    assert_close(got[1], da, TOL_BF16_GRAD, "dqkv")
    assert_close(got[2], db, TOL_BF16_GRAD, "dbias")
    again = run()
    for x, y in zip(got, again):
        assert torch.equal(x, y)


def test_stream_embed_and_cls_cat_match_conv_ln_cat():
    from esvit_b200 import ops
    torch.manual_seed(0)
    Cin, Cout, p, eps = 64, 96, 2, 1e-6
    geos = [(2, 14, 14), (3, 6, 6)]  # (B, H, W): one global row + H*W map rows per image
    rows = [B * (1 + H * W) for B, H, W in geos]
    x = torch.randn(sum(rows), Cin, device="cuda", dtype=torch.float64)
    w = torch.randn(Cout, Cin, p, p, device="cuda", dtype=torch.float64) * 0.05
    bconv = torch.randn(Cout, device="cuda", dtype=torch.float64) * 0.1
    gam = 1 + 0.1 * torch.randn(Cout, device="cuda", dtype=torch.float64)
    bet = 0.1 * torch.randn(Cout, device="cuda", dtype=torch.float64)
    cls = torch.randn(1, 1, Cout, device="cuda", dtype=torch.float64)
    gout = torch.randn(sum(B * (1 + (H // p) * (W // p)) for B, H, W in geos), Cout, device="cuda",
                       dtype=torch.float64)

    leaves = [t.float().requires_grad_(True) for t in (x, w, bconv, gam, bet, cls)]
    xf, wf, bf, gf, betf, cf = leaves
    w16 = wf.detach().reshape(Cout, -1).to(BF16)
    prev, r0 = [], 0
    for (B, H, W), n in zip(geos, rows):
        prev.append((B, 1 + H * W, 1, H, W, r0))
        r0 += n
    pe = ops.VilStreamEmbedFn.apply(xf, wf, w16, bf, tuple(prev), p)
    _, y = ops.add_layer_norm(None, pe, None, gf, betf, eps, y_bf16=False, delta_bias=bf)
    out = ops.ClsCatGroupsFn.apply(y, cf, tuple((B, (H // p) * (W // p)) for B, H, W in geos))
    grads = torch.autograd.grad(out, leaves, gout.float())

    ref_leaves = [t.clone().requires_grad_(True) for t in (x, w, bconv, gam, bet, cls)]
    xr, wr, br, gr, ber, cr = ref_leaves
    outs, r0 = [], 0
    for (B, H, W), n in zip(geos, rows):
        img = xr[r0:r0 + n].view(B, 1 + H * W, Cin)[:, 1:].transpose(1, 2).reshape(B, Cin, H, W)
        t = F.conv2d(img, wr, br, stride=p).flatten(2).transpose(1, 2)
        t = F.layer_norm(t, (Cout,), gr, ber, eps)
        outs.append(torch.cat([cr.expand(B, -1, -1), t], 1).reshape(-1, Cout))
        r0 += n
    want = torch.cat(outs)
    wgrads = torch.autograd.grad(want, ref_leaves, gout)
    assert_close(out, want, TOL_BF16_ACT, "stream")
    for name, a, b in zip(("dx", "dw", "dbias", "dgamma", "dbeta", "dcls"), grads, wgrads):
        assert_close(a, b, TOL_BF16_GRAD, name)


def _attn_modules():
    from esvit_b200 import vision_longformer as V
    torch.manual_seed(1)
    sc = V.Long2DSCSelfAttention(96, 3, qkv_bias=True, sharew=True, nglo=1, rpe=True, mode=1)
    d3 = V.Attention(384, 12, qkv_bias=True, rpe=True, wx=14, wy=14, nglo=1)
    d4 = V.Attention(768, 24, qkv_bias=True, rpe=True, wx=7, wy=7, nglo=0)
    return sc, d3, d4


def _ref_dense_bias(m, N, table, g2l, g2g):
    """the reference's Attention bias (vision_longformer.py:92-123) by autograd-able torch ops in fp64 on CPU"""
    nH, nglo = m.num_heads, m.nglo
    loc = table[m.relative_position_index.view(-1)].view(m.wx * m.wy, m.wx * m.wy, -1)
    npatch = N - nglo
    if npatch != m.wx * m.wy:
        loc = F.interpolate(loc.reshape(1, m.wx * m.wy, m.wx * m.wy, nH).permute(0, 3, 1, 2),
                            scale_factor=npatch / (m.wx * m.wy), mode='bicubic').permute(0, 2, 3, 1).squeeze(0)
    b = loc.permute(2, 0, 1)
    if nglo:
        top = torch.cat([g2g, g2l[0].unsqueeze(-1).expand(-1, -1, npatch)], -1)
        b = torch.cat([top, torch.cat([g2l[1].unsqueeze(1).expand(-1, npatch, -1), b], -1)], 1)
    return b


def test_bias_assembly_matches_gather_and_interpolate():
    from esvit_b200 import ops
    from esvit_b200 import vision_longformer as V
    from oracle import vil_attn as OV
    sc, d3, d4 = _attn_modules()
    for m, Ns in ((sc, [1 + 56 * 56, 1 + 24 * 24]), (d3, [197, 37]), (d4, [49, 9])):
        m = m.cuda()
        params = [m.local_relative_position_bias_table, getattr(m, "g2l_relative_position_bias", None),
                  getattr(m, "g2g_relative_position_bias", None)]
        (plan, offs) = V.bias_plan(m, Ns, "cuda")
        leaves = [p.detach().clone().requires_grad_(True) if p is not None else None for p in params]
        y = ops.RelBiasFn.apply(*leaves, plan)
        gy = torch.randn_like(y)
        got = torch.autograd.grad(y, [t for t in leaves if t is not None], gy)

        rl = [p.detach().double().cpu().requires_grad_(True) if p is not None else None for p in params]
        pieces = []
        for N, off in zip(Ns, offs):
            if m is sc:
                mm = type("M", (), {})()
                mm.num_heads, mm.local_relative_position_bias_table = m.num_heads, rl[0]
                mm.relative_position_index = m.relative_position_index.cpu()
                mm.g2l_relative_position_bias, mm.g2g_relative_position_bias = rl[1], rl[2]
                b, bg = OV.module_biases(mm, N)
                pieces += [(off[0], b), (off[1], bg)]
            else:
                m_cpu = type("M", (), {})()
                for k in ("num_heads", "nglo", "wx", "wy"):
                    setattr(m_cpu, k, getattr(m, k))
                m_cpu.relative_position_index = m.relative_position_index.cpu()
                pieces.append((off, _ref_dense_bias(m_cpu, N, rl[0], rl[1], rl[2])))
        gyc = gy.double().cpu()
        total = sum((gyc[o:o + t.numel()].view(t.shape) * t).sum() for o, t in pieces)
        want = torch.autograd.grad(total, [t for t in rl if t is not None])
        for o, t in pieces:
            assert_close(y[o:o + t.numel()].view(t.shape), t, 1e-5, "bias")
        for a, b in zip(got, want):
            assert_close(a, b, 1e-5, "dparam")


def test_sliding_chunk_groups_match_per_group():
    from esvit_b200 import ops
    torch.manual_seed(2)
    nH, C, scale = 3, 96, 32 ** -0.5
    geos = [(2, 14), (3, 7)]  # (B, side)
    Ns = [1 + s * s for _, s in geos]
    T = sum(B * N for (B, _), N in zip(geos, Ns))
    q = torch.randn(T, C, device="cuda").to(BF16)
    kv = torch.randn(T, 2 * C, device="cuda").to(BF16)
    bias = torch.randn(nH, 49, 442, device="cuda")
    bgs = [torch.randn(nH, N, device="cuda") for N in Ns]
    modes = torch.tensor([3, 0], dtype=torch.int32, device="cuda")
    dout = torch.randn(T, C, device="cuda").to(BF16)
    # one bias vector: each group's copy of the local bias, then its global-row bias
    vec, groups, o, r0 = [], [], 0, 0
    for (B, s), N, bg in zip(geos, Ns, bgs):
        bo, bgo = o, o + bias.numel()
        vec += [bias.view(-1), bg.view(-1)]
        groups.append((B, s, s, r0, bo, bgo))
        o = bgo + bg.numel()
        r0 += B * N
    vec = torch.cat(vec)
    leaves = [t.clone().requires_grad_(True) for t in (q, kv, vec)]
    out = ops.SlidingChunkAttnGroupsFn.apply(leaves[0], leaves[1], None, None, leaves[2], modes, tuple(groups), nH,
                                             scale)
    got = torch.autograd.grad(out, leaves, dout)
    for gi, ((B, s, _, r0, bo, bgo), N) in enumerate(zip(groups, Ns)):
        sl = slice(r0, r0 + B * N)
        pl = [q[sl].clone().requires_grad_(True), kv[sl].clone().requires_grad_(True),
              bias.clone().requires_grad_(True), bgs[gi].clone().requires_grad_(True)]
        o1 = ops.SlidingChunkAttnFn.apply(*pl, modes[gi:gi + 1].clone(), B, s, s, nH, scale)
        g1 = torch.autograd.grad(o1, pl, dout[sl])
        assert torch.equal(out[sl], o1)
        assert torch.equal(got[0][sl], g1[0]) and torch.equal(got[1][sl], g1[1])
        assert torch.equal(got[2][bo:bo + bias.numel()].view_as(bias), g1[2])
        assert torch.equal(got[2][bgo:bgo + N * nH].view(nH, N), g1[3])


# Gradient gate: TOL_BF16_GRAD for every parameter except the global-token biases `g2l_relative_position_bias`, whose
# gate is set from the reference ALGORITHM's own deviation under bf16 autocast from its fp32 run on the fixture's inputs
# (oracle/measure_vil_autocast.py, H100): up to 0.42 (layer2.1.attn.g2l; each head's one or two values collect the
# gradient of a whole bias row / column, a sum of many cancelling terms).
G2L_TOL = 0.45


def _tol(name: str) -> float:
    return G2L_TOL if name.endswith("g2l_relative_position_bias") else TOL_BF16_GRAD


# ---- the module against the reference fixture and the fp32 oracle ---------------------------------------------------
@pytest.fixture(scope="module")
def G():
    from oracle import make_golden_vil as MG
    return MG.load()


def _model(sd, dense, head_k=None):
    from esvit_b200 import vision_longformer as V
    from esvit_b200.vision_transformer import DINOHead
    from oracle import make_golden_vil as MG
    m = V.msvit(dict(MG.ARGS), use_dense_prediction=dense)
    if head_k:
        m.head = DINOHead(MG.OUT_DIM, head_k)
        if dense:
            m.head_dense = DINOHead(MG.OUT_DIM, head_k)
    else:
        m.head = torch.nn.Identity()
        if dense:
            m.head_dense = torch.nn.Identity()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def test_forward_and_n_last_against_fixture(G):
    F_ = G["features"]
    m = _model(F_["state_dict"], True).train()
    m.force_modes(F_["modes"])
    x = [c.cuda() for c in F_["crops"]]
    with torch.no_grad():
        cls, region, _, npatch = m(x)
    assert npatch == F_["npatch"] == [49, 9]
    assert m._forced_modes == []  # every recorded draw consumed, in the reference's order
    assert_close(*at_golden(cls.cpu(), F_["x_cls"]), TOL_BF16_ACT, "x_cls")
    assert_close(*at_golden(region.cpu(), F_["region"]), TOL_BF16_ACT, "region")
    m.eval()
    with torch.no_grad():
        nl = m.forward_return_n_last_blocks(torch.cat(x[:2]), G["n_last"], False, G["depth"])
    assert_close(*at_golden(nl.cpu(), F_["n_last"]), TOL_BF16_ACT, "n_last")


@pytest.mark.parametrize("name", ["ddino", "dino"])
def test_training_step_against_reference_fixture(G, name):
    """DINOHead heads at K = 4096, teacher and student in train mode, the reference's drawn modes forced: loss, head
    outputs, every parameter gradient"""
    from esvit_b200.losses import DDINOLoss, DINOLoss
    C = G["train"][name]
    K = G["K"]
    temp, stemp = G["temps"]
    m = _model(C["state_dict"], C["dense"], K).train()
    m.force_modes(C["modes"])
    x = [c.cuda() for c in C["crops"]]
    loss_mod = (DDINOLoss if C["dense"] else DINOLoss)(K, len(x), temp, temp, 0, 10, stemp, 0.9).cuda()
    with torch.no_grad():
        t = m(x[:2])
    s = m(x)
    assert m._forced_modes == []
    l = loss_mod(s, t, 1, None)
    l.backward()
    assert abs(float(l) - C["loss"]) < 5e-3 * abs(C["loss"]), (float(l), C["loss"])
    for i, o in enumerate(list(s[:3]) if C["dense"] else [s]):
        assert_close(*at_golden(o.detach().float().cpu(), C["outputs"][i]), TOL_BF16_ACT, f"output {i}")
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == sorted(C["grads"])
    worst = sorted(((rel(*at_golden(grads[k].cpu(), ref)), k) for k, ref in C["grads"].items()), reverse=True)
    print(name, "largest gradient deviations", worst[:6])
    for r, k in worst:
        assert r < _tol(k), (k, r, _tol(k))


def test_vil_2262_real_shape_against_oracle():
    """vil_2262 at 224^2 + 96^2, forced modes: train-mode dense forward and the n = 4 probe features (2304) against
    the fp32 oracle"""
    from esvit_b200 import vision_longformer as V
    from oracle import golden as GD
    from oracle import vil as O
    torch.manual_seed(5)
    m = V.msvit(use_dense_prediction=True, drop_path_rate=0.0)
    m.head_dense = torch.nn.Identity()
    sd = O.seeded(GD.recipe(m.state_dict()), 5)
    m.load_state_dict(sd, strict=True)
    m = m.cuda().train()
    g = torch.Generator().manual_seed(5)
    x = [torch.randn(1, 3, 224, 224, generator=g), torch.randn(1, 3, 96, 96, generator=g)]
    seq = [2, 7, 4, 6, 1, 8, 3, 5]
    m.force_modes(seq)
    with torch.no_grad():
        mout = m([t.cuda() for t in x])
        rcls, rregion, rnp = O.forward_dense(sd, x, iter(seq), True)
    assert mout[3] == rnp == [49, 9]
    print("real shape x_cls / x_region", rel(mout[0], rcls), rel(mout[2], rregion))
    assert_close(mout[0], rcls, TOL_BF16_ACT, "x_cls")
    assert_close(mout[2], rregion, TOL_BF16_ACT, "x_region")
    m.eval()
    depth = [c['n'] for c in m.layer_cfgs]
    with torch.no_grad():
        mn = m.forward_return_n_last_blocks(x[0].cuda(), 4, False, depth)
        rn = O.n_last_blocks(sd, x[0], 4)
    assert mn.shape == (1, 2 * 384 + 2 * 768)
    assert_close(mn, rn, TOL_BF16_ACT, "n_last")


# ---- the training step -------------------------------------------------------------------------------------------
def _crops(B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(B, 3, s, s, generator=g, device="cuda") for s in [224] * 2 + [96] * 8]


def test_step_graph_matches_eager_and_draws_fresh_modes():
    from esvit_b200 import engine
    B = 2
    outs = {}
    for graph in (False, True):
        step, student, teacher, _ = engine.make_step("vil_2262", out_dim=4096, drop_path=0.0, cuda_graph=graph, seed=0)
        nsc = len(student._sc_modules())
        fixed_s = torch.tensor([[3, 5], [1, 8], [2, 7], [4, 6]], dtype=torch.int32, device="cuda")[:nsc]
        fixed_t = fixed_s[:, :1].contiguous()
        student.force_modes(fixed_s)
        teacher.force_modes(fixed_t)
        losses = [float(step(_crops(B, 10 + i), 1, 5e-4, 0.04, 0.996)) for i in range(5)]
        assert len(step._graphs) == (1 if graph else 0)
        outs[graph] = (losses, [p.detach().clone() for p in student.parameters()])
    le, lg = outs[False][0], outs[True][0]
    for a, b in zip(le, lg):
        assert abs(a - b) <= 2e-3 * abs(a), (le, lg)
    # AdamW's normalised updates amplify last-bit gradient differences in parameters that start at zero (biases), so
    # the parameters are compared as one vector
    flat = [torch.cat([p.reshape(-1) for p in outs[k][1]]) for k in (False, True)]
    assert_close(flat[1], flat[0], 1e-3, "parameters")

    step, student, teacher, _ = engine.make_step("vil_2262", out_dim=4096, cuda_graph=True, seed=0)
    seen = []
    for i in range(6):
        step(_crops(B, 20 + i), 1, 5e-4, 0.04, 0.996)
        torch.cuda.synchronize()
        seen.append(student._last_modes.clone())
    assert len(step._graphs) == 1
    s = torch.stack(seen[3:])  # the captured step and its replays (the first three steps run eagerly)
    assert int(s.min()) >= 1 and int(s.max()) <= 8
    assert not all(torch.equal(seen[3], t) for t in seen[4:]), "replays drew the same modes"
    student.eval()
    with torch.no_grad():
        student(_crops(B, 30)[:2])
    assert int(student._last_modes.abs().max()) == 0


def test_drop_path_keeps_are_per_image_including_the_global_row():
    from esvit_b200 import vision_longformer as V
    m = V.msvit(drop_path_rate=0.5).cuda().train()
    st = ((3, 56, 56, 1 + 56 * 56, 0), (2, 24, 24, 1 + 24 * 24, 3 * (1 + 56 * 56)))
    k = m._stage_keeps(0, st, torch.device("cuda"))
    assert k.shape == (4, 3 * (1 + 56 * 56) + 2 * (1 + 24 * 24))
    r0 = 0
    for B, H, W, N, _ in st:
        for b in range(B):
            rows = k[:, r0:r0 + N]
            assert torch.all(rows == rows[:, :1])
            r0 += N
    probs = [blk.drop_prob for blk in m.layer1[1:]]
    for row, p in zip(k, probs):
        assert set(torch.unique(row).tolist()) <= {0.0, torch.tensor(1.0 / (1.0 - p)).float().item()}


def test_bad_inputs_raise():
    from esvit_b200 import vision_longformer as V
    m = V.msvit().cuda()
    with pytest.raises(ValueError):
        m(torch.randn(2, 1, 224, 224, device="cuda"))
    with pytest.raises(ValueError):
        m.forward_return_n_last_blocks(torch.randn(1, 3, 224, 224, device="cuda"), 4, False, [1, 1, 1, 1])
    m.force_modes(torch.zeros(3, 1, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError):
        m(torch.randn(1, 3, 224, 224, device="cuda"))
