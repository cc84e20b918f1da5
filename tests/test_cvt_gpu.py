"""GPU: the CvT backbone - the conv-embed gather / col2im, depthwise conv + BatchNorm and window-attention kernels against
fp64 torch, the QuickGELU GEMM epilogue, and esvit_b200.cvt_v4_transformer.CvT against the pinned reference fixture
(tests/golden/esvit_cvt.pt) and the fp32 oracle (oracle/cvt.py)."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, assert_close, at_golden, rel
from oracle import cvt as O
from oracle import golden as GD
from oracle import make_golden_cvt as MG

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
# CvT-13 stage geometries: (Cin, Cout, k, stride, pad, input side at 224, input side at 96)
EMBED = [(3, 64, 7, 4, 2, 224, 96), (64, 192, 3, 2, 1, 56, 24), (192, 384, 3, 2, 1, 28, 12), (384, 768, 3, 2, 1, 14, 6)]
EMBED_CASES = [(g, r) for g in EMBED for r in (0, 1)]
# (C, heads, map side) of every CvT-13 stage at 224^2 and 96^2
ATTN = [(64, 1, 56), (192, 3, 28), (384, 6, 14), (768, 12, 7), (64, 1, 24), (192, 3, 12), (384, 6, 6), (768, 12, 3)]


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---- conv embed -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geo,res", EMBED_CASES)
def test_conv_embed_against_conv2d(geo, res):
    from esvit_b200 import ops
    Cin, Cout, k, s, p = geo[:5]
    S = geo[5 + res]
    B = 4
    g = _gen(1)
    x = torch.randn(B, Cin, S, S, generator=g, device="cuda")
    w = torch.randn(Cout, Cin, k, k, generator=g, device="cuda") * 0.05
    bias = torch.randn(Cout, generator=g, device="cuda") * 0.1
    K = Cin * k * k
    w16 = F.pad(w.reshape(Cout, K), (0, -K % 8)).to(BF16)
    xb = x.to(BF16).float()   # the rows are bf16: compare against the conv of the same rounded input
    wp = w.detach().clone().requires_grad_(True)
    if Cin == 3:
        y = ops.ConvEmbedFn.apply(None, wp, w16, bias, [xb], None, k, s, p)
        xt = None
    else:
        xt = xb.permute(0, 2, 3, 1).reshape(-1, Cin).contiguous().requires_grad_(True)
        y = ops.ConvEmbedFn.apply(xt, wp, w16, bias, None, ((B, S, S, 0),), k, s, p)
    ref_in = xb.double().requires_grad_(True)
    ref = F.conv2d(ref_in, w16.float()[:, :K].reshape(w.shape).double(), bias.double(), stride=s, padding=p)
    So = ref.shape[-1]
    assert_close(y.float().view(B, So, So, Cout), ref.permute(0, 2, 3, 1), 4e-3, "conv embed fwd")
    gy = torch.randn(B * So * So, Cout, generator=g, device="cuda").to(BF16)
    y.backward(gy)
    ref.backward(gy.double().view(B, So, So, Cout).permute(0, 3, 1, 2))
    wr = w16.float()[:, :K].reshape(w.shape).double().requires_grad_(True)
    F.conv2d(xb.double(), wr, None, stride=s, padding=p).backward(gy.double().view(B, So, So, Cout).permute(0, 3, 1, 2))
    assert_close(wp.grad, wr.grad, 1e-5, "dW")
    if xt is not None:
        assert_close(xt.grad.view(B, S, S, Cin), ref_in.grad.permute(0, 2, 3, 1), 8e-3, "dx")   # bf16 rows gradient
        # reproducible
        xt.grad = None
        ops.ConvEmbedFn.apply(xt, wp, w16, bias, None, ((B, S, S, 0),), k, s, p).backward(gy)
        d1 = xt.grad.clone()
        xt.grad = None
        ops.ConvEmbedFn.apply(xt, wp, w16, bias, None, ((B, S, S, 0),), k, s, p).backward(gy)
        assert torch.equal(d1, xt.grad)


# ---- depthwise conv + BatchNorm -----------------------------------------------------------------------------------
def _dwbn_ref(y, B, H, W, w, Hp, Wp, bn, train):
    """fp64: pad -> dw conv -> BN on [B, C, Hp, Wp]; returns (out token-major [B*Hp*Wp, C], input leaf)"""
    C = y.shape[1]
    yi = y.double().view(B, H, W, C).permute(0, 3, 1, 2).detach().requires_grad_(True)
    t = F.conv2d(F.pad(yi, (0, Wp - W, 0, Hp - H)), w.double(), None, padding=1, groups=C)
    t = F.batch_norm(t, bn["rm"], bn["rv"], bn["g"], bn["b"], train, 0.1, 1e-5)
    return t.permute(0, 2, 3, 1).reshape(-1, C), yi


@pytest.mark.parametrize("train", [True, False])
def test_dwbn_two_groups_against_torch(train):
    """two resolution groups (56 -> window 7, no pad; 24 -> padded to 28) in one call: per-group statistics, running
    statistics updated group by group, num_batches_tracked, forward and every gradient; reruns bit-identical"""
    from esvit_b200 import ops
    C, g = 64, _gen(2)
    geos = [(2, 56, 56, 7), (3, 24, 24, 7)]
    groups, r0, p0 = [], 0, 0
    for B, H, W, w in geos:
        Hp, Wp = ops.win_padded(H, W, w)
        groups.append((B, H, W, w, r0, p0))
        r0 += B * H * W
        p0 += B * Hp * Wp
    y = (torch.randn(r0, C, generator=g, device="cuda") * 0.7 + 0.2).to(BF16)
    bn = nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.copy_(1 + 0.1 * torch.randn(C, generator=g, device="cuda"))
        bn.bias.copy_(0.1 * torch.randn(C, generator=g, device="cuda"))
        bn.running_mean.copy_(0.1 * torch.randn(C, generator=g, device="cuda"))
        bn.running_var.copy_(1 + torch.rand(C, generator=g, device="cuda"))
    w = (torch.randn(C, 1, 3, 3, generator=g, device="cuda") * 0.3).requires_grad_(True)
    bn0 = copy.deepcopy(bn)
    bn.train(train)
    yl = y.clone().requires_grad_(True)
    out = ops.DwBnFn.apply(yl, w, bn.weight, bn.bias, bn, tuple(groups), train, None)
    gout = torch.randn(out.shape, generator=g, device="cuda").to(BF16)
    out.backward(gout)
    st = dict(rm=bn0.running_mean.double().clone(), rv=bn0.running_var.double().clone(),
              g=bn0.weight.double().detach().clone().requires_grad_(True),
              b=bn0.bias.double().detach().clone().requires_grad_(True))
    wd = w.detach().double().requires_grad_(True)
    dy_ref = []
    for (B, H, W, ws, r0_, p0_) in groups:
        Hp, Wp = ops.win_padded(H, W, ws)
        o, yi = _dwbn_ref(y[r0_:r0_ + B * H * W], B, H, W, wd, Hp, Wp, st, train)
        assert_close(out[p0_:p0_ + B * Hp * Wp].float(), o, 1.5e-2, "dwbn fwd")   # bf16 conv output and store
        o.backward(gout[p0_:p0_ + B * Hp * Wp].double())
        dy_ref.append(yi.grad.permute(0, 2, 3, 1).reshape(-1, C))
    assert_close(yl.grad.float(), torch.cat(dy_ref), 2e-2, "dy")
    assert_close(w.grad, wd.grad, 1e-2, "dW")
    assert_close(bn.weight.grad, st["g"].grad, 1e-2, "dgamma")
    assert_close(bn.bias.grad, st["b"].grad, 1e-3, "dbeta")
    assert_close(bn.running_mean, st["rm"], 1e-4, "running_mean")
    assert_close(bn.running_var, st["rv"], 1e-4, "running_var")
    assert int(bn.num_batches_tracked) == (2 if train else 0)
    # reruns from the same buffers: bit-identical outputs and gradients
    res = []
    for _ in range(2):
        b2 = copy.deepcopy(bn0).train(train)
        w.grad = None
        yl.grad = None
        o = ops.DwBnFn.apply(yl, w, b2.weight, b2.bias, b2, tuple(groups), train, None)
        o.backward(gout)
        res.append((o, yl.grad.clone(), w.grad.clone(), b2.weight.grad.clone(), b2.running_var.clone()))
    for a, b in zip(*res):
        assert torch.equal(a, b)


# ---- window attention ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geo", ATTN)
def test_window_attention_against_fp64(geo):
    from esvit_b200 import ops
    C, nH, S = geo
    B = 2
    w = min(7, S)
    Hp, Wp = ops.win_padded(S, S, w)
    g = _gen(3)
    qkv = (torch.randn(B * Hp * Wp, 3 * C, generator=g, device="cuda") * 3).to(BF16).requires_grad_(True)
    grp = ((B, S, S, w, 0, 0),)
    scale = C ** -0.5
    out = ops.MhsaWinGroupsFn.apply(qkv, None, grp, nH, scale)
    q64 = qkv.detach().double().requires_grad_(True)
    t = q64.view(B, Hp // w, w, Wp // w, w, 3, nH, 64).permute(5, 0, 1, 3, 6, 2, 4, 7)
    t = t.reshape(3, B * (Hp // w) * (Wp // w), nH, w * w, 64)
    p = (t[0] @ t[1].transpose(-1, -2) * scale).softmax(-1)
    o = (p @ t[2]).view(B, Hp // w, Wp // w, nH, w, w, 64).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, Hp, Wp, C)
    o = o[:, :S, :S].reshape(-1, C)
    assert_close(out.float(), o, 1e-2, "out")
    go = torch.randn(out.shape, generator=g, device="cuda").to(BF16)
    out.backward(go)
    o.backward(go.double())
    assert_close(qkv.grad.float(), q64.grad, 2e-2, "dqkv")
    d1 = qkv.grad.clone()
    qkv.grad = None
    o2 = ops.MhsaWinGroupsFn.apply(qkv, None, grp, nH, scale)
    o2.backward(go)
    assert torch.equal(o2, out) and torch.equal(qkv.grad, d1)


# ---- QuickGELU epilogue ---------------------------------------------------------------------------------------------
def test_quick_gelu_epilogue_and_derivative():
    from esvit_b200 import ops
    g = _gen(4)
    a = (torch.randn(1000, 192, generator=g, device="cuda")).to(BF16)
    w = (torch.randn(768, 192, generator=g, device="cuda") * 0.2).to(BF16)
    b = torch.randn(768, generator=g, device="cuda")
    h, d = ops.gemm(a, w, b, act=2, want_pre=True)
    x = a.double() @ w.double().t() + b.double()
    s = torch.sigmoid(1.702 * x)
    assert_close(h.float(), x * s, 4e-3, "QuickGELU")
    assert_close(d.float(), s * (1 + 1.702 * x * (1 - s)), 4e-3, "QuickGELU'")
    h2, d2 = ops.gemm(a, w, b, act=2, want_pre=True)
    assert torch.equal(h, h2) and torch.equal(d, d2)
    with pytest.raises(ValueError):
        ops.gemm(a, w.t().contiguous(), b, act=2, b_mn=True)


# Gradient gates (DESIGN.md §2).  TOL_BF16_GRAD for every parameter except two classes, whose gate is set from the
# reference ALGORITHM's own deviation under bf16 autocast from its fp32 run on the same inputs (oracle/
# measure_cvt_autocast.py, H100): the attention PreNorm LayerNorm affine `layers.j.0.norm.*` (BatchNorm right after the
# depthwise conv cancels most of its gradient): reference up to 0.33 (fixture) and 0.44 (CvT-13 real shape); and
# stage0.0.proj.weight: reference 0.090 / 0.078, gated at 0.12 as the Swin / ViT patch-embedding weight.  At the real
# shape the reference's largest deviation over all OTHER parameters is 0.078 (median 0.027): there every other
# parameter is gated at 0.08 instead of TOL_BF16_GRAD.
PRENORM_LN_TOL, STAGE0_PROJ_TOL, REAL_OTHER_TOL = 0.45, 0.12, 0.08


def _tol(name: str, other: float = TOL_BF16_GRAD) -> float:
    if ".1.layers." in name and (name.endswith(".0.norm.weight") or name.endswith(".0.norm.bias")):
        return PRENORM_LN_TOL
    return STAGE0_PROJ_TOL if name == "stage0.0.proj.weight" else other


def _grad_gate(grads: dict, ref: dict, other: float = TOL_BF16_GRAD):
    """-> [(rel-L2 error / its gate, name, rel-L2 error)] sorted, largest first; every ratio must stay below 1"""
    return sorted(((rel(grads[k], r) / _tol(k, other), k, rel(grads[k], r)) for k, r in ref.items()), reverse=True)


# ---- the module against the reference fixture -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def G():
    return MG.load()


def _model(sd, dense, head_k=None):
    from esvit_b200 import cvt_v4_transformer as CV
    from esvit_b200.vision_transformer import DINOHead
    m = CV.cvt(MG.SPEC, use_dense_prediction=dense)
    if head_k:
        m.head = DINOHead(MG.SPEC["DIM_EMBED"][-1], head_k)
        if dense:
            m.head_dense = DINOHead(MG.SPEC["DIM_EMBED"][-1], head_k)
    else:
        m.head = nn.Identity()
        if dense:
            m.head_dense = nn.Identity()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def test_forward_running_stats_and_n_last_against_fixture(G):
    F_ = G["features"]
    m = _model(F_["state_dict"], True).train()
    x = [c.cuda() for c in F_["crops"]]
    with torch.no_grad():
        pooled, region, _, npatch = m(x)
    assert npatch == F_["npatch"]
    assert_close(*at_golden(pooled.cpu(), F_["pooled"]), TOL_BF16_ACT, "pooled")
    assert_close(*at_golden(region.cpu(), F_["region"]), TOL_BF16_ACT, "region")
    sd = m.state_dict()
    for k, v in F_["buffers"].items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v), k
        else:
            assert_close(sd[k].cpu(), v, 2e-2, k)
    m.eval()
    with torch.no_grad():
        nl = m.forward_return_n_last_blocks(torch.cat(x[:2]), G["n_last"], False, MG.SPEC["DEPTH"])
    assert_close(*at_golden(nl.cpu(), F_["n_last"]), TOL_BF16_ACT, "n_last")
    # eval mode leaves the running statistics alone
    assert all(torch.equal(a, b) for a, b in zip(sd.values(), m.state_dict().values()))


@pytest.mark.parametrize("name", ["ddino", "dino"])
def test_training_step_against_reference_fixture(G, name):
    """DINOHead heads at K = 4096, teacher and student in train mode: loss, head outputs, every parameter gradient"""
    from esvit_b200.losses import DDINOLoss, DINOLoss
    C = G["train"][name]
    K = G["K"]
    temp, stemp = G["temps"]
    m = _model(C["state_dict"], C["dense"], K).train()
    x = [c.cuda() for c in C["crops"]]
    loss_mod = (DDINOLoss if C["dense"] else DINOLoss)(K, len(x), temp, temp, 0, 10, stemp, 0.9).cuda()
    with torch.no_grad():
        t = m(x[:2])
    m.load_state_dict(C["state_dict"], strict=True)   # the reference's student starts from the initial buffers
    s = m(x)
    l = loss_mod(s, t, 1, None)
    l.backward()
    assert abs(float(l) - C["loss"]) < 5e-3 * abs(C["loss"]), (float(l), C["loss"])
    for i, o in enumerate(list(s[:3]) if C["dense"] else [s]):
        assert_close(*at_golden(o.detach().float().cpu(), C["outputs"][i]), TOL_BF16_ACT, f"output {i}")
    grads = {k: p.grad for k, p in m.named_parameters() if p.grad is not None}
    assert sorted(grads) == sorted(C["grads"])
    pairs = {k: at_golden(grads[k].cpu(), ref) for k, ref in C["grads"].items()}
    worst = _grad_gate({k: a for k, (a, _) in pairs.items()}, {k: r for k, (_, r) in pairs.items()})
    print(name, "largest gradient deviations / gate", worst[:6])
    for q, k, r in worst:
        assert q < 1, (k, r, _tol(k))


def test_sync_batchnorm_world_size_one(G):
    """convert_sync_batchnorm swaps the containers; at world size 1 the model computes what it computed before"""
    F_ = G["features"]
    x = [c.cuda() for c in F_["crops"]]
    m = _model(F_["state_dict"], True).train()
    ms = nn.SyncBatchNorm.convert_sync_batchnorm(_model(F_["state_dict"], True)).train()
    assert any(isinstance(mod, nn.SyncBatchNorm) for mod in ms.modules())
    with torch.no_grad():
        a, b = m(x), ms(x)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])


def test_invalid_specs_and_inputs(G):
    from esvit_b200 import cvt_v4_transformer as CV
    for key, val in (("REL_POS_EMBED", True), ("SHIFT", [True, False, False, False]), ("KERNEL_QKV", [5, 3, 3, 3]),
                     ("NUM_HEADS", [2, 2, 3, 4]), ("RES_STEM", True)):
        spec = dict(MG.SPEC)
        spec[key] = val
        with pytest.raises(NotImplementedError):
            CV.cvt(spec)
    m = _model(G["features"]["state_dict"], True)
    with pytest.raises(ValueError):
        m(torch.randn(2, 224, 224, device="cuda"))
    with pytest.raises(ValueError):
        m.forward_return_n_last_blocks(torch.randn(2, 3, 224, 224, device="cuda"), 2, False, [1, 1, 1, 1])


def test_cvt13_real_shape_against_oracle():
    """CvT-13 s1, K = 65536, 2 + 8 crops, B = 2 through engine.make_step's networks: forward outputs, loss, DDINO arg-max
    indices on shared features and every parameter gradient against the fp32 oracle in this process"""
    from esvit_b200 import engine
    from oracle import losses as LO
    torch.manual_seed(0)
    K = 65536
    step, student, teacher, loss_mod = engine.make_step(arch="cvt_13", out_dim=K, ncrops=10, drop_path=0.0)
    # the seeded weights (non-trivial biases, LN / BN affine and running statistics) on which the reference's own bf16
    # deviation was measured (oracle/measure_cvt_autocast.py, case "real": same recipe order, seed and crops)
    sd_seed = MG.seeded(GD.recipe(student.state_dict()), 11)
    student.load_state_dict(sd_seed)
    teacher.load_state_dict(sd_seed)
    gen = torch.Generator().manual_seed(5)
    crops = [torch.randn(2, 3, 224, 224, generator=gen) for _ in range(2)] + \
            [torch.randn(2, 3, 96, 96, generator=gen) for _ in range(8)]
    sd0 = {k: v.detach().cpu().clone() for k, v in student.state_dict().items()}
    x = [c.cuda() for c in crops]
    with torch.no_grad():
        t = teacher(x[:2])
    s = student(x)
    l = loss_mod(s, t, 0, None)
    l.backward()
    osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running_" not in k and not k.endswith("weight_g"))
           for k, v in sd0.items()}
    with torch.no_grad():
        ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, O.buffers(sd0), crops[:2], True)
    os_ = O.multicrop_forward(osd, O.buffers(sd0), crops, True)
    zero = torch.zeros(1, K)
    ol = LO.ddino_loss(os_, ot, zero, zero, 10, 0.04, 0.1)
    ol.backward()
    assert abs(float(l) - float(ol)) < 5e-3 * abs(float(ol)), (float(l), float(ol))
    for i in range(3):
        assert_close(s[i].detach().float().cpu(), os_[i].detach(), TOL_BF16_ACT, f"output {i}")
    # arg-max indices: bit-exact when the oracle's matcher is fed the CUDA path's features
    B = 2
    s_feas = torch.split(s[2].detach().float().cpu(), [49 * B] * 2 + [9 * B] * 8)
    t_feas = t[2].detach().float().cpu().chunk(2)
    for iq in range(2):
        for v in range(10):
            if v == iq:
                continue
            T = 49 if v < 2 else 9
            want = LO.region_match(s_feas[v].view(B, T, -1), t_feas[iq].view(B, 49, -1))
            assert torch.equal(loss_mod.last_indices[iq, v, :, :T].cpu(), want), (iq, v)
    got, ref = {}, {}
    for k, p in student.named_parameters():
        if osd[k].grad is None:
            assert p.grad is None or k.endswith("weight_g"), k
            continue
        got[k], ref[k] = p.grad.cpu(), osd[k].grad
    worst = _grad_gate(got, ref, REAL_OTHER_TOL)
    print("largest gradient deviations / gate", worst[:8])
    for q, k, r in worst:
        assert q < 1, (k, r, _tol(k, REAL_OTHER_TOL))


def test_cuda_graph_step_equals_eager_step_with_running_stats():
    from esvit_b200 import engine
    spec = dict(cvt_spec=MG.SPEC, drop_path_rate=0.0)
    gen = torch.Generator().manual_seed(1)
    imgs = [torch.randn(2, 3, 224, 224, generator=gen).cuda() for _ in range(2)] + \
           [torch.randn(2, 3, 96, 96, generator=gen).cuda() for _ in range(2)]
    runs = []
    for graph in (False, True):
        step, student, teacher, _ = engine.make_step(spec=spec, out_dim=1024, ncrops=4, seed=0, cuda_graph=graph)
        ls = [float(step(imgs, 1, 1e-4, 0.04, 0.996)) for _ in range(6)]
        bufs = [b.detach().clone() for n, b in student.named_buffers()] + \
               [b.detach().clone() for n, b in teacher.named_buffers()]
        runs.append((ls, [p.detach().clone() for p in student.parameters()], bufs, len(step._graphs)))
    (le, pe, be, _), (lg, pg, bg, ng) = runs
    assert ng == 1
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)
    assert_close(torch.cat([p.reshape(-1) for p in pg]), torch.cat([p.reshape(-1) for p in pe]), 2e-3, "parameters")
    for a, b in zip(be, bg):
        if a.dtype == torch.long:
            assert torch.equal(a, b)
        else:
            assert_close(b, a, 5e-3, "running statistics")   # batch statistics of the (2e-3-close) weights


def test_weight_gradient_gemm_as_first_call_of_a_thread():
    """autograd runs the backward in its own thread.  When a GEMM is that thread's first CUDA call, no context is
    current there yet and the tensor-map encode returned CUDA_ERROR_INVALID_CONTEXT (seen as ESVIT_ERR_BAD_ARG from the
    conv-embed weight gradient).  A fresh thread whose first CUDA work is the weight-gradient GEMM gives the main
    thread's bits."""
    import threading
    from esvit_b200 import ops
    g = _gen(7)
    dy = torch.randn(12544, 64, generator=g, device="cuda").to(BF16)
    x = torch.randn(12544, 152, generator=g, device="cuda").to(BF16)
    want = ops.gemm_wgrad(dy, x)
    got = {}

    def run():
        try:
            got["dw"] = ops.gemm_wgrad(dy, x)
        except Exception as e:  # reported below, with the assertion
            got["err"] = e

    t = threading.Thread(target=run)
    t.start()
    t.join()
    assert "err" not in got, got.get("err")
    assert torch.equal(got["dw"], want)
