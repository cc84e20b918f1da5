"""GPU: CvT at head dim 32 (experiments/imagenet/cvt_v4/s3.yaml, windows 7, and win_size/s3.yaml, windows 14 / 14 / 14 /
7) - the head-dim-32 window mode of the mhsa kernels against fp64 attention at every window geometry of the 2 + 8-crop
step, esvit_b200.cvt_v4_transformer.CvT against the pinned reference fixtures (tests/golden/esvit_cvt_s3.pt and
esvit_cvt_s3_w14.pt), and the cvt_s3 / cvt_s3_w14 training steps and entry points against the fp32 oracle (oracle/cvt.py
run at head dim 32 by oracle/make_golden_cvt_s3.py)."""
import pytest
import torch
import torch.nn as nn

from helpers import TOL_BF16_ACT, assert_close, at_golden, rel
from oracle import cvt as O
from oracle import golden as GD
from oracle import make_golden_cvt as MG
from oracle import make_golden_cvt_s3 as M3

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
# (C, heads, map side, window) of every stage map of the 2 + 8-crop step at C / heads 64/2, 128/4, 256/8, 512/16.
# s3 (windows 7): 224^2 56, 28, 14, 7 (L = 49); 96^2 24 -> padded 28, 12 -> padded 14 (w 7), 6 (w 6), 3 (w 3).
# win_size/s3: 224^2 56, 28, 14 at w 14 (L = 196, 4 x 4 tiles), 7 at w 7; 96^2 24 -> padded 28 at w 14, 12 (w 12,
# L = 144), 6, 3.
ATTN = [(64, 2, 56, 7), (128, 4, 28, 7), (256, 8, 14, 7), (512, 16, 7, 7), (64, 2, 24, 7), (128, 4, 12, 7),
        (256, 8, 6, 6), (512, 16, 3, 3),
        (64, 2, 56, 14), (128, 4, 28, 14), (256, 8, 14, 14), (64, 2, 24, 14), (128, 4, 12, 12)]


# Gradient gates, set as tests/test_cvt_gpu.py sets them: from the reference ALGORITHM's own rel-L2 deviation under bf16
# autocast from its fp32 run on the same inputs (oracle/measure_cvt_s3_autocast.py, NVIDIA H100 80GB HBM3, 700 W): the
# attention PreNorm LayerNorm affine `layers.j.0.norm.*` up to 0.35 / 0.49 (fixture w7 / w14) and 0.50 / 0.83 (real
# s3 / win_size/s3), every other parameter up to 0.089 / 0.057 (fixture) and 0.071 / 0.093 (real shape, both
# stage0.0.proj.weight).  This path measured at most 0.54 and 0.083 against those gates.
PRENORM_LN_TOL, OTHER_TOL = 0.85, 0.12


def _tol(name: str) -> float:
    if ".1.layers." in name and (name.endswith(".0.norm.weight") or name.endswith(".0.norm.bias")):
        return PRENORM_LN_TOL
    return OTHER_TOL


def _grad_gate(grads: dict, ref: dict):
    """-> [(rel-L2 error / its gate, name, rel-L2 error)] sorted, largest first; every ratio must stay below 1"""
    return sorted(((rel(grads[k], r) / _tol(k), k, rel(grads[k], r)) for k, r in ref.items()), reverse=True)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _groups(geos):
    """((B, H, W, w), ...) -> MhsaWinGroupsFn groups ((B, H, W, w, row0, padded row0), ...), rows T, padded rows Tp"""
    from esvit_b200 import ops
    out, r0, p0 = [], 0, 0
    for B, H, W, w in geos:
        Hp, Wp = ops.win_padded(H, W, w)
        out.append((B, H, W, w, r0, p0))
        r0 += B * H * W
        p0 += B * Hp * Wp
    return tuple(out), r0, p0


def _attn_fp64(q64, groups, nH, scale):
    """fp64 window attention (the reference's Attention.forward :180-218) of the padded qkv rows -> cropped [T, C]"""
    from esvit_b200 import ops
    C = q64.shape[1] // 3
    hd = C // nH
    outs = []
    for B, H, W, w, _, p0 in groups:
        Hp, Wp = ops.win_padded(H, W, w)
        t = q64[p0:p0 + B * Hp * Wp].view(B, Hp // w, w, Wp // w, w, 3, nH, hd).permute(5, 0, 1, 3, 6, 2, 4, 7)
        t = t.reshape(3, B * (Hp // w) * (Wp // w), nH, w * w, hd)
        p = (t[0] @ t[1].transpose(-1, -2) * scale).softmax(-1)
        o = (p @ t[2]).view(B, Hp // w, Wp // w, nH, w, w, hd).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, Hp, Wp, C)
        outs.append(o[:, :H, :W].reshape(-1, C))
    return torch.cat(outs)


def _lse_fp64(q64, groups, nH, scale):
    """fp64 log-sum-exp of the scaled scores, [windows, nH, L] per group, concatenated as the kernels lay it out"""
    from esvit_b200 import ops
    C = q64.shape[1] // 3
    hd = C // nH
    outs = []
    for B, H, W, w, _, p0 in groups:
        Hp, Wp = ops.win_padded(H, W, w)
        t = q64[p0:p0 + B * Hp * Wp].view(B, Hp // w, w, Wp // w, w, 3, nH, hd).permute(5, 0, 1, 3, 6, 2, 4, 7)
        t = t.reshape(3, B * (Hp // w) * (Wp // w), nH, w * w, hd)
        outs.append(torch.logsumexp(t[0] @ t[1].transpose(-1, -2) * scale, -1).reshape(-1))
    return torch.cat(outs)


def _padded_query_rows(groups, Tp):
    """bool [Tp]: rows of the padded maps that are padding (their dq must be exactly 0)"""
    from esvit_b200 import ops
    pad = torch.zeros(Tp, dtype=torch.bool)
    for B, H, W, w, _, p0 in groups:
        Hp, Wp = ops.win_padded(H, W, w)
        m = torch.ones(B, Hp, Wp, dtype=torch.bool)
        m[:, :H, :W] = False
        pad[p0:p0 + B * Hp * Wp] = m.reshape(-1)
    return pad


def _check_attention(geos, C, nH, seed):
    """MhsaWinGroupsFn against fp64 attention on the same bf16 qkv: out, the forward's LSE, dqkv, the qkv-bias gradient
    (the column sums of dqkv), exact zeros for the dq of padded query rows, and bit-identical reruns"""
    from esvit_b200 import _lib, ops
    assert C == 32 * nH
    groups, T, Tp = _groups(geos)
    g = _gen(seed)
    qkv = (torch.randn(Tp, 3 * C, generator=g, device="cuda") * 3).to(BF16).requires_grad_(True)
    bias = torch.zeros(3 * C, device="cuda", requires_grad=True)
    scale = C ** -0.5     # the reference's dim_out ** -0.5, not head_dim ** -0.5
    out = ops.MhsaWinGroupsFn.apply(qkv, bias, groups, nH, scale)
    assert out.shape == (T, C)
    q64 = qkv.detach().double().requires_grad_(True)
    o = _attn_fp64(q64, groups, nH, scale)
    assert_close(out.float(), o, 1e-2, "out")
    lse = torch.empty(Tp * nH, dtype=torch.float32, device="cuda")
    o2 = torch.empty_like(out)
    for B, H, W, w, r0, p0 in groups:
        _lib.call("esvit_mhsa_win_fwd", ops._po(qkv.detach(), p0 * 3 * C), ops._po(o2, r0 * C), ops._po(lse, p0 * nH),
                  B, H, W, w, C, nH, scale, ops._stream())
    assert torch.equal(o2, out)
    assert_close(lse.double(), _lse_fp64(q64.detach(), groups, nH, scale), 1e-5, "lse")
    go = torch.randn(out.shape, generator=g, device="cuda").to(BF16)
    out.backward(go)
    o.backward(go.double())
    assert_close(qkv.grad.float(), q64.grad, 2e-2, "dqkv")
    assert_close(bias.grad, q64.grad.sum(0), 2e-2, "qkv bias grad")
    pad = _padded_query_rows(groups, Tp).cuda()
    assert int(pad.sum()) == Tp - T
    assert not qkv.grad[pad, :C].any()
    d1, b1 = qkv.grad.clone(), bias.grad.clone()
    qkv.grad = bias.grad = None
    o3 = ops.MhsaWinGroupsFn.apply(qkv, bias, groups, nH, scale)
    o3.backward(go)
    assert torch.equal(o3, out) and torch.equal(qkv.grad, d1) and torch.equal(bias.grad, b1)


# ---- window attention kernels ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("geo", ATTN, ids=[f"C{c}-h{h}-S{s}-w{w}" for c, h, s, w in ATTN])
def test_window_attention_against_fp64(geo):
    C, nH, S, window = geo
    _check_attention([(2, S, S, min(window, S))], C, nH, 3)


def test_window_attention_two_groups_in_one_tensor():
    """a 224-derived and a 96-derived stage-0 group (56 unpadded; 24 -> padded to 28) in one buffer, at w 7 and w 14"""
    _check_attention([(2, 56, 56, 7), (3, 24, 24, 7)], 64, 2, 4)
    _check_attention([(2, 56, 56, 14), (3, 24, 24, 14)], 64, 2, 4)


def test_window_attention_rectangular_map_padded_both_ways():
    """30 x 17 in windows of 14 (padded to 42 x 28) and of 7 (padded to 35 x 21), odd head count"""
    _check_attention([(2, 30, 17, 14)], 96, 3, 5)
    _check_attention([(2, 30, 17, 7)], 160, 5, 5)


def test_padded_query_rows_leave_the_output_untouched():
    """a padded map's forward writes exactly the cropped rows: canary rows before and after the output keep their
    bits, and no row of the output keeps the canary"""
    from esvit_b200 import _lib, ops
    for w in (7, 14):
        B, H, W, C, nH = 3, 24, 24, 64, 2
        Hp, Wp = ops.win_padded(H, W, w)
        g = _gen(6)
        qkv = (torch.randn(B * Hp * Wp, 3 * C, generator=g, device="cuda") * 3).to(BF16)
        T, pad = B * H * W, 256
        canary = torch.full((pad + T + pad, C), float("nan"), dtype=BF16, device="cuda")
        buf = canary.clone()
        lse = torch.empty(B * Hp * Wp * nH, dtype=torch.float32, device="cuda")
        _lib.call("esvit_mhsa_win_fwd", ops._p(qkv), ops._po(buf, pad * C), ops._p(lse), B, H, W, w, C, nH, C ** -0.5,
                  ops._stream())
        torch.cuda.synchronize()
        assert torch.equal(buf[:pad].view(torch.int16), canary[:pad].view(torch.int16))
        assert torch.equal(buf[pad + T:].view(torch.int16), canary[pad + T:].view(torch.int16))
        assert not buf[pad:pad + T].isnan().any()
        ref = ops.MhsaWinGroupsFn.apply(qkv, None, ((B, H, W, w, 0, 0),), nH, C ** -0.5)
        assert torch.equal(buf[pad:pad + T], ref)


def test_window_mode_rejects_other_head_dims():
    """esvit_mhsa_win_fwd / _bwd serve C = 64 nH and C = 32 nH only (C = 48 nH and 16 nH are refused before any
    launch); the dense esvit_mhsa_fwd stays at head dim 64"""
    from esvit_b200 import _lib, ops
    B, H, W, w, nH = 2, 14, 14, 7, 2
    for C in (48 * nH, 16 * nH, 32 * nH, 64 * nH):
        qkv = torch.zeros(B * H * W, 3 * C, dtype=BF16, device="cuda")
        out = torch.zeros(B * H * W, C, dtype=BF16, device="cuda")
        lse = torch.empty(B * H * W * nH, dtype=torch.float32, device="cuda")
        dvec = torch.empty_like(lse)
        dqkv = torch.empty_like(qkv)
        args = (B, H, W, w, C, nH, C ** -0.5, ops._stream())
        fwd = lambda: _lib.call("esvit_mhsa_win_fwd", ops._p(qkv), ops._p(out), ops._p(lse), *args)  # noqa: E731
        bwd = lambda: _lib.call("esvit_mhsa_win_bwd", ops._p(qkv), ops._p(out), ops._p(out), ops._p(lse),  # noqa: E731
                                ops._p(dvec), ops._p(dqkv), *args)
        if C in (32 * nH, 64 * nH):
            fwd()
            bwd()
        else:
            with pytest.raises(ValueError):
                fwd()
            with pytest.raises(ValueError):
                bwd()
    torch.cuda.synchronize()
    with pytest.raises(ValueError):
        ops.mhsa(torch.zeros(1, 10, 3 * 64, dtype=BF16, device="cuda"), 2, 0.1)   # dense mode, head dim 32


# ---- the module against the reference fixture -----------------------------------------------------------------------
@pytest.fixture(scope="module")
def G():
    return M3.load()


def _model(spec, sd, dense, head_k=None):
    from esvit_b200 import cvt_v4_transformer as CV
    from esvit_b200.vision_transformer import DINOHead
    m = CV.cvt(spec, use_dense_prediction=dense)
    if head_k:
        m.head = DINOHead(spec["DIM_EMBED"][-1], head_k)
        if dense:
            m.head_dense = DINOHead(spec["DIM_EMBED"][-1], head_k)
    else:
        m.head = nn.Identity()
        if dense:
            m.head_dense = nn.Identity()
    m.load_state_dict(sd, strict=True)
    return m.cuda()


@pytest.mark.parametrize("run", ["w7", "w14"])
def test_forward_running_stats_and_n_last_against_fixture(G, run):
    R_ = G["runs"][run]
    F_ = R_["features"]
    m = _model(R_["spec"], F_["state_dict"], True).train()
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
        nl = m.forward_return_n_last_blocks(torch.cat(x[:2]), G["n_last"], False, R_["spec"]["DEPTH"])
    assert_close(*at_golden(nl.cpu(), F_["n_last"]), TOL_BF16_ACT, "n_last")
    assert all(torch.equal(a, b) for a, b in zip(sd.values(), m.state_dict().values()))


@pytest.mark.parametrize("run,name", [("w7", "ddino"), ("w7", "dino"), ("w14", "ddino")])
def test_training_step_against_reference_fixture(G, run, name):
    """DINOHead heads at K = 4096, teacher and student in train mode: loss, head outputs, every parameter gradient"""
    from esvit_b200.losses import DDINOLoss, DINOLoss
    R_ = G["runs"][run]
    C = R_["train"][name]
    K = G["K"]
    temp, stemp = G["temps"]
    m = _model(R_["spec"], C["state_dict"], C["dense"], K).train()
    x = [c.cuda() for c in C["crops"]]
    loss_mod = (DDINOLoss if C["dense"] else DINOLoss)(K, len(x), temp, temp, 0, 10, stemp, 0.9).cuda()
    with torch.no_grad():
        t = m(x[:2])
    m.load_state_dict(C["state_dict"], strict=True)
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
    print(run, name, "largest gradient deviations / gate", worst[:6])
    for q, k, r in worst:
        assert q < 1, (k, r, _tol(k))


# ---- the real specs -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["cvt_s3", "cvt_s3_w14"])
def test_s3_real_shape_against_oracle(arch):
    """cvt(S3_SPEC) / cvt(S3_W14_SPEC), K = 65536, 2 + 8 crops, B = 2 through engine.make_step's networks: forward
    outputs, loss, DDINO arg-max indices on shared features and every parameter gradient against the fp32 oracle"""
    from esvit_b200 import engine
    from oracle import losses as LO
    torch.manual_seed(0)
    K = 65536
    spec = engine.CVT_SPECS[arch]["cvt_spec"]
    step, student, teacher, loss_mod = engine.make_step(arch=arch, out_dim=K, ncrops=10, drop_path=0.0)
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
    with M3.oracle(spec):
        with torch.no_grad():
            ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, O.buffers(sd0), crops[:2], True)
        os_ = O.multicrop_forward(osd, O.buffers(sd0), crops, True)
    zero = torch.zeros(1, K)
    ol = LO.ddino_loss(os_, ot, zero, zero, 10, 0.04, 0.1)
    ol.backward()
    assert abs(float(l) - float(ol)) < 5e-3 * abs(float(ol)), (float(l), float(ol))
    for i in range(3):
        assert_close(s[i].detach().float().cpu(), os_[i].detach(), TOL_BF16_ACT, f"output {i}")
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
    worst = _grad_gate(got, ref)
    print(arch, "largest gradient deviations / gate", worst[:8])
    for q, k, r in worst:
        assert q < 1, (k, r, _tol(k))


@pytest.mark.parametrize("arch", ["cvt_s3", "cvt_s3_w14"])
@pytest.mark.parametrize("dense", [True, False])
def test_cuda_graph_step_equals_eager_step_with_running_stats(arch, dense):
    """make_step(arch) with the DDINO and the DINO loss: graph replay against eager steps, parameters and the
    BatchNorm running statistics of both networks"""
    from esvit_b200 import engine
    gen = torch.Generator().manual_seed(1)
    imgs = [torch.randn(2, 3, 224, 224, generator=gen).cuda() for _ in range(2)] + \
           [torch.randn(2, 3, 96, 96, generator=gen).cuda() for _ in range(2)]
    runs = []
    for graph in (False, True):
        step, student, teacher, _ = engine.make_step(arch, out_dim=1024, ncrops=4, dense=dense, drop_path=0.0,
                                                     seed=0, cuda_graph=graph)
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
            assert_close(b, a, 5e-3, "running statistics")


@pytest.mark.parametrize("arch", ["cvt_s3", "cvt_s3_w14"])
def test_cuda_graph_step_with_drop_path(arch):
    """the shipped spec (drop_path_rate 0.2) under graph replay against eager steps: the same losses from the same
    DropPath draws, finite, one graph"""
    from esvit_b200 import engine
    gen = torch.Generator().manual_seed(2)
    imgs = [torch.randn(2, 3, 224, 224, generator=gen).cuda() for _ in range(2)] + \
           [torch.randn(2, 3, 96, 96, generator=gen).cuda() for _ in range(8)]
    runs = []
    for graph in (False, True):
        step, student, _, _ = engine.make_step(arch, out_dim=4096, ncrops=10, seed=0, cuda_graph=graph)
        assert student._stage(0)[1].window_size == (14 if arch == "cvt_s3_w14" else 7)
        assert student._stage(3)[1].window_size == 7
        assert max(student._stage(3)[1].drop_probs) == pytest.approx(0.2)
        runs.append(([float(step(imgs, 1, 1e-4, 0.04, 0.996)) for _ in range(5)], len(step._graphs)))
    (le, _), (lg, ng) = runs
    assert ng == 1
    assert all(torch.isfinite(torch.tensor(le + lg))), (le, lg)
    for a, b in zip(le, lg):
        assert abs(a - b) < 2e-3 * abs(a), (le, lg)


# ---- evaluation entry points ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["cvt_s3", "cvt_s3_w14"])
def test_eval_entry_points_against_oracle(arch):
    """the full s3 backbone in eval mode: forward_return_n_last_blocks (eval_linear.py), forward_features and forward
    (eval_knn.py) against the oracle with the running statistics"""
    from esvit_b200 import cvt_v4_transformer as CV
    from esvit_b200 import engine
    spec = engine.CVT_SPECS[arch]["cvt_spec"]
    m = CV.cvt(spec)
    sd = MG.seeded(GD.recipe(m.state_dict()), 12)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    x = torch.randn(3, 3, 224, 224, generator=torch.Generator().manual_seed(8))
    depth = spec["DEPTH"]
    assert depth == [2, 2, 10, 4]
    with torch.no_grad():
        nl = m.forward_return_n_last_blocks(x.cuda(), 5, False, depth)
        pooled = m.forward_features(x.cuda())
        out = m(x.cuda())
        with M3.oracle(spec):
            o_nl = O.n_last_blocks(sd, O.buffers(sd), x, 5)
            o_pooled, _ = O.forward_features(sd, O.buffers(sd), x, False)
    assert nl.shape == o_nl.shape == (3, 256 + 4 * 512)   # the last 5 blocks: 1 of stage 2, 4 of stage 3
    assert_close(nl.cpu(), o_nl, TOL_BF16_ACT, "n_last")
    assert_close(pooled.cpu(), o_pooled, TOL_BF16_ACT, "forward_features")
    assert torch.equal(out, pooled)


def test_invalid_specs():
    """mixed head dims and head dims other than 32 / 64 raise; every other unsupported option still raises"""
    from esvit_b200 import cvt_v4_transformer as CV
    for key, val in (("NUM_HEADS", [2, 2, 3, 4]), ("NUM_HEADS", [4, 8, 12, 16]), ("NUM_HEADS", [2, 4, 6, 4]),
                     ("REL_POS_EMBED", True), ("SHIFT", [True, False, False, False]), ("RES_STEM", True)):
        spec = dict(M3.SPEC)
        spec[key] = val
        with pytest.raises(NotImplementedError):
            CV.cvt(spec)
