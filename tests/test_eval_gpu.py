"""GPU: the evaluation entry points - forward_return_n_last_blocks (eval_linear.py's probe features) and the exact k-NN
classifier (esvit_b200.knn, eval_knn.py's knn_classifier) - against the pinned reference fixture
(tests/golden/esvit_eval.pt), the CPU oracle at real model shapes and fp32 torch at real k-NN sizes."""
import os
from functools import partial

import pytest
import torch
import torch.nn as nn

from helpers import TOL_BF16_ACT, TOL_FP32_KERNEL, assert_close
from oracle import eval as E
from oracle import golden as GD
from oracle import swin as S

pytestmark = pytest.mark.gpu

GOLDEN_EVAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_eval.pt")
U = 2.0 ** -8  # bf16 unit roundoff


@pytest.fixture(scope="module")
def G():
    return E.load_golden_eval(GOLDEN_EVAL)


def _model(img_size, spec, seed=0):
    """CUDA Swin backbone (num_classes = 0) with seeded non-trivial weights -> (model, CPU state_dict)"""
    from esvit_b200.swin_transformer import SwinTransformer
    m = SwinTransformer(img_size=img_size, num_classes=0, drop_path_rate=0.0, norm_layer=partial(nn.LayerNorm, eps=1e-6),
                        **spec)
    sd = GD.seeded_state_dict(GD.recipe(m.state_dict()), seed)
    m.load_state_dict(sd)
    return m.cuda().eval(), sd


def _widths(spec, n):
    w = [spec["embed_dim"] * 2 ** i for i, d in enumerate(spec["depths"]) for _ in range(d)]
    return w[-n:]


# ---- linear-probe features -------------------------------------------------------------------------------------------
def test_n_last_blocks_matches_reference_fixture(G):
    P = G["probe"]
    sp = dict(P["spec"])
    img = sp.pop("img_size")
    m, _ = _model(img, sp)
    m.load_state_dict(P["state_dict"])
    x = P["images"].cuda()
    with torch.no_grad():
        for n, ref in P["features"].items():
            out = m.forward_return_n_last_blocks(x, n, False, list(sp["depths"]))
            assert out.shape == ref.shape and out.dtype == torch.float32, n
            assert_close(out, ref, TOL_BF16_ACT, f"n = {n}")


@pytest.mark.parametrize("arch,ns", [("swin_t_w7", (4,)), ("swin_b_w14", (4, 1))])
def test_n_last_blocks_real_shapes_match_oracle(arch, ns):
    spec = dict(S.SWIN_T_W7 if arch == "swin_t_w7" else S.SWIN_B_W14)
    m, sd = _model(224, spec, seed=5)
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(9))
    ospec = S.SwinSpec(img_size=224, **spec)
    for n in ns:
        with torch.no_grad():
            out = m.forward_return_n_last_blocks(x.cuda(), n, False, list(spec["depths"])).cpu()
            ref = E.n_last_blocks(x, sd, ospec, n)
        widths = _widths(spec, n)
        assert out.shape == (4, sum(widths)), (out.shape, widths)
        if arch == "swin_t_w7" and n == 4:
            assert sum(widths) == 2304
        c0 = 0
        for i, c in enumerate(widths):
            assert_close(out[:, c0:c0 + c], ref[:, c0:c0 + c], TOL_BF16_ACT, f"{arch} n = {n} slice {i}")
            c0 += c


def test_n_last_blocks_consistent_with_knn_features():
    """eval_knn.extract_features runs model(samples) with head = Identity: its pooled features match the oracle, and
    n = 1 gives the same vector (same GEMM / attention kernels on the same rows)."""
    spec = dict(S.SWIN_T_W7)
    m, sd = _model(224, spec, seed=6)
    m.head = nn.Identity()
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(10))
    with torch.no_grad():
        f = m(x.cuda())
        f1 = m.forward_return_n_last_blocks(x.cuda(), 1, False, list(spec["depths"]))
        ref, _ = S.forward_features(x, sd, S.SwinSpec(img_size=224, **spec))
    assert_close(f, ref, TOL_BF16_ACT, "model(x) pooled")
    assert_close(f1, f, TOL_FP32_KERNEL, "n = 1 vs model(x)")


def test_n_last_blocks_rejects_invalid_input():
    m, _ = _model(112, dict(embed_dim=32, depths=(2, 2, 2), num_heads=(1, 2, 4), window_size=7))
    x = torch.randn(1, 3, 112, 112, device="cuda")
    for n, depth in ((1, []), (1, [2, 2]), (1, [2, 2, 3]), (0, [2, 2, 2]), (7, [2, 2, 2]), (-1, [2, 2, 2])):
        with pytest.raises(ValueError):
            m.forward_return_n_last_blocks(x, n, False, depth)


# ---- k-NN ------------------------------------------------------------------------------------------------------------
def _fp32_sims_at(train, test, idx):
    """fp32 similarity of every (test row, neighbour) pair"""
    return (test[:, None, :] * train[idx]).sum(-1)


def _assert_neighbours(sims, idx, ref_sims, ref_idx, train, test, tol=1e-5, name=""):
    """sims within tol; indices equal except swaps between neighbours whose fp32 similarities differ by less than tol"""
    assert sims.shape == ref_sims.shape and idx.dtype == torch.int64
    assert float((sims - ref_sims).abs().max()) <= tol, (name, float((sims - ref_sims).abs().max()))
    diff = idx != ref_idx
    if diff.any():
        rows = diff.any(1).nonzero().view(-1)
        a = _fp32_sims_at(train, test[rows], idx[rows])
        b = _fp32_sims_at(train, test[rows], ref_idx[rows])
        gap = float((a - b).abs()[diff[rows]].max())
        assert gap < tol, (name, gap, int(diff.sum()))
        # a swap, not a different neighbour set (up to ties at the k-th value)
        assert float((a.sort(1, descending=True).values - b.sort(1, descending=True).values).abs().max()) < tol


def test_knn_matches_reference_fixture(G):
    from esvit_b200 import knn
    K = G["knn"]
    xtr, ytr, xte, yte = (t.cuda() for t in K["features"])
    C = K["params"]["num_classes"]
    for k in K["ks"]:
        assert knn.knn_classifier(xtr, ytr, xte, yte, k, K["T"], C) == K["accuracy"][k], k
    kmax = K["idx"].shape[1]
    sims, idx = knn.knn_topk(xtr, xte, kmax)
    ref = K["idx"].cuda()
    ref_sims = _fp32_sims_at(xtr, xte, ref)
    _assert_neighbours(sims, idx, ref_sims, ref, xtr, xte, name="fixture")


@pytest.fixture(scope="module")
def no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = saved


@pytest.mark.parametrize("D", [768, 2304])
def test_knn_real_size_matches_fp32_torch(D, no_tf32):
    from esvit_b200 import knn, ops
    N, M, C, T = 200003, 512, 1000, 0.07
    xtr, ytr, xte, yte = E.clustered_features(21, N, M, D, C, noise=2.0, device="cuda")
    ref_sims, ref_idx = E.knn_topk(xtr, xte, 200)
    for k in (1, 10, 20, 100, 200):
        sims, idx = knn.knn_topk(xtr, xte, k)
        _assert_neighbours(sims, idx, ref_sims[:, :k], ref_idx[:, :k], xtr, xte, name=f"D {D} k {k}")
        top = knn.knn_classifier(xtr, ytr, xte, yte, k, T, C)
        h1, h5 = E.knn_vote(ref_sims[:, :k], ref_idx[:, :k], ytr, yte, T, C)
        assert top == (h1 * 100.0 / M, h5 * 100.0 / M), (D, k, top, h1, h5)
    # the bf16 GEMM's error against the exact product stays inside delta's constant (this tests that wgmma accumulates
    # no worse than D 2^-23 relative)
    rows = slice(0, 64)
    s16 = ops.gemm(xte[rows].to(torch.bfloat16), torch.cat([xtr, xtr.new_zeros(5, D)]).to(torch.bfloat16))[:, :N]
    exact = xte[rows].double() @ xtr.double().t()
    bound = xte[rows].norm(dim=1).double()[:, None] * xtr.norm(dim=1).double()[None, :]
    worst = float(((s16.double() - exact).abs() / bound).max())
    assert worst < 3 * U + 4 * U * U + D * 2.0 ** -23, worst


@pytest.mark.parametrize("scale", [10.0, 0.1])
def test_knn_non_unit_norm_features(scale, no_tf32):
    from esvit_b200 import knn
    xtr, _, xte, _ = E.clustered_features(22, 50003, 256, 768, 1000, noise=2.0, device="cuda")
    xtr, xte = xtr * scale, xte * scale
    ref_sims, ref_idx = E.knn_topk(xtr, xte, 100)
    sims, idx = knn.knn_topk(xtr, xte, 100)
    _assert_neighbours(sims, idx, ref_sims, ref_idx, xtr, xte, tol=1e-5 * scale * scale, name=f"scale {scale}")


def test_knn_capacity_rerun_stays_exact(no_tf32):
    """5000 train rows within delta of one another (perturbations far below bf16 resolution) put more candidates into
    a row than its buffer holds: the row is rerun with a buffer of the reported size and stays exact."""
    from esvit_b200 import knn
    g = torch.Generator(device="cuda").manual_seed(23)
    xtr, _, xte, _ = E.clustered_features(23, 20000, 64, 768, 100, noise=2.0, device="cuda")
    v = xte[0]
    near = torch.nn.functional.normalize(v + 1e-4 * torch.randn(5000, 768, generator=g, device="cuda") / 768 ** 0.5,
                                         dim=1)
    xtr = torch.cat([xtr, near])
    ref_sims, ref_idx = E.knn_topk(xtr, xte, 10)
    sims, idx = knn.knn_topk(xtr, xte, 10)
    assert knn.last_stats["rerun_rows"] > 0 and knn.last_stats["max_candidates"] > 10 + knn._CAP_SLACK, knn.last_stats
    _assert_neighbours(sims, idx, ref_sims, ref_idx, xtr, xte, name="rerun")


def test_knn_is_deterministic():
    from esvit_b200 import knn
    xtr, ytr, xte, yte = E.clustered_features(24, 100003, 256, 768, 1000, noise=2.0, device="cuda")
    a = knn.knn_topk(xtr, xte, 20)
    b = knn.knn_topk(xtr, xte, 20)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert knn.knn_classifier(xtr, ytr, xte, yte, 20, 0.07) == knn.knn_classifier(xtr, ytr, xte, yte, 20, 0.07)


def test_knn_rejects_invalid_input():
    from esvit_b200 import knn
    xtr, ytr, xte, yte = E.clustered_features(25, 1000, 16, 64, 10, device="cuda")
    with pytest.raises(ValueError):  # D % 8 != 0
        knn.knn_topk(xtr[:, :60].contiguous(), xte[:, :60].contiguous(), 5)
    with pytest.raises(ValueError):  # k > N
        knn.knn_topk(xtr, xte, 1001)
    with pytest.raises(ValueError):  # class scores beyond shared memory
        knn.knn_classifier(xtr, ytr, xte, yte, 5, 0.07, num_classes=knn.MAX_CLASSES + 1)
    with pytest.raises(ValueError):  # train label outside [0, num_classes)
        knn.knn_classifier(xtr, ytr, xte, yte, 5, 0.07, num_classes=int(ytr.max()))
    with pytest.raises(ValueError):  # negative test label
        knn.knn_classifier(xtr, ytr, xte, yte - 100, 5, 0.07, num_classes=10)
    with pytest.raises(ValueError):  # CPU features
        knn.knn_topk(xtr.cpu(), xte.cpu(), 5)
    with pytest.raises(ValueError):  # non-fp32 features
        knn.knn_topk(xtr.half(), xte.half(), 5)
