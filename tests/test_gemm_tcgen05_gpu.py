"""wgmma / TMA GEMM with fused bias (+GELU) epilogue against torch (bf16 inputs, fp32 reference math)."""
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.mark.parametrize("M,K,N", [(4096, 96, 384), (1000, 192, 768), (300, 384, 1536), (256, 768, 3072),
                                   (512, 3072, 768), (777, 64, 96), (128, 128, 288), (33, 96, 288), (20000, 96, 96)])
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_bias_act(M, K, N, act):
    from esvit_b200 import ops
    torch.manual_seed(M + K + N)
    d = torch.device("cuda:0")
    a = (torch.randn(M, K, device=d) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=d) / K ** 0.5).to(BF16)
    b = torch.randn(N, device=d) * 0.2
    ref_pre = a.float() @ w.float().t() + b
    ref = F.gelu(ref_pre) if act else ref_pre
    if act:
        out, gp = ops.gemm_bias_act(a, w, b, act=1, want_pre=True)
        xr = ref_pre.clone().requires_grad_(True)
        F.gelu(xr).sum().backward()
        assert_close(gp, xr.grad, 5e-3, "gelu'(pre-activation)")
    else:
        out = ops.gemm_bias_act(a, w, b, act=0)
    torch.cuda.synchronize()
    assert_close(out, ref, 5e-3, "out")
    out2 = ops.gemm_bias_act(a, w, None, act=0)
    assert_close(out2, ref_pre - b, 5e-3, "no bias")


def test_gemm_speed_vs_library(capsys):
    """prints achieved throughput next to the cuBLASLt GEMM + separate GELU kernel it replaces (informational)."""
    from esvit_b200 import ops
    d = torch.device("cuda:0")
    rows = []
    for (M, K, N) in [(696320, 96, 384), (174080, 192, 768), (43520, 384, 1536), (10880, 768, 3072), (43520, 1536, 384)]:
        a = (torch.randn(M, K, device=d) * 0.5).to(BF16)
        w = (torch.randn(N, K, device=d) / K ** 0.5).to(BF16)
        b = torch.randn(N, device=d) * 0.2
        bb = b.to(BF16)

        def mine():
            return ops.gemm_bias_act(a, w, b, act=1, want_pre=True)

        def lib():
            h = F.linear(a, w, bb)
            return ops.GeluFn.apply(h)

        res = []
        for f in (mine, lib):
            for _ in range(3):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                f()
            e1.record()
            torch.cuda.synchronize()
            res.append(e0.elapsed_time(e1) / 10)
        rows.append((M, K, N, res[0], res[1], 2.0 * M * K * N / res[0] / 1e9))
    with capsys.disabled():
        for r in rows:
            print("wgmma gemm+bias+gelu M=%d K=%d N=%d: %.3f ms (library gemm + gelu kernel %.3f ms) %.0f TFLOP/s" % r)


@pytest.mark.parametrize("M,K,N", [(4096, 96, 384), (1000, 192, 768), (300, 384, 1536), (256, 768, 3072),
                                   (777, 64, 96), (33, 96, 288), (20000, 96, 384), (40000, 128, 512)])
def test_gemm_mul_colsum(M, K, N):
    """third epilogue: out = (a @ w^T) * mult, colsum += column sums (fc2 dgrad fused with the GELU backward)."""
    from esvit_b200 import _lib, ops
    torch.manual_seed(M + K + N + 1)
    d = torch.device("cuda:0")
    a = (torch.randn(M, K, device=d) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=d) / K ** 0.5).to(BF16)
    mult = torch.randn(M, N, device=d).to(BF16)
    out = torch.empty(M, N, device=d, dtype=BF16)
    colsum = torch.full((N,), 0.25, device=d)  # accumulates on top of what is there
    ws = torch.empty(ops.GEMM_COLSUM_WS_ROWS * N, device=d)
    _lib.call("esvit_gemm_mul_colsum", ops._p(a), ops._p(w), ops._p(mult), ops._p(out), ops._p(colsum), ops._p(ws), M, N, K,
              ops._stream())
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().t()) * mult.float()
    assert_close(out, ref, 5e-3, "out")
    assert_close(colsum - 0.25, out.float().sum(0), 2e-3, "colsum (of the bf16 outputs)")


def test_mlp_fn_matches_unfused_chain():
    """ops.MlpFn (fused backward) against LinearGeluFn + LinearBiasFn + their separate multiply kernel."""
    from esvit_b200 import ops
    torch.manual_seed(3)
    d = torch.device("cuda:0")
    T, C = 3000, 192
    x = (torch.randn(T, C, device=d) * 0.5).to(BF16)
    w1 = (torch.randn(4 * C, C, device=d) / C ** 0.5).to(BF16)
    w2 = (torch.randn(C, 4 * C, device=d) / (4 * C) ** 0.5).to(BF16)
    b1 = torch.randn(4 * C, device=d) * 0.2
    b2 = (torch.randn(C, device=d) * 0.2).to(BF16)
    g = torch.randn(T, C, device=d).to(BF16)
    outs = []
    for fused in (True, False):
        xs, w1s, w2s, b1s = (t.clone().requires_grad_(True) for t in (x, w1, w2, b1))
        if fused:
            y = ops.MlpFn.apply(xs, w1s, b1s, w2s, b2, w2s.detach().t().contiguous())
        else:
            y = ops.LinearBiasFn.apply(ops.LinearGeluFn.apply(xs, w1s, b1s), w2s, b2)
        y.backward(g)
        outs.append((y, xs.grad, w1s.grad, w2s.grad, b1s.grad))
    torch.cuda.synchronize()
    for name, a, b in zip(("y", "dx", "dw1", "dw2", "db1"), *outs):
        assert_close(a, b, 1e-2, name)


def test_gemm_mul_colsum_speed(capsys):
    """fused fc2-dgrad kernel next to the library GEMM + multiply/bias-gradient kernel it replaces (informational)."""
    from esvit_b200 import _lib, ops
    d = torch.device("cuda:0")
    rows = []
    for (M, C) in [(696320, 96), (174080, 192), (43520, 384), (10880, 768)]:
        N = 4 * C
        a = (torch.randn(M, C, device=d) * 0.5).to(BF16)
        w2 = (torch.randn(C, N, device=d) / N ** 0.5).to(BF16)
        w2t = w2.t().contiguous()
        mult = torch.randn(M, N, device=d).to(BF16)
        out = torch.empty(M, N, device=d, dtype=BF16)
        db = torch.zeros(N, device=d)
        ws = torch.empty(ops.GEMM_COLSUM_WS_ROWS * N, device=d)

        def mine():
            _lib.call("esvit_gemm_mul_colsum", ops._p(a), ops._p(w2t), ops._p(mult), ops._p(out), ops._p(db), ops._p(ws),
                      M, N, C, ops._stream())

        def lib():
            dh = a @ w2
            _lib.call("esvit_mul_bwd_dbias", ops._p(mult), ops._p(dh), ops._p(out), ops._p(db), M, N, ops._stream())

        res = []
        for f in (mine, lib):
            for _ in range(3):
                f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                f()
            e1.record()
            torch.cuda.synchronize()
            res.append(e0.elapsed_time(e1) / 10)
        rows.append((M, C, N, res[0], res[1], (2.0 * M * N * 2 + M * C * 2) / res[0] / 1e6))
    with capsys.disabled():
        for r in rows:
            print("wgmma dgrad*gelu'+colsum M=%d K=%d N=%d: %.3f ms (library gemm + multiply kernel %.3f ms) %.0f GB/s" % r)
