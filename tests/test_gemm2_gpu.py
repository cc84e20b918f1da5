"""wgmma / TMA GEMM family (csrc/gemm2_wgmma.cu) against fp32 torch on the same bf16 inputs:
forward (K-major operands), input gradient (MN-major B = the Linear weight as it lies), weight gradient (MN-major A and
B, split-K fp32 partials), every epilogue, the automatic tile choice and every tile shape (1 / 2 consumer warpgroups x
BN 128 / 256), ragged M / N / K."""
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
TILES = [0, 1128, 1256, 2128, 2256]  # 0: the automatic choice; else consumer warpgroups * 1000 + BN

FWD_SHAPES = [(4096, 96, 384), (1000, 192, 768), (300, 384, 1536), (256, 768, 3072), (512, 3072, 768), (777, 64, 96),
              (128, 128, 288), (33, 96, 288), (20000, 96, 96), (640, 256, 4096), (1111, 2048, 256), (260, 96, 16),
              (340, 768, 256), (340, 2048, 2048)]   # DINO head: a depth-1 head's Linear, a hidden Linear


def _mk(M, K, N, seed):
    torch.manual_seed(seed)
    d = torch.device("cuda:0")
    a = (torch.randn(M, K, device=d) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=d) / K ** 0.5).to(BF16)
    b = torch.randn(N, device=d) * 0.2
    return a, w, b


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("M,K,N", FWD_SHAPES)
def test_forward_bias_and_gelu(M, K, N, tile):
    from esvit_b200 import ops
    a, w, b = _mk(M, K, N, M + K + N)
    ref_pre = a.float() @ w.float().t() + b
    out = ops.gemm(a, w, b, tile=tile)
    assert_close(out, ref_pre, 5e-3, "bias epilogue")
    out = ops.gemm(a, w, None, tile=tile)
    assert_close(out, ref_pre - b, 5e-3, "no bias")
    h, gp = ops.gemm(a, w, b, act=1, want_pre=True, tile=tile)
    xr = ref_pre.clone().requires_grad_(True)
    F.gelu(xr).sum().backward()
    assert_close(h, F.gelu(ref_pre), 5e-3, "gelu")
    assert_close(gp, xr.grad, 5e-3, "gelu'")
    h2 = ops.gemm(a, w, b, act=1, tile=tile)
    assert torch.equal(h2, h)


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("M,K,N", [(4096, 384, 96), (1000, 768, 192), (300, 1536, 384), (512, 768, 3072), (777, 96, 64),
                                   (33, 288, 96), (20000, 96, 96), (2000, 4096, 256), (130, 288, 128)])
def test_dgrad_reads_weight_as_it_lies(M, K, N, tile):
    """dx[M,N] = dy[M,K] @ w[K,N] with w the nn.Linear weight [out_features = K, in_features = N]: B is MN-major."""
    from esvit_b200 import ops
    torch.manual_seed(M + K + N + 2)
    d = torch.device("cuda:0")
    dy = (torch.randn(M, K, device=d) * 0.5).to(BF16)
    w = (torch.randn(K, N, device=d) / K ** 0.5).to(BF16)
    out = ops.gemm(dy, w, None, b_mn=True, tile=tile)
    assert_close(out, dy.float() @ w.float(), 5e-3, "dgrad")


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("T,N,K", [(4096, 288, 96), (10000, 96, 96), (3000, 384, 96), (1000, 768, 192), (520, 1536, 384),
                                   (777 * 8, 96, 384), (264, 768, 3072), (1024, 4096, 256), (40, 64, 32), (100000, 96, 288)])
def test_wgrad_split_k(T, N, K, tile):
    """dw[N,K] = dy[T,N]^T @ x[T,K] in fp32, both operands MN-major, deterministic split-K fold."""
    from esvit_b200 import ops
    torch.manual_seed(T + N + K)
    d = torch.device("cuda:0")
    dy = (torch.randn(T, N, device=d) * 0.5).to(BF16)
    x = (torch.randn(T, K, device=d) * 0.5).to(BF16)
    ref = (dy.double().t() @ x.double()).float()
    dw = ops.gemm_wgrad(dy, x, tile=tile)
    assert dw.dtype == torch.float32 and dw.shape == (N, K)
    assert_close(dw, ref, 1e-4, "wgrad")
    dw2 = ops.gemm_wgrad(dy, x, tile=tile)
    assert torch.equal(dw, dw2), "split-K fold must be bit-reproducible"
    acc = torch.ones(N, K, device=d)
    ops.gemm_wgrad(dy, x, out=acc, accumulate=True, tile=tile)
    assert_close(acc, ref + 1, 1e-4, "wgrad accumulate")


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("b_mn", [False, True])
@pytest.mark.parametrize("M,K,N", [(4096, 96, 384), (1000, 192, 768), (300, 384, 1536), (256, 768, 3072), (777, 64, 96),
                                   (33, 96, 288), (20000, 96, 384), (40000, 128, 512)])
def test_mul_colsum(M, K, N, b_mn, tile):
    """out = (a @ w^T) * mult, colsum += column sums (fc2 dgrad fused with the GELU backward), bit-reproducible."""
    from esvit_b200 import ops
    torch.manual_seed(M + K + N + 1)
    d = torch.device("cuda:0")
    a = (torch.randn(M, K, device=d) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=d) / K ** 0.5).to(BF16)   # GEMM B operand [N, K]; the Linear weight W2 is its transpose
    mult = torch.rand(M, N, device=d).to(BF16)
    ref = (a.float() @ w.float().t()) * mult.float()
    colsum = torch.full((N,), 0.5, device=d)
    bop = w.t().contiguous() if b_mn else w
    out = ops.gemm_mul_colsum(a, bop, mult, colsum, b_mn=b_mn, tile=tile)
    assert_close(out, ref, 5e-3, "out")
    assert_close(colsum, out.float().sum(0) + 0.5, 2e-4, "colsum of the bf16 output")
    colsum2 = torch.full((N,), 0.5, device=d)
    out2 = ops.gemm_mul_colsum(a, bop, mult, colsum2, b_mn=b_mn, tile=tile)
    assert torch.equal(out2, out) and torch.equal(colsum2, colsum), "column sums must be bit-reproducible"

