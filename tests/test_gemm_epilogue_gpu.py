"""bf16 GEMM epilogues (csrc/gemm2_wgmma.cu) staged through shared memory and written by TMA tile stores.

* Real Swin-T stage-0 shapes (M = 696 320 tokens: ~80 work items per CTA at 128 x 256), so that every staging buffer
  and every multiplier buffer is reused many times by the same CTA: checked against fp32 torch on a row sample and
  run twice for bit-identical results.
* Clipping: ragged M and narrow / ragged N for every tile shape, the output written into the head of a larger
  sentinel-filled buffer whose rows past M must come back untouched."""
import pytest
import torch
import torch.nn.functional as F

from helpers import assert_close

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
TILES = [1128, 1256, 2128, 2256]  # consumer warpgroups * 1000 + BN
M_STAGE0 = 64 * 2 * 56 * 56 + 64 * 8 * 24 * 24  # student tokens of stage 0: B = 64, 2 x 224^2 + 8 x 96^2 crops
SENTINEL = -1234.0                                # exactly representable in bf16


def _dev():
    return torch.device("cuda:0")


def _rows(M, seed=0):
    """a seeded sample of rows that still touches every 128-row tile, plus the last row"""
    g = torch.Generator().manual_seed(seed)
    idx = torch.arange(0, M, 128) + torch.randint(0, 128, (M // 128 + 1,), generator=g)[: (M + 127) // 128]
    idx = torch.cat([idx.clamp_max(M - 1), torch.tensor([M - 1])])
    return idx.to(_dev())


def test_stage0_fc1_gelu_many_items_per_cta():
    from esvit_b200 import ops
    M, K, N = M_STAGE0, 96, 384
    torch.manual_seed(1)
    a = (torch.randn(M, K, device=_dev()) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=_dev()) / K ** 0.5).to(BF16)
    b = torch.randn(N, device=_dev()) * 0.2
    h, gp = ops.gemm(a, w, b, act=1, want_pre=True)
    idx = _rows(M)
    pre = (a[idx].float() @ w.float().t() + b).requires_grad_(True)
    F.gelu(pre).sum().backward()
    assert_close(h[idx], F.gelu(pre.detach()), 5e-3, "gelu")
    assert_close(gp[idx], pre.grad, 5e-3, "gelu'")
    h2, gp2 = ops.gemm(a, w, b, act=1, want_pre=True)
    assert torch.equal(h2, h) and torch.equal(gp2, gp)


def test_stage0_qkv_many_items_per_cta():
    from esvit_b200 import ops
    M, K, N = M_STAGE0, 96, 288   # tiles as 256 + 32 columns
    torch.manual_seed(2)
    a = (torch.randn(M, K, device=_dev()) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=_dev()) / K ** 0.5).to(BF16)
    b = torch.randn(N, device=_dev()) * 0.2
    out = ops.gemm(a, w, b)
    idx = _rows(M, 1)
    assert_close(out[idx], a[idx].float() @ w.float().t() + b, 5e-3, "qkv")
    assert torch.equal(ops.gemm(a, w, b), out)


def test_stage0_fc2_dgrad_gelu_colsum_many_items_per_cta():
    """d(pre-activation) = (dy @ W2) * gelu' with the fc1 bias gradient as column sums; W2 read as it lies"""
    from esvit_b200 import ops
    M, C, H = M_STAGE0, 96, 384
    torch.manual_seed(3)
    dy = (torch.randn(M, C, device=_dev()) * 0.5).to(BF16)
    w2 = (torch.randn(C, H, device=_dev()) / C ** 0.5).to(BF16)   # nn.Linear(H, C).weight
    mult = torch.rand(M, H, device=_dev()).to(BF16)
    colsum = torch.full((H,), 0.5, device=_dev())
    out = ops.gemm_mul_colsum(dy, w2, mult, colsum, b_mn=True)
    idx = _rows(M, 2)
    assert_close(out[idx], (dy[idx].float() @ w2.float()) * mult[idx].float(), 5e-3, "out")
    assert_close(colsum, out.float().sum(0) + 0.5, 2e-4, "colsum of the bf16 output")
    colsum2 = torch.full((H,), 0.5, device=_dev())
    out2 = ops.gemm_mul_colsum(dy, w2, mult, colsum2, b_mn=True)
    assert torch.equal(out2, out) and torch.equal(colsum2, colsum), "column sums must be bit-reproducible"


def test_stage0_fc1_input_gradient_mn_major_b():
    from esvit_b200 import ops
    M, H, C = M_STAGE0, 384, 96
    torch.manual_seed(4)
    dh = (torch.randn(M, H, device=_dev()) * 0.5).to(BF16)
    w1 = (torch.randn(H, C, device=_dev()) / H ** 0.5).to(BF16)   # nn.Linear(C, H).weight
    dx = ops.gemm(dh, w1, None, b_mn=True)
    idx = _rows(M, 3)
    assert_close(dx[idx], dh[idx].float() @ w1.float(), 5e-3, "dgrad")
    assert torch.equal(ops.gemm(dh, w1, None, b_mn=True), dx)


def _sentinel(rows, N):
    return torch.full((rows, N), SENTINEL, device=_dev(), dtype=BF16)


@pytest.mark.parametrize("tile", TILES)
@pytest.mark.parametrize("N", [16, 96, 288])
@pytest.mark.parametrize("M", [1037, 1100, 77])
def test_tma_store_clips_rows_and_columns(M, N, tile):
    """bias, GELU (+ gelu') and multiplier epilogues write exactly [M, N]: rows past M of the buffer stay untouched"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    K, pad = 96, 192
    torch.manual_seed(M + N + tile)
    a = (torch.randn(M, K, device=_dev()) * 0.5).to(BF16)
    w = (torch.randn(N, K, device=_dev()) / K ** 0.5).to(BF16)
    b = torch.randn(N, device=_dev()) * 0.2
    ref = a.float() @ w.float().t() + b

    out_buf, pre_buf = _sentinel(M + pad, N), _sentinel(M + pad, N)
    _lib.call("esvit_gemm_bf16", _p(a), _p(w), _p(b), _p(out_buf), None, M, N, K, 0, 0, 0, tile, _stream())
    assert_close(out_buf[:M], ref, 5e-3, "bias")
    assert (out_buf[M:] == SENTINEL).all(), "bias epilogue wrote past row M"

    out_buf.fill_(SENTINEL)
    _lib.call("esvit_gemm_bf16", _p(a), _p(w), _p(b), _p(out_buf), _p(pre_buf), M, N, K, 0, 0, 1, tile, _stream())
    xr = ref.clone().requires_grad_(True)
    F.gelu(xr).sum().backward()
    assert_close(out_buf[:M], F.gelu(ref), 5e-3, "gelu")
    assert_close(pre_buf[:M], xr.grad, 5e-3, "gelu'")
    assert (out_buf[M:] == SENTINEL).all() and (pre_buf[M:] == SENTINEL).all(), "GELU epilogue wrote past row M"

    mult = torch.rand(M, N, device=_dev()).to(BF16)
    out_buf.fill_(SENTINEL)
    colsum = torch.zeros(N, device=_dev())
    ws = torch.empty(160 * N, device=_dev())
    _lib.call("esvit_gemm_mul_colsum2", _p(a), _p(w), _p(mult), _p(out_buf), _p(colsum), _p(ws), M, N, K, 0, tile,
              _stream())
    assert_close(out_buf[:M], (ref - b) * mult.float(), 5e-3, "multiplier")
    assert_close(colsum, out_buf[:M].float().sum(0), 2e-4, "colsum")
    assert (out_buf[M:] == SENTINEL).all(), "multiplier epilogue wrote past row M"


def test_misaligned_output_is_rejected():
    """TMA tile stores need 16-byte aligned base addresses: an output that starts 2 bytes into a buffer is refused"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _po, _stream
    M, K, N = 256, 64, 64
    a = torch.randn(M, K, device=_dev()).to(BF16)
    w = torch.randn(N, K, device=_dev()).to(BF16)
    buf = torch.empty(M * N + 8, device=_dev(), dtype=BF16)
    with pytest.raises(ValueError):
        _lib.call("esvit_gemm_bf16", _p(a), _p(w), None, _po(buf, 1), None, M, N, K, 0, 0, 0, 0, _stream())
    mult = torch.rand(M, N, device=_dev()).to(BF16)
    ws = torch.empty(160 * N, device=_dev())
    colsum = torch.zeros(N, device=_dev())
    with pytest.raises(ValueError):
        _lib.call("esvit_gemm_mul_colsum2", _p(a), _p(w), _p(mult), _po(buf, 1), _p(colsum), _p(ws), M, N, K, 0, 0,
                  _stream())
