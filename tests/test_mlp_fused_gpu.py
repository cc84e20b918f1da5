"""Back-to-back MLP forward (esvit_mlp_fwd, csrc/gemm2_wgmma.cu): y = GELU(x . W1^T + b1) . W2^T + b2 in one kernel.

* At the real Swin-T stage-0 / stage-1 token counts (B = 64, 2 x 224^2 + 8 x 96^2 crops) and at a ragged M, in student
  mode (h and gelu' written) and teacher mode (y only): y, h and gelu' equal the two-launch esvit_gemm_bf16 chain bit for
  bit, and a rerun is bit-identical.
* Rows past M of sentinel-filled outputs come back untouched; unsupported C and misaligned buffers are rejected."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
M_STAGE0 = 64 * 2 * 56 * 56 + 64 * 8 * 24 * 24   # 696 320 student tokens at C = 96
M_STAGE1 = 64 * 2 * 28 * 28 + 64 * 8 * 12 * 12   # 174 080 student tokens at C = 192
SENTINEL = -1234.0                                 # exactly representable in bf16


def _dev():
    return torch.device("cuda:0")


def _operands(M, C, seed):
    torch.manual_seed(seed)
    d = _dev()
    x = (torch.randn(M, C, device=d) * 0.5).to(BF16)
    w1 = (torch.randn(4 * C, C, device=d) / C ** 0.5).to(BF16)
    b1 = torch.randn(4 * C, device=d) * 0.2
    w2 = (torch.randn(C, 4 * C, device=d) / (4 * C) ** 0.5).to(BF16)
    b2 = torch.randn(C, device=d) * 0.2
    return x, w1, b1, w2, b2


def _mismatch(a, b):
    return f"max |diff| {(a.float() - b.float()).abs().max().item():.3e}, {(a != b).sum().item()} of {a.numel()} differ"


# M = 77 / 200: fewer rows than one 128-row item (77), or a second item of 72 rows (200)
@pytest.mark.parametrize("M,C", [(M_STAGE0, 96), (M_STAGE1, 192), (1000, 96), (1000, 128), (1000, 192), (77, 128),
                                 (200, 192)])
def test_equals_two_gemm_chain(M, C):
    from esvit_b200 import ops
    x, w1, b1, w2, b2 = _operands(M, C, seed=C + M % 97)
    # student: h and gelu' kept for the backward
    h_ref, g_ref = ops.gemm(x, w1, b1, act=1, want_pre=True)
    y_ref = ops.gemm(h_ref, w2, b2)
    y, h, g = ops.mlp_fwd(x, w1, b1, w2, b2, want_h=True)
    assert torch.equal(h, h_ref), _mismatch(h, h_ref)
    assert torch.equal(g, g_ref), _mismatch(g, g_ref)
    assert torch.equal(y, y_ref), _mismatch(y, y_ref)
    y2, h2, g2 = ops.mlp_fwd(x, w1, b1, w2, b2, want_h=True)
    assert torch.equal(y2, y) and torch.equal(h2, h) and torch.equal(g2, g)
    # teacher: no gradient, y only
    del h, g, h2, g2, y2, g_ref
    yt = ops.mlp_fwd(x, w1, b1, w2, b2)
    assert torch.equal(yt, y_ref), _mismatch(yt, y_ref)
    assert torch.equal(ops.mlp_fwd(x, w1, b1, w2, b2), yt)
    torch.cuda.synchronize()


def test_no_bias_equals_chain():
    from esvit_b200 import ops
    x, w1, _, w2, _ = _operands(777, 96, seed=5)
    h_ref = ops.gemm(x, w1, None, act=1)
    assert torch.equal(ops.mlp_fwd(x, w1, None, w2, None), ops.gemm(h_ref, w2, None))


def _call(x, w1, b1, w2, b2, y, h, g, M, C, stream=None):
    from esvit_b200 import _lib, ops
    p = ops._p
    _lib.call("esvit_mlp_fwd", p(x), p(w1), p(b1), p(w2), p(b2), y, h, g, M, C,
              stream if stream is not None else ops._stream())


@pytest.mark.parametrize("C", [96, 192])
def test_rows_past_m_untouched(C):
    from esvit_b200 import ops
    M, pad = 1000, 136   # the last 128-row item is ragged; the padding spans more than one item
    x, w1, b1, w2, b2 = _operands(M, C, seed=11)
    y = torch.full((M + pad, C), SENTINEL, dtype=BF16, device=_dev())
    h = torch.full((M + pad, 4 * C), SENTINEL, dtype=BF16, device=_dev())
    g = torch.full((M + pad, 4 * C), SENTINEL, dtype=BF16, device=_dev())
    _call(x, w1, b1, w2, b2, ops._p(y), ops._p(h), ops._p(g), M, C)
    y_ref, h_ref, g_ref = ops.mlp_fwd(x, w1, b1, w2, b2, want_h=True)
    for out, ref in ((y, y_ref), (h, h_ref), (g, g_ref)):
        assert torch.equal(out[:M], ref)
        assert bool((out[M:] == SENTINEL).all())
    yt = torch.full((M + pad, C), SENTINEL, dtype=BF16, device=_dev())
    _call(x, w1, b1, w2, b2, ops._p(yt), None, None, M, C)
    assert torch.equal(yt[:M], y_ref) and bool((yt[M:] == SENTINEL).all())


@pytest.mark.parametrize("C", [32, 64, 160, 256, 384])
def test_unsupported_width_rejected(C):
    from esvit_b200 import ops
    x, w1, b1, w2, b2 = _operands(256, C, seed=2)
    y = torch.empty(256, C, dtype=BF16, device=_dev())
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, ops._p(y), None, None, 256, C)


def test_bad_arguments_rejected():
    from esvit_b200 import ops
    M, C = 256, 96
    x, w1, b1, w2, b2 = _operands(M, C, seed=3)
    buf = torch.empty(M * C + 8, dtype=BF16, device=_dev())
    hb = torch.empty(M * 4 * C + 8, dtype=BF16, device=_dev())
    ok = ops._p(buf)
    off = ctypes.c_void_p(buf.data_ptr() + 2)        # 2-byte offset: not 16-byte aligned
    h_ok, h_off = ops._p(hb), ctypes.c_void_p(hb.data_ptr() + 2)
    g = torch.empty(M, 4 * C, dtype=BF16, device=_dev())
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, off, None, None, M, C)                 # misaligned y
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, ok, h_off, ops._p(g), M, C)            # misaligned h
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, ok, h_ok, None, M, C)                  # h without gelu'
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, ok, None, ops._p(g), M, C)             # gelu' without h
    with pytest.raises(ValueError):
        _call(x, w1, b1, w2, b2, ok, None, None, 0, C)                  # empty M
    torch.cuda.synchronize()


def test_mlp_fn_dispatch_matches_chain():
    """linear.MlpFn takes the fused kernel at C = 96 and keeps the two-GEMM path at C = 384; both give the same forward
    output and gradients as the explicit chain"""
    from esvit_b200 import linear, ops
    for C in (96, 384):
        x, w1, b1, w2, b2 = _operands(600, C, seed=C)
        w1p = w1.float().requires_grad_(True)
        w2p = w2.float().requires_grad_(True)
        b1p = b1.clone().requires_grad_(True)
        xg = x.clone().requires_grad_(True)
        y = linear.MlpFn.apply(xg, w1p, w1, b1p, w2p, w2, b2)
        y_ref = ops.gemm(ops.gemm(x, w1, b1, act=1), w2, b2)
        assert torch.equal(y, y_ref), (C, _mismatch(y, y_ref))
        with torch.no_grad():
            assert torch.equal(linear.MlpFn.apply(x, w1p, w1, b1p, w2p, w2, b2), y_ref)
        y.float().square().sum().backward()
        assert xg.grad is not None and torch.isfinite(xg.grad.float()).all()
        assert w1p.grad is not None and w2p.grad is not None and b1p.grad is not None
