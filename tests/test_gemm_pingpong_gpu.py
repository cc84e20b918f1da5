"""Ping-pong schedule of the 64-row GEMM tiles (tile codes 1128 / 1256, csrc/gemm2_wgmma.cu): two consumer warpgroups
take a CTA's items alternately and share one operand ring.

Every output element keeps its k16 accumulation order, so the bf16 results must equal the cooperative kernel's
(2128 / 2256) bit for bit for every epilogue and operand major, at ragged M / N / K, and at item counts below, equal to
and just above the grid, and odd (one warpgroup with one item more than the other, or none at all).  Column sums and
fp32 weight gradients are bit-identical run to run and equal to the cooperative result up to fp32 re-association.
Outputs are written into sentinel-filled buffers taller than M: rows past M must come back untouched (a write past
column N would land in the next row and break the equality)."""
import pytest
import torch

from helpers import assert_close

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
SENTINEL = -1234.0   # exactly representable in bf16
PAD = 70             # rows of sentinel past M
PAIRS = [(1128, 2128), (1256, 2256)]   # (ping-pong, cooperative) of one BN


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bf16_call(a, b, bias, M, N, K, a_mn, b_mn, act, want_pre, tile):
    """esvit_gemm_bf16 into sentinel buffers; returns (out, pre) cut to [M, N] after checking the rows past M"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    out = torch.full((M + PAD, N), SENTINEL, device=_dev(), dtype=BF16)
    pre = torch.full((M + PAD, N), SENTINEL, device=_dev(), dtype=BF16) if want_pre else None
    _lib.call("esvit_gemm_bf16", _p(a), _p(b), _p(bias), _p(out), _p(pre), M, N, K, a_mn, b_mn, act, tile, _stream())
    assert (out[M:] == SENTINEL).all(), f"tile {tile} wrote past row M"
    if pre is not None:
        assert (pre[M:] == SENTINEL).all(), f"tile {tile} wrote gelu' past row M"
        pre = pre[:M]
    return out[:M], pre


def _mul_call(a, b, mult, M, N, K, b_mn, tile):
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    out = torch.full((M + PAD, N), SENTINEL, device=_dev(), dtype=BF16)
    colsum = torch.zeros(N, device=_dev())
    ws = torch.empty(160 * N, device=_dev())
    _lib.call("esvit_gemm_mul_colsum2", _p(a), _p(b), _p(mult), _p(out), _p(colsum), _p(ws), M, N, K, b_mn, tile,
              _stream())
    assert (out[M:] == SENTINEL).all(), f"tile {tile} wrote past row M"
    return out[:M], colsum


def _operands(M, N, K, a_mn, b_mn, seed):
    torch.manual_seed(seed)
    a = (torch.randn(K, M, device=_dev()) if a_mn else torch.randn(M, K, device=_dev())) * 0.5
    b = (torch.randn(K, N, device=_dev()) if b_mn else torch.randn(N, K, device=_dev())) / K ** 0.5
    return a.to(BF16), b.to(BF16)


def _check_bf16(M, N, K, a_mn, b_mn, seed):
    a, b = _operands(M, N, K, a_mn, b_mn, seed)
    bias = torch.randn(N, device=_dev()) * 0.2
    for pp, coop in PAIRS:
        for act, want_pre, bb in ((0, False, bias), (0, False, None), (1, True, bias), (1, False, bias), (2, True, bias)):
            if act == 2 and (a_mn or b_mn):
                continue   # QuickGELU: K-major operands only
            out, pre = _bf16_call(a, b, bb, M, N, K, a_mn, b_mn, act, want_pre, pp)
            ref, ref_pre = _bf16_call(a, b, bb, M, N, K, a_mn, b_mn, act, want_pre, coop)
            assert torch.equal(out, ref), (pp, act, want_pre, bb is None)
            if want_pre:
                assert torch.equal(pre, ref_pre), (pp, act, "gelu'")
        # and against fp32 torch, so that agreeing with the cooperative kernel means something
        fa = a.float().t() if a_mn else a.float()
        fb = b.float() if b_mn else b.float().t()
        out, _ = _bf16_call(a, b, bias, M, N, K, a_mn, b_mn, 0, False, pp)
        assert_close(out, fa @ fb + bias, 5e-3, f"bias epilogue at {pp}")


def _check_mul(M, N, K, b_mn, seed):
    a, b = _operands(M, N, K, 0, b_mn, seed)
    mult = torch.rand(M, N, device=_dev()).to(BF16)
    for pp, coop in PAIRS:
        out, cs = _mul_call(a, b, mult, M, N, K, b_mn, pp)
        ref, ref_cs = _mul_call(a, b, mult, M, N, K, b_mn, coop)
        assert torch.equal(out, ref), pp
        out2, cs2 = _mul_call(a, b, mult, M, N, K, b_mn, pp)
        assert torch.equal(out2, out) and torch.equal(cs2, cs), f"column sums at {pp} must be bit-reproducible"
        assert_close(cs, ref_cs, 1e-5, f"column sums at {pp} against {coop}")
        assert_close(cs, out.double().sum(0), 1e-5, f"column sums at {pp} of the stored bf16 output")


def _check_wgrad(T, N, K, splits, seed):
    from esvit_b200 import ops
    torch.manual_seed(seed)
    dy = (torch.randn(T, N, device=_dev()) * 0.5).to(BF16)
    x = (torch.randn(T, K, device=_dev()) * 0.5).to(BF16)
    for pp, coop in PAIRS:
        dw = ops.gemm_wgrad(dy, x, tile=splits * 10000 + pp)
        assert torch.equal(ops.gemm_wgrad(dy, x, tile=splits * 10000 + pp), dw), f"wgrad at {pp} must be bit-reproducible"
        assert_close(dw, ops.gemm_wgrad(dy, x, tile=splits * 10000 + coop), 1e-5, f"wgrad at {pp} against {coop}")
        assert_close(dw, (dy.double().t() @ x.double()).float(), 1e-4, f"wgrad at {pp}")


@pytest.mark.parametrize("b_mn", [0, 1])
@pytest.mark.parametrize("a_mn", [0, 1])
@pytest.mark.parametrize("M,N,K", [(1037, 96, 104), (2000, 288, 96), (300, 520, 200), (64, 128, 40), (777, 384, 776)])
def test_bf16_epilogues_match_cooperative(M, N, K, a_mn, b_mn):
    if a_mn:
        M -= M % 8   # an MN-major A needs M % 8 == 0 (its rows are the TMA's contiguous dimension)
    _check_bf16(M, N, K, a_mn, b_mn, M + N + K + 2 * a_mn + b_mn)


@pytest.mark.parametrize("b_mn", [0, 1])
@pytest.mark.parametrize("M,N,K", [(1037, 96, 104), (2000, 288, 96), (300, 520, 200), (777, 384, 776)])
def test_multiplier_colsum_matches_cooperative(M, N, K, b_mn):
    _check_mul(M, N, K, b_mn, M + N + K + b_mn)


@pytest.mark.parametrize("T,N,K,splits", [(4096, 96, 104, 3), (3000, 200, 96, 1), (20000, 64, 288, 7), (777 * 8, 136, 384, 0)])
def test_wgrad_split_k_matches_cooperative(T, N, K, splits):
    _check_wgrad(T, N, K, splits, T + N + K)


# items = (64-row tiles) x (BN-column tiles) relative to the grid (one CTA per SM): below, equal, just above, odd counts
# (a CTA with 3 items: warpgroup 0 takes two, warpgroup 1 one) and several rounds per warpgroup
@pytest.mark.parametrize("rel", ["sms-1", "sms", "sms+1", "2sms+1", "3sms", "5sms+3"])
def test_item_counts_around_the_grid(rel):
    sms = _sms()
    items = {"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1, "3sms": 3 * sms,
             "5sms+3": 5 * sms + 3}[rel]
    M = 64 * (items - 1) + 37   # ragged last row tile; N = 128 and 256 are one column tile at 1128 and 1256
    for N in (128, 256):
        _check_bf16(M, N, 96, 0, 0, items + N)
        _check_bf16(M, N, 136, 0, 1, items + N + 1)
        _check_mul(M, N, 192, 1, items + N + 2)
    # weight gradient without split: GEMM M = out features, one column tile of 128 in-features at either BN
    _check_wgrad(512, 64 * (items - 1) + 40, 128, 1, items)


# real shapes of the Swin-T 2 + 8-crop step (B = 64): tokens per stage, stage widths and the DINO head's last layers
T2, T3 = 64 * (2 * 14 * 14 + 8 * 6 * 6), 64 * (2 * 7 * 7 + 8 * 3 * 3)


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(T2, 1152, 384, 0, 0), (T2, 384, 1152, 0, 1), (T3, 768, 3072, 0, 1),
                                             (T3, 2304, 768, 0, 0), (T3, 65536, 256, 0, 0), (640, 256, 65536, 0, 1)])
def test_step_shapes_bf16(M, N, K, a_mn, b_mn):
    _check_bf16(M, N, K, a_mn, b_mn, N + K)


@pytest.mark.parametrize("M,N,K", [(T2, 1536, 384), (T3, 3072, 768), (640, 2048, 2048)])
def test_step_shapes_multiplier(M, N, K):
    _check_mul(M, N, K, 1, N + K)
