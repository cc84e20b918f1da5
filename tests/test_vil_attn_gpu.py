"""GPU: the Vision Longformer sliding-chunk attention with a global token (ops.SlidingChunkAttnFn, csrc/vil_attn.cu)
against the dense fp64 restatement of layers/longformer2d.py Long2DSCSelfAttention.forward in oracle/vil_attn.py.
Forward, dq / dkv and both bias gradients at every sliding-chunk geometry of vil_2262 (224^2 and 96^2 crops, stages
1-2) in modes -1, 0 and 1..8, batches whose dq segments hold several images, bit-identical reruns, out-of-range modes,
and a CUDA graph that follows the mode written before each replay."""
import pytest
import torch

from helpers import TOL_BF16_ACT, TOL_BF16_GRAD, assert_close
from oracle import vil_attn as O

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16
W, NB = O.W, O.NB
# (map side, heads) of the sliding-chunk stages of vil_2262: stage 1 / 2 at 224^2, then at 96^2
GEOS = [(56, 3), (28, 6), (24, 3), (12, 6)]
CASES = [(s, h, m) for s, h in GEOS for m in range(-1, 9)]


def _inputs(side, nH, B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, C = 1 + side * side, 32 * nH
    q = torch.randn(B * N, C, generator=g, device="cuda").to(BF16)
    kv = torch.randn(B * N, 2 * C, generator=g, device="cuda").to(BF16)
    bias = torch.randn(nH, W * W, NB, generator=g, device="cuda") * 0.5
    bias_g = torch.randn(nH, N, generator=g, device="cuda") * 0.5
    dout = torch.randn(B * N, C, generator=g, device="cuda").to(BF16)
    return q, kv, bias, bias_g, dout


def _run(q, kv, bias, bias_g, mode_t, dout, B, side, nH, scale):
    from esvit_b200 import ops
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, kv, bias, bias_g)]
    out = ops.SlidingChunkAttnFn.apply(*leaves, mode_t, B, side, side, nH, scale)
    grads = torch.autograd.grad(out, leaves, dout)
    return (out.detach(),) + tuple(grads)


def _check(side, nH, mode, B, seed):
    N = 1 + side * side
    scale = 32 ** -0.5
    q, kv, bias, bias_g, dout = _inputs(side, nH, B, seed)
    mode_t = torch.tensor([mode], dtype=torch.int32, device="cuda")
    got = _run(q, kv, bias, bias_g, mode_t, dout, B, side, nH, scale)

    idx = O.dense_index(side, side, mode, "cuda")
    leaves = [t.detach().double().requires_grad_(True) for t in (q, kv, bias, bias_g)]
    want = O.dense_attention(*leaves, idx, B, N, nH, scale)
    wgrads = torch.autograd.grad(want, leaves, dout.double())
    assert_close(got[0], want, TOL_BF16_ACT, "out")
    for name, a, b in zip(("dq", "dkv", "dbias", "dbias_g"), got[1:], wgrads):
        assert_close(a, b, TOL_BF16_GRAD, name)
    keep = torch.zeros(NB, dtype=torch.bool, device="cuda")  # columns of the chunks the mode skips get no gradient
    keep[0] = True
    for j in O.mode_chunks(mode):
        keep[1 + j * W * W: 1 + (j + 1) * W * W] = True
    assert torch.all(got[3][:, :, ~keep] == 0)

    again = _run(q, kv, bias, bias_g, mode_t, dout, B, side, nH, scale)
    for a, b in zip(got, again):
        assert torch.equal(a, b), "reruns must be bit-identical"


@pytest.mark.parametrize("side,nH,mode", CASES)
def test_sliding_chunk_against_fp64(side, nH, mode):
    _check(side, nH, mode, B=2, seed=10 * side + mode + 1)


# batches for which the dq kernel's image segments hold several images (3 per segment at 56^2 / 3 heads, B = 6; 3 at
# 12^2 / 6 heads, B = 24), so the per-image loop and the bias sum across images run as at training batch sizes
@pytest.mark.parametrize("side,nH,B,mode", [(56, 3, 6, 0), (56, 3, 6, 3), (12, 6, 24, 0), (12, 6, 24, 6)])
def test_sliding_chunk_multi_image_segments(side, nH, B, mode):
    _check(side, nH, mode, B=B, seed=100 + mode)


def test_sliding_chunk_out_of_range_mode_is_clamped():
    side, nH, B = 12, 6, 2
    q, kv, bias, bias_g, dout = _inputs(side, nH, B, seed=7)

    def run(mode):
        return _run(q, kv, bias, bias_g, torch.tensor([mode], dtype=torch.int32, device="cuda"), dout, B, side, nH,
                    32 ** -0.5)

    for bad, clamped in ((9, 8), (1000, 8), (-2, -1), (-1000, -1)):
        for a, b in zip(run(bad), run(clamped)):
            assert torch.equal(a, b), f"mode {bad}"


def test_sliding_chunk_graph_follows_mode():
    """one captured forward + backward, replayed after writing modes 3, 0 and 7, equals eager calls in each mode"""
    from esvit_b200 import ops
    side, nH, B = 24, 3, 4
    scale = 32 ** -0.5
    q, kv, bias, bias_g, dout = _inputs(side, nH, B, seed=5)
    mode_t = torch.tensor([1], dtype=torch.int32, device="cuda")
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, kv, bias, bias_g)]

    def step():
        out = ops.SlidingChunkAttnFn.apply(*leaves, mode_t, B, side, side, nH, scale)
        return (out,) + tuple(torch.autograd.grad(out, leaves, dout))

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for mode in (3, 0, 7):
        mode_t.fill_(mode)
        graph.replay()
        eager = _run(q, kv, bias, bias_g, torch.tensor([mode], dtype=torch.int32, device="cuda"), dout, B, side, nH,
                     scale)
        for a, b in zip(static, eager):
            assert torch.equal(a.detach(), b), f"mode {mode}"


def test_sliding_chunk_rejects_bad_shapes():
    from esvit_b200 import ops
    q, kv, bias, bias_g, _ = _inputs(12, 6, 1, seed=0)
    mode_t = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError):
        ops.SlidingChunkAttnFn.apply(q, kv, bias, bias_g, mode_t, 1, 12, 11, 6, 1.0)
    with pytest.raises(ValueError):
        ops.SlidingChunkAttnFn.apply(q, kv, bias[:, :, :-1], bias_g, mode_t, 1, 12, 12, 6, 1.0)
