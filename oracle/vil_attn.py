"""Dense restatement of the Vision Longformer attention with one global token (layers/longformer2d.py
Long2DSCSelfAttention.forward :139-330, exact = 0, rpe, sharew, W = 7) in the layout of esvit_b200.ops.SlidingChunkAttnFn.

Every local query sees the global key and the keys of its mode's neighbour chunks that lie on the unpadded map; the
global query sees all N tokens; one softmax per row.  Written as one masked N x N attention, so it shares no structure
with the chunked kernels it checks.  `python -m oracle.vil_attn` compares it with the unmodified reference module in
fp64 (needs the reference under oracle/_ref/ and `einops`, which the reference imports).
"""
from __future__ import annotations

import random
import sys

import torch

W = 7
NB = 1 + 9 * W * W  # bias columns: the global key, then 9 neighbour chunks of 49 keys


def mode_chunks(mode: int):
    """neighbour chunks j (= 3 (dx + 1) + (dy + 1)) a query chunk sees: slidingchunk_qk :34-76, mask columns :341-350"""
    if mode == -1:
        return (4,)
    if mode == 0:
        return tuple(range(9))
    return (4, mode if mode > 4 else mode - 1)


def dense_index(nx: int, ny: int, mode: int, device="cpu") -> torch.Tensor:
    """[nx*ny, N] int64: for local query token i (row 1 + i) the flat index into one head's [49, NB] bias of every key it
    attends to (column 0 = the global token), -1 where the reference's zero mask puts -inf or the mode skips the chunk"""
    n = nx * ny
    X = torch.arange(nx, device=device).repeat_interleave(ny)
    Y = torch.arange(ny, device=device).repeat(nx)
    l = (X % W) * W + Y % W
    idx = torch.full((n, 1 + n), -1, dtype=torch.long, device=device)
    idx[:, 0] = l * NB
    r = torch.arange(W * W, device=device)
    qi = torch.arange(n, device=device)[:, None].expand(n, W * W)
    for j in mode_chunks(mode):
        Xk = (X // W + j // 3 - 1)[:, None] * W + (r // W)[None]
        Yk = (Y // W + j % 3 - 1)[:, None] * W + (r % W)[None]
        ok = (Xk >= 0) & (Xk < nx) & (Yk >= 0) & (Yk < ny)
        val = (l[:, None] * NB + 1 + j * W * W + r[None]).expand(n, W * W)
        idx[qi[ok], (1 + Xk * ny + Yk)[ok]] = val[ok]
    return idx


def dense_attention(q, kv, bias, bias_g, idx, B: int, N: int, nH: int, scale: float):
    """softmax(scale q k^T + [bias_g ; local bias, -inf off the chunk neighbourhood]) v -> [B*N, C] (q [B*N, C], kv
    [B*N, 2C] as [k|v], bias [nH, 49, NB], bias_g [nH, N])"""
    C = 32 * nH
    qh = q.view(B, N, nH, 32).transpose(1, 2)
    kh = kv[:, :C].reshape(B, N, nH, 32).transpose(1, 2)
    vh = kv[:, C:].reshape(B, N, nH, 32).transpose(1, 2)
    loc = bias.reshape(nH, -1)[:, idx.clamp_min(0)]
    loc = loc.masked_fill((idx < 0)[None], float("-inf"))
    s = scale * qh @ kh.transpose(-1, -2) + torch.cat([bias_g[:, None, :], loc], 1)[None]
    return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B * N, C)


def module_biases(m, N: int):
    """(bias [nH, 49, NB], bias_g [nH, N]) of a reference Long2DSCSelfAttention (rpe, one global token): the gathers
    of :238-254 and :316-322 with every chunk's columns"""
    nH = m.num_heads
    lb = m.local_relative_position_bias_table[m.relative_position_index.view(-1)].view(W * W, NB - 1, nH)
    bias = torch.cat([m.g2l_relative_position_bias[1][:, :, None].expand(nH, W * W, 1), lb.permute(2, 0, 1)], -1)
    bias_g = torch.cat([m.g2g_relative_position_bias[:, 0, :], m.g2l_relative_position_bias[0].expand(nH, N - 1)], -1)
    return bias, bias_g


def compare_with_reference(cases=((12, 2), (10, 1)), B: int = 2, seed: int = 0):
    """max |dense restatement - reference| of the module output (fp64, after proj) per (side, heads, mode); mode -1 is
    the reference's own-chunk-only setting, modes 1..8 are forced through its random.randrange draw"""
    from oracle import reference_import as RI
    assert RI.available(), f"reference tree not found at {RI.REF_ROOT}"
    RI._install_shims()
    if RI.REF_ROOT not in sys.path:
        sys.path.insert(0, RI.REF_ROOT)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from layers.longformer2d import Long2DSCSelfAttention
    torch.manual_seed(seed)
    out = {}
    for side, nH in cases:
        C, N = 32 * nH, 1 + side * side
        for mode in range(-1, 9):
            m = Long2DSCSelfAttention(C, nH, qkv_bias=True, w=W, sharew=True, nglo=1, exact=0, rpe=True,
                                      mode=1 if mode > 0 else mode).double()
            m.train(mode > 0)
            x = torch.randn(B, N, C, dtype=torch.double)
            draw = random.randrange
            random.randrange = lambda a, b, _m=mode: _m
            try:
                with warnings.catch_warnings(), torch.no_grad():
                    warnings.simplefilter("ignore")
                    ref = m(x, side, side)
            finally:
                random.randrange = draw
            with torch.no_grad():
                q, kv = m.query(x).reshape(B * N, C), m.kv(x).reshape(B * N, 2 * C)
                bias, bias_g = module_biases(m, N)
                ctx = dense_attention(q, kv, bias, bias_g, dense_index(side, side, mode), B, N, nH, m.scale)
                mine = m.proj(ctx.view(B, N, C))
            out[(side, nH, mode)] = float((mine - ref).abs().max())
    return out


if __name__ == "__main__":
    for k, v in compare_with_reference().items():
        print(k, f"{v:.3e}")
