"""The Swin window-attention training kernels (esvit_window_attn_fwd / _bwd, csrc/window_attn7.cuh and window_attn14.cuh)
against an fp64 reference of their C-ABI contract, at every geometry the Swin-T W7 / Swin-S W14 / Swin-B W14 steps and
evaluation launch, plus the contract itself: fully written outputs, accumulated gradients, the pre-expanded ws-7 bias,
the persistent-loop grid, reproducibility, resolution groups and argument rejection.

The reference (CPU tests, not `gpu`-marked) is pinned to the oracle's attention path of `oracle.swin.swin_block`, and
each plausible kernel bug of a list below is shown to move the reference by at least 5x the gate the GPU test uses."""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from helpers import rel
from oracle import swin as S

HD = 32
LOG2E = 1.4426950408889634

# Gates (rel-L2 unless noted), at about 3x the largest error measured on an H100 over every case below and never looser
# than the starting gates of the other attention kernels (DESIGN.md §4.6).  Measured maxima: DESIGN.md §4.3.
#   out / out_win: global / largest per-(window, head) rel-L2 of the output over real tokens
#   lse: max |lse - lse_ref| over real-token query slots (natural log)
#   dqkv / dqkv_win: global / largest per-(window, q|k|v, head) rel-L2 of dqkv over real tokens
#   dtable / dbias: the rel-pos-table and the complete qkv-bias gradient
#   large logits replace dqkv_win by dv_win (v only, against exact fp64) and dqk_win_D: dq / dk per (window, head)
#     against fp64 gradients that take D = rowsum(dO * O) from the kernel's bf16 O, as the kernels do (dqk_win_bf16_o_D)
GATES = {
    "normal": dict(out=7e-3, out_win=9e-3, lse=4e-6, dqkv=1.2e-2, dqkv_win=2e-2, dtable=7e-3, dbias=6e-3),
    "large": dict(out=3e-3, out_win=5e-3, lse=1.3e-4, dqkv=2e-2, dv_win=6e-3, dqk_win_D=1.5e-2, dtable=2e-2, dbias=2e-2),
}

Case = namedtuple("Case", "C nH H W ws shift B scale large")


def _case(C, H, ws, shift, W=None, B=None, scale=HD ** -0.5, large=False):
    W = H if W is None else W
    if B is None:
        B = 1 if max(H, W) >= 56 else 2
    return Case(C, C // HD, H, W, ws, shift, B, scale, large)


# ---- the geometries of the step and of evaluation ---------------------------------------------------------------------
# ws 7 (Swin-T W7 and the ws-7 stage 3 of the W14 models): maps 56/28/14/7 at 224², 24/12/6/3 at 96²; shift 3 wherever
# the nominal (224²) resolution exceeds 7, so map 6 (nominal 14) is a single padded window that still gets a shift mask
CASES = {}
for C, maps in ((96, (56, 24)), (128, (56, 24)), (192, (28, 12)), (384, (14, 6))):  # 128: the Swin-B W7 width
    for m in maps:
        for s in (0, 3):
            CASES[f"w7_c{C}_m{m}_s{s}"] = _case(C, m, 7, s)
for C in (768, 1024):  # last stage, nominal 7: ws 7 without shift (also the last stage of the W14 models)
    for m in (7, 3):
        CASES[f"w7_c{C}_m{m}_s0"] = _case(C, m, 7, 0)
# ws 14 (Swin-S / Swin-B W14): both shifts at maps 56/24 and 28/12 (map 12: one padded window, shifted); the third
# stage (nominal 14) runs ws 14 without shift at maps 14 and 6
for C, maps in ((96, (56, 24)), (128, (56, 24)), (192, (28, 12)), (256, (28, 12))):
    for m in maps:
        for s in (0, 7):
            CASES[f"w14_c{C}_m{m}_s{s}"] = _case(C, m, 14, s)
for C in (384, 512):
    for m in (14, 6):
        CASES[f"w14_c{C}_m{m}_s0"] = _case(C, m, 14, 0)
# non-square maps (the ABI takes H and W separately; an H / W swap in the slot geometry shows here)
CASES["w7_h24_w28_s3"] = _case(96, 24, 7, 3, W=28)
CASES["w14_h28_w12_s7"] = _case(128, 28, 14, 7, W=12)
# a non-default scale, and large logits (qkv x 8, table entries in [-8, 8]): the -100 mask no longer saturates
CASES["w7_scale0.1"] = _case(96, 24, 7, 3, scale=0.1)
CASES["w14_scale0.1"] = _case(128, 24, 14, 7, scale=0.1)
CASES["w7_large"] = _case(96, 24, 7, 3, large=True)
CASES["w14_large"] = _case(128, 24, 14, 7, large=True)
CASES["w7_large_pad"] = _case(384, 6, 7, 3, large=True)
CASES["w14_large_pad"] = _case(256, 12, 14, 7, large=True)


def _gates(case):
    return GATES["large" if case.large else "normal"]


def _pad(n, ws):
    return -(-n // ws) * ws


def _partition(x, ws):
    """[B, Hp, Wp, D] -> [B * nWy * nWx, ws * ws, D] (window_partition, models/swin_transformer.py:51-62)"""
    B, Hp, Wp, D = x.shape
    return x.view(B, Hp // ws, ws, Wp // ws, ws, D).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, D)


def _reverse(xw, B, Hp, Wp, ws):
    """window_reverse (models/swin_transformer.py:65-78)"""
    D = xw.shape[-1]
    return xw.view(B, Hp // ws, Wp // ws, ws, ws, D).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, D)


def slot_tokens(B, H, W, ws, shift):
    """[B * nW, ws * ws] token row (b * H * W + y * W + x) at every window slot after pad + roll, -1 for padded slots"""
    Hp, Wp = _pad(H, ws), _pad(W, ws)
    t = torch.full((B, Hp, Wp, 1), -1, dtype=torch.long)
    t[:, :H, :W, 0] = torch.arange(B * H * W).view(B, H, W)
    if shift:
        t = torch.roll(t, shifts=(-shift, -shift), dims=(1, 2))
    return _partition(t, ws)[..., 0]


def _mask_regions_from_unpadded(H, W, ws, shift):
    """a wrong shift mask (regions cut at H - ws, H - shift instead of Hp - ws, Hp - shift), for the sensitivity check"""
    Hp, Wp = _pad(H, ws), _pad(W, ws)

    def rid(n, ext):
        p = torch.arange(ext)
        return (p >= n - ws).long() + (p >= n - shift).long()

    reg = rid(H, Hp)[:, None] * 3 + rid(W, Wp)[None, :]
    reg = reg.view(Hp // ws, ws, Wp // ws, ws).permute(0, 2, 1, 3).reshape(-1, ws * ws)
    return (reg[:, None, :] != reg[:, :, None]).float() * -100.0


BUGS = ("bias_transposed", "shift_from_unpadded", "pad_zeros", "no_padded_bias_grad", "mask_inf", "scale_fixed")


def _scores(q, k, table, B, H, W, nH, ws, shift, scale, bug=None):
    """(q * scale) k^T + table[rel_pos_index] (+ the -100 shift mask) of windows q, k [B_, nH, N, 32]"""
    N = ws * ws
    s = (q * (HD ** -0.5 if bug == "scale_fixed" else scale)) @ k.transpose(-2, -1)
    idx = S.rel_pos_index(ws).to(table.device)
    if bug == "bias_transposed":
        idx = idx.t()
    s = s + table[idx.reshape(-1)].view(N, N, nH).permute(2, 0, 1)
    if shift:
        mask = (_mask_regions_from_unpadded if bug == "shift_from_unpadded" else S.shift_mask)(H, W, ws, shift).to(s)
        if bug == "mask_inf":
            mask = mask.masked_fill(mask != 0, -math.inf)
        s = (s.view(B, -1, nH, N, N) + mask[None, :, None]).view(-1, nH, N, N)
    return s


def ref_window_attention(qkv, qkv_bias_bf16, table, B, H, W, nH, ws, shift, scale, bug=None):
    """fp64 (shifted-)window attention of the kernel contract, SwinTransformerBlock.forward / WindowAttention.forward
    (models/swin_transformer.py:283-325, :120-152) on the qkv Linear's output: pad to Hp x Wp with the qkv bias (the
    reference pads the normalised activations with zeros, so a padded slot's q / k / v is the bias), roll by -shift,
    partition, (q * scale) k^T + table[rel_pos_index] + the additive -100 shift mask, softmax, @ v, reverse, roll back,
    crop.  qkv [B, H*W, 3C], qkv_bias_bf16 [3C] (the bf16-rounded bias the kernel gives padded slots), table
    [(2ws-1)^2, nH].  Returns out [B, H*W, C] and the natural-log lse [B*nW, nH, ws*ws].  `bug` selects a perturbed
    variant (BUGS) for the sensitivity check."""
    C = qkv.shape[-1] // 3
    Hp, Wp, N = _pad(H, ws), _pad(W, ws), ws * ws
    fill = torch.zeros_like(qkv_bias_bf16) if bug == "pad_zeros" else qkv_bias_bf16
    x = qkv.reshape(B, H, W, 3 * C)
    x = torch.cat([x, fill.expand(B, H, Wp - W, 3 * C)], 2)
    x = torch.cat([x, fill.expand(B, Hp - H, Wp, 3 * C)], 1)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    q, k, v = _partition(x, ws).view(-1, N, 3, nH, HD).permute(2, 0, 3, 1, 4)  # each [B_, nH, N, 32]
    s = _scores(q, k, table, B, H, W, nH, ws, shift, scale, bug)
    lse = torch.logsumexp(s, -1)
    o = (s.softmax(-1) @ v).transpose(1, 2).reshape(-1, N, C)
    o = _reverse(o, B, Hp, Wp, ws)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    return o[:, :H, :W].reshape(B, H * W, C), lse


def ref_all(inp, case, bug=None):
    """out, lse and, through autograd for inp["dout"], dqkv, dtable and the complete qkv-bias gradient dbias (the
    padded-slot leaf's gradient plus the column sums of the real-token dqkv), all fp64"""
    qkv = inp["qkv"].double().requires_grad_()
    qb = inp["qb"].double().requires_grad_()
    table = inp["table"].double().requires_grad_()
    out, lse = ref_window_attention(qkv, qb, table, case.B, case.H, case.W, case.nH, case.ws, case.shift, case.scale, bug)
    dqkv, dqb_pad, dtable = torch.autograd.grad(out, (qkv, qb, table), inp["dout"].double(), allow_unused=True)
    if dqb_pad is None:
        dqb_pad = torch.zeros_like(qb)
    dbias = dqkv.reshape(-1, dqkv.shape[-1]).sum(0)
    if bug != "no_padded_bias_grad":
        dbias = dbias + dqb_pad
    return dict(out=out.detach(), lse=lse.detach(), dqkv=dqkv, dtable=dtable, dbias=dbias)


def make_inputs(case, seed, device="cpu"):
    """bf16 qkv / dout, the bf16-rounded qkv bias, an fp32 table; drawn on the CPU so every device sees the same values"""
    g = torch.Generator().manual_seed(seed)
    C3 = 3 * case.C
    amp = 8.0 if case.large else 1.0
    qkv = (torch.randn(case.B, case.H * case.W, C3, generator=g) * amp).to(torch.bfloat16)
    qb = (torch.randn(C3, generator=g) * amp).to(torch.bfloat16)
    nb = (2 * case.ws - 1) ** 2
    if case.large:
        table = torch.rand(nb, case.nH, generator=g) * 16 - 8
    else:
        table = torch.randn(nb, case.nH, generator=g)
    dout = torch.randn(case.B, case.H * case.W, case.C, generator=g).to(torch.bfloat16)
    return {k: v.to(device) for k, v in dict(qkv=qkv, qb=qb, table=table, dout=dout).items()}


def _per_window_max(got, ref, tok, groups):
    """largest rel-L2 over (window, group, head) of token-major [T, groups * nH * 32] tensors, real-token slots only"""
    real = (tok >= 0).to(got.device)
    idx = tok.clamp_min(0).to(got.device)

    def win(t):
        t = t.double().reshape(-1, groups, t.shape[-1] // (groups * HD), HD)[idx]  # [nWin, N, groups, nH, 32]
        return t * real[:, :, None, None, None]

    a, b = win(got), win(ref)
    num = (a - b).pow(2).sum((1, 4)).sqrt()
    den = b.pow(2).sum((1, 4)).sqrt().clamp_min(1e-30)
    return float((num / den).max())


def errors(got, ref, case):
    """every metric the GPU test gates (see GATES), of kernel results `got` against the reference `ref`"""
    tok = slot_tokens(case.B, case.H, case.W, case.ws, case.shift)
    real = (tok >= 0)[:, None, :].expand(-1, case.nH, -1).to(got["lse"].device)
    dl = (got["lse"].double().view(real.shape) - ref["lse"].view(real.shape)).abs()
    return dict(
        out=rel(got["out"], ref["out"]),
        out_win=_per_window_max(got["out"].reshape(-1, case.C), ref["out"].reshape(-1, case.C), tok, 1),
        lse=float(dl[real].max()),
        dqkv=rel(got["dqkv"], ref["dqkv"]),
        dqkv_win=_per_window_max(got["dqkv"].reshape(-1, 3 * case.C), ref["dqkv"].reshape(-1, 3 * case.C), tok, 3),
        dtable=rel(got["dtable"], ref["dtable"]),
        dbias=rel(got["dbias"], ref["dbias"]))


def dqk_win_bf16_o_D(got, inp, case):
    """largest per-(window, q|k, head) rel-L2 of the kernel's dq / dk against fp64 gradients whose softmax-backward row
    term D_i = sum_j P_ij dP_ij is taken as rowsum(dO_i * O_i) of the kernel's bf16 output O, as the kernels compute
    it.  With large logits every softmax row of some (window, head) pairs is one-hot to fp64 precision; their dq / dk
    are a cancellation dP_ij - D_i that the rounding of O to bf16 dominates, so this is the comparison that can see a
    kernel bug in those windows."""
    B, H, W, C, nH, ws = case.B, case.H, case.W, case.C, case.nH, case.ws
    Hp, Wp, N = _pad(H, ws), _pad(W, ws), ws * ws
    tok = slot_tokens(B, H, W, ws, case.shift).to(got["out"].device)
    real = (tok >= 0)[:, None, :, None].double()

    def windows(t, fill):  # token-major [B, H*W, D] -> [nWin, N, D] after pad (with `fill`) and roll
        x = fill.double().expand(B, Hp, Wp, t.shape[-1]).clone()
        x[:, :H, :W] = t.double().reshape(B, H, W, -1)
        if case.shift:
            x = torch.roll(x, shifts=(-case.shift, -case.shift), dims=(1, 2))
        return _partition(x, ws)

    zero = torch.zeros(C, device=tok.device)
    q, k, v = windows(inp["qkv"], inp["qb"]).view(-1, N, 3, nH, HD).permute(2, 0, 3, 1, 4)
    dO = windows(inp["dout"], zero).view(-1, N, nH, HD).transpose(1, 2)
    O = windows(got["out"], zero).view(-1, N, nH, HD).transpose(1, 2)
    P = _scores(q, k, inp["table"].double(), B, H, W, nH, ws, case.shift, case.scale).softmax(-1)
    dS = P * (dO @ v.transpose(-2, -1) - (dO * O).sum(-1, keepdim=True))
    want = (dS @ k * case.scale, dS.transpose(-2, -1) @ q * case.scale)
    kern = got["dqkv"].double().reshape(-1, 3, nH, HD)[tok.clamp_min(0)].permute(2, 0, 3, 1, 4)  # [3, nWin, nH, N, 32]
    worst = 0.0
    for a, b in zip(kern[:2], want):
        a, b = a * real, b * real
        # a pair whose gradient is below 1 % of the median pair's is measured against that 1 %: there dP_ij - D_i is
        # below the fp32 rounding of its two terms (measured: 2e-6 of the median at w7_large)
        norm = b.pow(2).sum((2, 3)).sqrt()
        r = (a - b).pow(2).sum((2, 3)).sqrt() / norm.clamp_min(1e-2 * float(norm.median()))
        worst = max(worst, float(r.max()))
    return worst


# ================================ 1. the reference (CPU) ===============================================================
PIN_CASES = [(7, 14, 0), (7, 14, 3), (7, 10, 3), (7, 6, 3), (7, 3, 0), (14, 28, 0), (14, 28, 7), (14, 12, 7),
             (14, 20, 0), (14, 6, 0)]


@pytest.mark.parametrize("ws,side,shift", PIN_CASES)
def test_reference_matches_oracle_attention_path(ws, side, shift):
    """the reference against a float64 run of the pad / roll / partition / oracle.swin.window_attention / reverse / roll /
    crop lines of oracle.swin.swin_block, with a random qkv Linear, an identity proj and random stand-in activations"""
    g = torch.Generator().manual_seed(1000 * ws + 10 * side + shift)
    B, nH = 2, 2
    C = nH * HD
    H = W = side
    dd = dict(dtype=torch.float64)
    y = torch.randn(B, H, W, C, generator=g, **dd).requires_grad_()
    wq = (torch.randn(3 * C, C, generator=g, **dd) * C ** -0.5).requires_grad_()
    bq = torch.randn(3 * C, generator=g, **dd).requires_grad_()
    table = torch.randn((2 * ws - 1) ** 2, nH, generator=g, **dd).requires_grad_()
    sd = {"a.qkv.weight": wq, "a.qkv.bias": bq, "a.relative_position_bias_table": table,
          "a.proj.weight": torch.eye(C, **dd), "a.proj.bias": torch.zeros(C, **dd)}
    dout = torch.randn(B, H * W, C, generator=g, **dd)

    # oracle.swin.swin_block, attention branch
    pad_r, pad_b = (ws - W % ws) % ws, (ws - H % ws) % ws
    yp = F.pad(y, (0, 0, 0, pad_r, 0, pad_b))
    Hp, Wp = H + pad_b, W + pad_r
    mask = None
    if shift > 0:
        yp = torch.roll(yp, shifts=(-shift, -shift), dims=(1, 2))
        mask = S.shift_mask(H, W, ws, shift).to(yp)
    yw = yp.view(B, Hp // ws, ws, Wp // ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, C)
    aw = S.window_attention(yw, sd, "a", nH, ws, mask)
    o = aw.view(B, Hp // ws, Wp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Wp, C)
    if shift > 0:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    o = o[:, :H, :W, :].reshape(B, H * W, C)
    dy, dbq, dtab = torch.autograd.grad(o, (y, bq, table), dout)

    case = Case(C, nH, H, W, ws, shift, B, HD ** -0.5, False)
    inp = dict(qkv=F.linear(y, wq, bq).detach().reshape(B, H * W, 3 * C), qb=bq.detach(), table=table.detach(), dout=dout)
    r = ref_all(inp, case)
    assert rel(r["out"], o) < 1e-12
    assert rel(r["dtable"], dtab) < 1e-12
    # padded y rows are zero, so the oracle's qkv-bias gradient includes the padded slots: the kernel's semantics
    assert rel(r["dbias"], dbq) < 1e-12
    assert rel((r["dqkv"] @ wq.detach()).view(B, H, W, C), dy) < 1e-12
    assert r["lse"].shape == (B * (Hp // ws) * (Wp // ws), nH, ws * ws)
    # the padded slots' share of the bias gradient; at map 10, ws 7, shift 3 the padded band is a shift region of its
    # own, so the -100 mask cuts it off from every real query and the share is e^-100
    share = rel(r["dbias"], r["dqkv"].reshape(-1, 3 * C).sum(0))
    assert share > 1e-3 if (pad_r and (ws, side, shift) != (7, 10, 3)) else share < 1e-30


# each bug must move the reference by >= 5x the gate of the metric named, on the GPU case named
SENSITIVITY = [
    ("bias_transposed", "w7_c96_m24_s3", "out"),
    ("bias_transposed", "w14_c128_m24_s7", "out"),
    ("shift_from_unpadded", "w7_c384_m6_s3", "out_win"),
    ("shift_from_unpadded", "w14_c192_m12_s7", "out_win"),
    ("pad_zeros", "w7_c768_m3_s0", "out"),
    ("pad_zeros", "w14_c384_m6_s0", "out"),
    ("no_padded_bias_grad", "w7_c768_m3_s0", "dbias"),
    ("no_padded_bias_grad", "w7_c384_m6_s3", "dbias"),
    ("no_padded_bias_grad", "w14_c192_m12_s7", "dbias"),
    ("mask_inf", "w7_large", "out_win"),
    ("mask_inf", "w14_large", "out_win"),
    ("scale_fixed", "w7_scale0.1", "out"),
    ("scale_fixed", "w14_scale0.1", "out"),
]


def _seed(name):
    return sum(ord(ch) * 31 ** i for i, ch in enumerate(name)) % (1 << 31)


@pytest.mark.parametrize("bug,name,metric", SENSITIVITY)
def test_gates_see_plausible_kernel_bugs(bug, name, metric):
    case = CASES[name]
    inp = make_inputs(case, _seed(name))
    good = ref_all(inp, case)
    bad = ref_all(inp, case, bug)
    assert all(torch.isfinite(t).all() for t in bad.values())
    err = errors(bad, good, case)[metric]
    gate = _gates(case)[metric]
    print(f"sensitivity {bug} on {name}: {metric} {err:.3e} = {err / gate:.1f}x gate")
    assert err >= 5 * gate, (bug, name, metric, err, gate)


def test_geometry_covers_every_launch_of_the_swin_models():
    """each (width, map, ws, shift) that a Swin-T W7 / Swin-S W14 / Swin-B W14 block launches on 224² and 96² crops is
    a kernel case"""
    have = {(c.C, c.H, c.ws, c.shift) for c in CASES.values() if c.H == c.W and not c.large and c.scale == HD ** -0.5}
    for spec in (S.SWIN_T_W7, S.SWIN_S_W14, S.SWIN_B_W14):
        sp = S.SwinSpec(img_size=224, **spec)
        for i in range(len(sp.depths)):
            for j in range(min(2, sp.depths[i])):
                ws, shift = sp.block_window_shift(i, j)
                for m in (sp.stage_resolution(i), 96 // sp.patch_size // 2 ** i):
                    key = (sp.embed_dim * 2 ** i, m, ws, shift)
                    assert key in have, f"no kernel case for C={key[0]} map={m} ws={ws} shift={shift}"


# ================================ 2. kernel vs reference (GPU) =========================================================
def _run_kernel(inp, case, *, bias_ws=None, ready=0, nan_fill=False, acc=0.0):
    """esvit_window_attn_fwd then _bwd through the C ABI; dtable / dbias start at `acc` (they are accumulated into)"""
    from esvit_b200 import _lib
    from esvit_b200.ops import ATTN_WS_FLOATS, _p, _stream
    B, H, W, C, nH, ws = case.B, case.H, case.W, case.C, case.nH, case.ws
    dev = inp["qkv"].device
    nwin = B * (_pad(H, ws) // ws) * (_pad(W, ws) // ws)
    out = torch.empty(B, H * W, C, dtype=torch.bfloat16, device=dev)
    lse = torch.empty(nwin, nH, ws * ws, dtype=torch.float32, device=dev)
    dqkv = torch.empty_like(inp["qkv"])
    if nan_fill:
        for t in (out, lse, dqkv):
            t.fill_(math.nan)
    dtable = torch.full_like(inp["table"], acc)
    dbias = torch.full((3 * C,), acc, dtype=torch.float32, device=dev)
    if bias_ws is None:
        bias_ws = torch.full((nH * ATTN_WS_FLOATS,), math.nan, dtype=torch.float32, device=dev)
    _lib.call("esvit_window_attn_fwd", _p(inp["qkv"]), _p(inp["qb"]), _p(inp["table"]), _p(bias_ws), ready, _p(out),
              _p(lse), B, H, W, C, nH, ws, case.shift, case.scale, _stream())
    _lib.call("esvit_window_attn_bwd", _p(inp["qkv"]), _p(inp["qb"]), _p(inp["table"]), _p(bias_ws), ready, _p(out),
              _p(inp["dout"]), _p(lse), _p(dqkv), _p(dtable), _p(dbias), B, H, W, C, nH, ws, case.shift, case.scale,
              _stream())
    torch.cuda.synchronize()
    return dict(out=out, lse=lse, dqkv=dqkv, dtable=dtable - acc, dbias=dbias - acc)


def _check(got, ref, case, tag, inp):
    for k in ("out", "lse", "dqkv", "dtable", "dbias"):
        assert torch.isfinite(got[k]).all(), (tag, k)
    err = errors(got, ref, case)
    gates = _gates(case)
    if "dqk_win_D" in gates:
        err["dqk_win_D"] = dqk_win_bf16_o_D(got, inp, case)
        # v has no D term: its per-window error against exact fp64 stays gated
        err["dv_win"] = _per_window_max(got["dqkv"].reshape(-1, 3, case.C)[:, 2], ref["dqkv"].reshape(-1, 3, case.C)[:, 2],
                                        slot_tokens(case.B, case.H, case.W, case.ws, case.shift), 1)
    print(f"window-attn {tag}: " + " ".join(f"{k} {v:.2e}" for k, v in err.items()))
    bad = {k: (err[k], g) for k, g in gates.items() if not err[k] < g}
    assert not bad, (tag, bad)
    return err


def _gpu_case(name):
    case = CASES[name]
    inp = make_inputs(case, _seed(name), "cuda")
    return case, inp, ref_all(inp, case)


@pytest.fixture(autouse=True)
def _no_debug_env(monkeypatch):
    monkeypatch.delenv("ESVIT_ATTN_DBG", raising=False)
    monkeypatch.delenv("ESVIT_ATTN_GY", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_kernel_matches_fp64(name):
    case, inp, ref = _gpu_case(name)
    got = _run_kernel(inp, case)
    _check(got, ref, case, name, inp)
    tok = slot_tokens(case.B, case.H, case.W, case.ws, case.shift)
    pad = tok < 0
    if pad.any():
        # the padded slots' share of the qkv-bias gradient is well above its gate, unless the padded band is a shift
        # region of its own (map 24, ws 7, shift 3) and the -100 mask separates it from every real query
        nW = tok.shape[0] // case.B
        cut = S.shift_mask(case.H, case.W, case.ws, case.shift) != 0 if case.shift else torch.zeros(nW, 1, 1, dtype=bool)
        real_pad_pairs = (~pad[:nW, :, None]) & pad[:nW, None, :]
        if not (cut.expand_as(real_pad_pairs)[real_pad_pairs]).all():
            share = rel(ref["dbias"], ref["dqkv"].reshape(-1, 3 * case.C).sum(0))
            assert share > 2 * _gates(case)["dbias"], (name, share)


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="the backward's D = rowsum(dO * O) uses the bf16 O; where every softmax row of a "
                                       "(window, head) is one-hot, its dq / dk are a cancellation that this rounding "
                                       "dominates (DESIGN.md §4.3)")
def test_large_logit_dq_dk_per_window_against_exact_fp64():
    case, inp, ref = _gpu_case("w7_large")
    got = _run_kernel(inp, case)
    err = errors(got, ref, case)["dqkv_win"]
    print(f"window-attn w7_large: dqkv_win against exact fp64 {err:.2e}")
    assert err < GATES["normal"]["dqkv_win"]


# ================================ 3. the C-ABI contract (GPU) ==========================================================
PADDED = ["w7_c768_m3_s0", "w7_c384_m6_s3", "w14_c384_m6_s0", "w14_c192_m12_s7", "w14_h28_w12_s7"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", PADDED + ["w7_c96_m24_s3", "w14_c128_m24_s7"])
def test_outputs_fully_written_and_gradients_accumulated(name):
    """out / lse / dqkv start as NaN (all-padding query tiles included: the forward must write their lse, the backward
    must not read garbage); dtable / dbias start at 0.75 and end at 0.75 + the gradient; bias_ws starts as NaN (ws 14:
    the backward clears its own accumulator)"""
    case, inp, ref = _gpu_case(name)
    got = _run_kernel(inp, case, nan_fill=True, acc=0.75)
    _check(got, ref, case, name + " nan-filled, accumulated", inp)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w7_c96_m24_s3", "w7_c384_m6_s3", "w7_c768_m3_s0", "w7_c1024_m7_s0"])
def test_pre_expanded_bias_is_the_same_computation(name):
    from esvit_b200 import ops
    case, inp, ref = _gpu_case(name)
    bexp = ops.expand_rel_pos_bias(inp["table"], case.nH, 7)
    e = bexp.view(case.nH, 64, 64).cpu()
    # [nH][64][64]: log2-scaled table at (query i, key j) for i, j < 49, -inf in every column >= 49
    want = (inp["table"].cpu() * torch.tensor(LOG2E, dtype=torch.float32))[S.rel_pos_index(7).view(-1)]
    assert torch.allclose(e[:, :49, :49], want.view(49, 49, case.nH).permute(2, 0, 1), rtol=1e-7, atol=0)
    assert torch.isneginf(e[:, :, 49:]).all()
    a = _run_kernel(inp, case)
    b = _run_kernel(inp, case, bias_ws=bexp.clone(), ready=1)
    for k in ("out", "lse", "dqkv"):
        assert torch.equal(a[k], b[k]), k
    _check(b, ref, case, name + " bias_ready", inp)
    assert torch.equal(bexp.view(case.nH, 64, 64).cpu(), e)  # the kernels never write a ready expansion


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w7_c96_m24_s3", "w7_c384_m6_s3", "w14_c128_m24_s7", "w14_c192_m12_s7",
                                  "w7_h24_w28_s3", "w14_h28_w12_s7"])
def test_persistent_window_loops(monkeypatch, name):
    """ESVIT_ATTN_GY = 1, 2, 3 CTAs per head walk many windows each (both cp.async stages, the odd / even stage order):
    out / lse / dqkv bit-identical to the default grid, gradients against the reference"""
    case, inp, ref = _gpu_case(name)
    base = _run_kernel(inp, case)
    for gy in ("1", "2", "3"):
        monkeypatch.setenv("ESVIT_ATTN_GY", gy)
        got = _run_kernel(inp, case)
        for k in ("out", "lse", "dqkv"):
            assert torch.equal(got[k], base[k]), (gy, k)
        _check(got, ref, case, f"{name} GY={gy}", inp)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w7_c192_m28_s3", "w14_c256_m28_s7", "w7_c768_m3_s0"])
def test_reruns_are_bit_identical(name):
    case, inp, _ = _gpu_case(name)
    a, b = _run_kernel(inp, case), _run_kernel(inp, case)
    for k in ("out", "lse", "dqkv"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("ws,shift,C", [(7, 3, 96), (14, 7, 128)])
def test_resolution_groups_equal_one_group_calls(ws, shift, C):
    """WindowAttentionGroupsFn over the step's layout (2 global 56² maps then 8 local 24² maps in one tensor, one shared
    ws-7 expansion) against one call per group on its own slice: out and dqkv bit-identical, the table / qkv-bias
    gradients (float atomics, accumulated over both groups) within fp32 summation noise"""
    from esvit_b200 import ops
    nH = C // HD
    g = torch.Generator().manual_seed(17 + ws)
    groups = ((2, 56, 56, 0), (8, 24, 24, 2 * 56 * 56))
    T = sum(B * H * W for B, H, W, _ in groups)
    qkv0 = torch.randn(T, 3 * C, generator=g).to(torch.bfloat16).cuda()
    bias0 = torch.randn(3 * C, generator=g).cuda()
    table0 = torch.randn((2 * ws - 1) ** 2, nH, generator=g).cuda()
    dout = torch.randn(T, C, generator=g).to(torch.bfloat16).cuda()
    scale = HD ** -0.5

    def leaves():
        return (qkv0.clone().requires_grad_(), bias0.clone().requires_grad_(), table0.clone().requires_grad_())

    qkv, bias, table = leaves()
    out = ops.WindowAttentionGroupsFn.apply(qkv, bias, table, groups, nH, ws, shift, scale,
                                            ops.expand_rel_pos_bias(table, nH, ws))
    out.backward(dout)
    qkv2, bias2, table2 = leaves()
    bexp = ops.expand_rel_pos_bias(table2, nH, ws)
    outs = []
    for B, H, W, r0 in groups:
        outs.append(ops.WindowAttentionGroupsFn.apply(qkv2[r0:r0 + B * H * W], bias2, table2, ((B, H, W, 0),), nH, ws,
                                                      shift, scale, bexp))
    out2 = torch.cat(outs)
    out2.backward(dout)
    assert torch.equal(out, out2)
    assert torch.equal(qkv.grad, qkv2.grad)
    assert rel(table.grad, table2.grad) < 1e-5
    assert rel(bias.grad, bias2.grad) < 1e-5


@pytest.mark.gpu
def test_invalid_geometry_is_rejected():
    """every shape make_geo refuses raises ValueError (ESVIT_ERR_BAD_ARG) before any launch; the buffers are real"""
    from esvit_b200 import _lib
    from esvit_b200.ops import ATTN_WS_FLOATS, _p, _stream
    C, nH = 64, 2
    qkv = torch.zeros(2 * 14 * 14 * 3 * C, dtype=torch.bfloat16, device="cuda")
    qb = torch.zeros(3 * C, dtype=torch.bfloat16, device="cuda")
    table = torch.zeros(27 * 27 * 32, device="cuda")
    ws_buf = torch.zeros(32 * ATTN_WS_FLOATS, device="cuda")
    out = torch.zeros(2 * 14 * 14 * 32 * HD, dtype=torch.bfloat16, device="cuda")
    lse = torch.zeros(2 * 4 * 32 * 196, device="cuda")
    dqkv, dtable, dbias = torch.zeros_like(qkv), torch.zeros_like(table), torch.zeros(3 * 32 * HD, device="cuda")
    bad = [  # (B, H, W, C, nH, ws, shift)
        (2, 14, 14, C, nH, 5, 0), (2, 14, 14, C, nH, 8, 0), (2, 14, 14, C, nH, 0, 0),
        (2, 14, 14, C, nH, 7, -1), (2, 14, 14, C, nH, 7, 7), (2, 14, 14, C, nH, 14, 14),
        (2, 14, 14, 96, nH, 7, 0), (2, 14, 14, C, 3, 14, 0), (2, 14, 14, 0, 0, 7, 0),
        (0, 14, 14, C, nH, 7, 0), (-1, 14, 14, C, nH, 14, 0),
        (2, 0, 14, C, nH, 7, 0), (2, 14, 0, C, nH, 14, 7), (2, -7, 14, C, nH, 7, 3), (2, 14, -1, C, nH, 14, 0),
    ]
    for B, H, W, Cc, h, ws, shift in bad:
        for ready in (0, 1):
            with pytest.raises(ValueError):
                _lib.call("esvit_window_attn_fwd", _p(qkv), _p(qb), _p(table), _p(ws_buf), ready, _p(out), _p(lse),
                          B, H, W, Cc, h, ws, shift, 0.1, _stream())
            with pytest.raises(ValueError):
                _lib.call("esvit_window_attn_bwd", _p(qkv), _p(qb), _p(table), _p(ws_buf), ready, _p(out), _p(out),
                          _p(lse), _p(dqkv), _p(dtable), _p(dbias), B, H, W, Cc, h, ws, shift, 0.1, _stream())
    for h, ws in ((0, 7), (-1, 7), (2, 5)):
        with pytest.raises(ValueError):
            _lib.call("esvit_window_attn_expand_bias", _p(table), _p(ws_buf), h, ws, _stream())
    torch.cuda.synchronize()
    assert not dqkv.any() and not dtable.any() and not dbias.any() and not out.any() and not lse.any()
