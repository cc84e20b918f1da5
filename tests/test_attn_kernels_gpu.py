"""The ViT, CvT and ViL attention kernels (csrc/mhsa.cu: esvit_mhsa_fwd / _bwd, esvit_mhsa_win_fwd / _bwd;
csrc/vil_attn.cu: esvit_vil_sc_fwd / _bwd; csrc/vil_dense.cu: esvit_vil_dense_fwd / _bwd) against an fp64 reference of
their C-ABI contract, called through the C ABI with explicitly allocated buffers at every launch of an eager 2 + 8-crop
step (K = 65 536) of the nine backbones that use them, at the bench batch and at synthetic edge geometries.

The reference (CPU tests, not `gpu`-marked) mirrors the header, layouts included:
  mhsa   qkv [B*L, 3C] as [q|k|v][head][64] -> out [B*L, C], lse [B, nH, L] (natural log), D, dqkv [B*L, 3C];
  win    windows of the zero-padded Hp x Wp map (images, then windows row-major): padded keys take part, padded query
         rows are not stored and their dq is exactly 0; lse / dvec [windows, nH, w*w] including padded query slots;
  sc     oracle/vil_attn.dense_index / dense_attention's masked N x N attention for out and the gradients, plus lse
         [B, nH, chunks, 49] (padded slots of an edge chunk: q = 0, so the scores are the bias), lse_g [B, nH], the
         written dbias [nH, 49, 442] (0 in the columns of chunks the mode skips) and dbias_g [nH, N];
  dense  softmax(scale q k^T + bias) v with bias [nH, L, L]; dbias is the sum of dS over the images.
It is pinned to 1e-12 against float64 autograd of oracle.vit.attention, oracle.cvt.attention (on a padded map),
oracle.vil.sc_attention with oracle.vil_attn.dense_attention, and oracle.vil.full_attention.  Each plausible kernel bug
of SENSITIVITY, emulated in the fp64 reference, moves its named metric by at least 5x the gate on a named GPU case.

Metrics (see GATES), over every query row the contract defines:
  out / out_seq     global rel-L2; worst rel-L2 per (sequence | window | image chunk, head); ViL's global row is a
                    group of its own
  lse               max |lse - lse_ref| (natural log), lse_g included
  dqkv / dqkv_seq   global rel-L2; worst per (sequence | window, q|k|v, head) (ViL: dq | dkv per image); window mode
                    over all B*Hp*Wp rows, so a non-zero dq on a padded row counts
  dbias / dbias_head, dbias_g / dbias_g_head (ViL): global and worst per-head rel-L2
Regimes: normal, large logits, late maximum, uniform (make_inputs).  Where one key dominates a row (large logits, late
maximum: the "peaked" gate class) dq / dk per (sequence, head) are gated as dqk_seq_D against fp64 gradients that take
D = rowsum(dO * O) from the kernel's bf16 O, as the kernels do, and so are the bias gradients (*_D); dv_seq and the
global dqkv stay against exact fp64.

TABLE lists every distinct launch signature of the second eager B = 2 step; test_table_matches_the_step checks it.
Measured maxima and gates: DESIGN.md §4.19."""
import ctypes
import math
import struct
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

from oracle import vil_attn as VA

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
LOG2E = 1.4426950408889634
BENCH_B, TABLE_B = 64, 2
PAD = 37            # sentinel rows past the end of every buffer in the contract test
SENTINEL = -1234.0  # exactly representable in bf16
W2, NB = VA.W * VA.W, VA.NB
VIL_SCALE = 32 ** -0.5
INF = float("inf")


def f32(x):
    """the fp32 value a float argument reaches the kernel as"""
    return struct.unpack("f", struct.pack("f", x))[0]


# Gates, per family and gate class (gate_class), at about 3x the largest error measured on an H100 over every case
# below (DESIGN.md §4.19) and never looser than the per-backbone tests' gates (mhsa: out 1e-2, dqkv 2e-2, lse 2e-4;
# win: out 1e-2, dqkv 2e-2; ViL: out 2e-2, dq / dkv / dbias 6e-2).  The exception is the lse of the peaked class:
# large-logit rows have |lse| up to ~1e3, where 1e-4 is a few fp32 ulps.  Peaked rows gate dq / dk (dqk_seq_D) and
# the bias gradients (*_D) against fp64 with D from the kernel's bf16 O; dv and the global dqkv against exact fp64.
GATES = {
    "mhsa": {
        "normal": dict(out=6e-3, out_seq=7e-3, lse=1e-5, dqkv=1.3e-2, dqkv_seq=2e-2),
        "peaked": dict(out=5e-3, out_seq=6e-3, lse=9.2e-4, dqkv=2e-2, dv_seq=9e-3, dqk_seq_D=1.3e-2),
    },
    "win": {
        "normal": dict(out=7e-3, out_seq=9e-3, lse=9e-6, dqkv=1e-2, dqkv_seq=2.7e-2),
        "peaked": dict(out=5.5e-3, out_seq=7e-3, lse=4.5e-4, dqkv=2e-2, dv_seq=1.2e-2, dqk_seq_D=1.5e-2),
    },
    "sc": {
        "normal": dict(out=5.5e-3, out_seq=8e-3, lse=7.5e-6, dqkv=1e-2, dqkv_seq=1.4e-2, dbias=6.5e-3,
                       dbias_head=9e-3, dbias_g=1.1e-2, dbias_g_head=1.3e-2),
        "peaked": dict(out=5.5e-3, out_seq=8e-3, lse=3.2e-4, dqkv=4.5e-2, dv_seq=8e-3, dqk_seq_D=1.2e-2,
                       dbias_D=7e-5, dbias_head_D=7e-5, dbias_g_D=1.8e-3, dbias_g_head_D=1.9e-3),
    },
    "vd": {
        "normal": dict(out=5.5e-3, out_seq=8e-3, lse=1.2e-5, dqkv=9e-3, dqkv_seq=6e-2, dbias=7.5e-3,
                       dbias_head=1.8e-2),
        "peaked": dict(out=5e-3, out_seq=6e-3, lse=6.7e-4, dqkv=2.6e-2, dv_seq=8e-3, dqk_seq_D=7.5e-3, dbias_D=9e-5,
                       dbias_head_D=1.5e-3),
    },
}
REGIMES = ("normal", "large", "late", "uniform")


def gate_class(regime):
    """normal: the normal and uniform regimes; peaked: large logits and the late maximum, where rows are dominated by
    one key and dq / dk are gated against the fp64 gradients that take D from the kernel's bf16 O"""
    return "peaked" if regime in ("large", "late") else "normal"


# ---- cases -------------------------------------------------------------------------------------------------------------
# fam: mhsa (B, L, C, nH, scale), win (B, H, W, w, C, nH, scale), sc (B, nx, ny, nH; scale 32^-0.5), vd (B, L, C, nH,
# scale 32^-0.5)
Case = namedtuple("Case", "fam B C nH scale L H W w nx ny", defaults=(0, 0, 0, 0, 0, 0))


def mhsa(B, L, C, nH, scale=0.125):
    return Case("mhsa", B, C, nH, f32(scale), L=L)


def win(B, H, W, w, C, nH, scale=None):
    return Case("win", B, C, nH, f32(C ** -0.5 if scale is None else scale), H=H, W=W, w=w)


def sc(B, nx, ny, nH):
    return Case("sc", B, 32 * nH, nH, f32(VIL_SCALE), nx=nx, ny=ny)


def vd(B, L, C, nH):
    return Case("vd", B, C, nH, f32(VIL_SCALE), L=L)


def name_of(c):
    if c.fam == "mhsa":
        return f"mhsa_B{c.B}_L{c.L}_C{c.C}_h{c.nH}" + ("" if c.scale == f32(0.125) else f"_s{c.scale:.3g}")
    if c.fam == "win":
        return f"win_B{c.B}_{c.H}x{c.W}_w{c.w}_C{c.C}_h{c.nH}"
    if c.fam == "sc":
        return f"sc_B{c.B}_{c.nx}x{c.ny}_h{c.nH}"
    return f"vd_B{c.B}_L{c.L}_C{c.C}_h{c.nH}"


# the table's signature of a case's launches (fwd and bwd share it)
def sig_of(c):
    if c.fam == "mhsa":
        return (c.B, c.L, c.C, c.nH, c.scale)
    if c.fam == "win":
        return (c.B, c.H, c.W, c.w, c.C, c.nH, c.scale)
    if c.fam == "sc":
        return (c.B, c.nx, c.ny, c.nH)
    return (c.B, c.L, c.C, c.nH)


def case_of(fam, sig):
    if fam == "mhsa":
        B, L, C, nH, s = sig
        return mhsa(B, L, C, nH, s)
    if fam == "win":
        B, H, W, w, C, nH, s = sig
        return win(B, H, W, w, C, nH, s)
    if fam == "sc":
        return sc(*sig)
    return vd(*sig)


ENTRY = {"esvit_mhsa_fwd": ("mhsa", "fwd"), "esvit_mhsa_bwd": ("mhsa", "bwd"),
         "esvit_mhsa_win_fwd": ("win", "fwd"), "esvit_mhsa_win_bwd": ("win", "bwd"),
         "esvit_vil_sc_fwd": ("sc", "fwd"), "esvit_vil_sc_bwd": ("sc", "bwd"),
         "esvit_vil_dense_fwd": ("vd", "fwd"), "esvit_vil_dense_bwd": ("vd", "bwd")}


def _vit(C, nH, Lg, Ll):
    return [(f"mhsa_{d}", B, L, C, nH, f32(0.125)) for d in ("fwd", "bwd") for B, L in ((4, Lg), (16, Ll))]


def _cvt(dims, heads, wins):
    out = []
    for i, (C, nH, ws) in enumerate(zip(dims, heads, wins)):
        for B, m in ((4, 56 >> i), (16, (24 >> i))):
            out += [(f"win_{d}", B, m, m, min(ws, m), C, nH, f32(C ** -0.5)) for d in ("fwd", "bwd")]
    return out


_VIL = ([(f"sc_{d}", B, m, m, nH) for d in ("fwd", "bwd") for B, m, nH in ((4, 56, 3), (16, 24, 3), (4, 28, 6),
                                                                             (16, 12, 6))]
        + [(f"vd_{d}", B, L, C, nH) for d in ("fwd", "bwd") for B, L, C, nH in ((4, 197, 384, 12), (16, 37, 384, 12),
                                                                                 (4, 49, 768, 24), (16, 9, 768, 24))])

# TABLE[arch]: the step's launches of the eight entry points at B = 2 (2 global crops -> 4 sequences, 8 local crops ->
# 16), one tuple (entry, *signature) per distinct signature
TABLE = {
    "deit_tiny_p16": _vit(192, 3, 197, 37),
    "deit_small_p16": _vit(384, 6, 197, 37),
    "deit_small_p8": _vit(384, 6, 785, 145),
    "vit_base_p16": _vit(768, 12, 197, 37),
    "cvt_13": _cvt((64, 192, 384, 768), (1, 3, 6, 12), (7, 7, 7, 7)),
    "cvt_13_w14": _cvt((64, 192, 384, 768), (1, 3, 6, 12), (14, 14, 14, 7)),
    "cvt_s3": _cvt((64, 128, 256, 512), (2, 4, 8, 16), (7, 7, 7, 7)),
    "cvt_s3_w14": _cvt((64, 128, 256, 512), (2, 4, 8, 16), (14, 14, 14, 7)),
    "vil_2262": _VIL,
}


def table_cases(scale_b=1):
    """name -> case of every geometry of TABLE (its fwd and bwd launch), at B * scale_b"""
    out = {}
    for ents in TABLE.values():
        for e in ents:
            fam = e[0].rsplit("_", 1)[0]
            c = case_of(fam, e[1:])
            c = c._replace(B=c.B * scale_b)
            out[name_of(c)] = c
    return out


SYNTHETIC = (
    # whole-sequence: partial and single key tiles, one query, nH 3 and 12, a non-default scale
    [mhsa(2, L, 64 * nH, nH) for L in (1, 63, 64, 65, 128, 129, 256) for nH in (3, 12)]
    + [mhsa(2, 65, 192, 3, 0.3)]
    # windows: w 1..14, w = H, rectangular padded maps, odd head counts at head dim 32 (the prep kernel's head pairs)
    + [win(2, 5, 3, 1, 64, 2), win(2, 3, 3, 3, 64, 1), win(2, 6, 6, 6, 128, 4), win(2, 7, 7, 7, 192, 3),
       win(2, 12, 12, 12, 256, 8), win(2, 14, 14, 14, 384, 6), win(2, 30, 17, 7, 192, 3), win(2, 30, 17, 14, 128, 4),
       win(2, 17, 30, 14, 64, 1), win(2, 26, 13, 12, 96, 3), win(3, 9, 20, 6, 160, 5)]
    # ViL sliding chunk: non-square maps padded in both directions, a single (padded) chunk
    + [sc(2, 10, 17, 3), sc(3, 16, 9, 6), sc(2, 3, 5, 3)]
    # ViL dense: one token, a 9-token map, the largest L, more images than the 16 dq parts
    + [vd(2, 1, 96, 3), vd(2, 9, 768, 24), vd(2, 256, 128, 4), vd(17, 49, 192, 6), vd(33, 37, 384, 12)]
)
SYNTHETIC = {name_of(c): c for c in SYNTHETIC}
MODES = tuple(range(-1, 9))


def modes_for(c, regime, bench=False):
    """ViL modes a case runs: every mode on the synthetic maps and, in the normal regime, on the table geometries"""
    if c.fam != "sc":
        return (None,)
    if bench:
        return (0, 3)
    if regime == "normal" or name_of(c) in SYNTHETIC:
        return MODES
    return (-1, 0, 6)


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _pad(n, w):
    return -(-n // w) * w


def rows_of(c):
    """token rows of the qkv (q) input"""
    if c.fam in ("mhsa", "vd"):
        return c.B * c.L
    if c.fam == "win":
        return c.B * _pad(c.H, c.w) * _pad(c.W, c.w)
    return c.B * (1 + c.nx * c.ny)


def out_rows(c):
    return c.B * c.H * c.W if c.fam == "win" else rows_of(c)


def hd_of(c):
    return c.C // c.nH


def _last_key_rows(c):
    """the rows whose keys the late-max regime raises: the last key of every sequence / window"""
    if c.fam in ("mhsa", "vd"):
        return torch.arange(c.B) * c.L + c.L - 1
    return win_maps(c)[0][:, -1]


def make_inputs(c, regime, dev, seed, mode=0):
    """bf16 qkv (or q / kv) ~ N(0, 1.5^2) and dout ~ N(0, 1), fp32 biases ~ N(0, 1); large: qkv x 8, biases in
    [-8, 8]; late: every row's maximum score sits on the last key (the last, partial key tile; ViL: the neighbour
    chunks after the own one); uniform: q = 0 and zero biases, so every softmax row is exactly uniform.  Drawn on the
    CPU for CPU devices and with a device generator otherwise (same values on every run of a device)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    amp = 1.5 * (8.0 if regime == "large" else 1.0)

    def n(*s):
        return torch.randn(*s, generator=g, device=dev)

    def bias(*s):
        if regime == "large":
            return torch.rand(*s, generator=g, device=dev) * 16 - 8
        if regime == "uniform":
            return torch.zeros(*s, device=dev)
        return n(*s)

    C, hd = c.C, hd_of(c)
    R = rows_of(c)
    ins = {}
    if c.fam == "sc":
        q, kv = n(R, C) * amp, n(R, 2 * C) * amp
        if regime == "uniform":
            q.zero_()
        ins.update(q=q, kv=kv, bias=bias(c.nH, W2, NB), bias_g=bias(c.nH, 1 + c.nx * c.ny))
        if regime == "late":  # every neighbour chunk after the own one (tile 0) sits 5 above it
            ins["bias"][:, :, 1:].view(c.nH, W2, 9, W2)[:, :, [j for j in range(9) if j != 4]] += 5.0
    else:
        qkv = n(R, 3 * C) * amp
        if regime == "uniform":
            qkv[:, :C] = 0
        if regime == "late":  # q += s, last key = kappa s for a fixed sign vector s: its score sits 1.5 above the
            # expected largest other score of a row (sigma sqrt(2 ln L)), so the row's softmax is not one-hot
            L = c.w * c.w if c.fam == "win" else c.L
            sigma = math.hypot(1.5 * math.hypot(1.5, 1.0) * math.sqrt(hd) * c.scale, 1.0 if c.fam == "vd" else 0.0)
            s = torch.where(n(hd) > 0, 1.0, -1.0)
            qkv[:, :C] += s.repeat(c.nH)
            rows = _last_key_rows(c).to(dev)
            kappa = (sigma * math.sqrt(2 * math.log(L)) + 1.5) / (hd * c.scale)
            qkv[rows, C:2 * C] = (kappa * s).repeat(c.nH)
        ins["qkv"] = qkv
        if c.fam == "vd":
            ins["bias"] = bias(c.nH, c.L, c.L)
    dout = n(out_rows(c), C)
    ins = {k: (v.to(BF16) if k in ("q", "kv", "qkv") else v) for k, v in ins.items()}
    ins["dout"] = dout.to(BF16)
    return ins


# ================================ the fp64 reference ===================================================================
def _slices(n, per_item, budget=1 << 25):
    step = max(1, budget // max(per_item, 1))
    return [(a, min(n, a + step)) for a in range(0, n, step)]


def _attn(q, k, v, dO, scale, bias=None, O=None, D=None, no_rescale_tile=None):
    """fp64 softmax(scale q k^T + bias) v and its backward with explicit formulas (q, k, v, dO [..., L, d]); D = rowsum
    (dO * O) of the exact output unless O (another output) or D is given.  no_rescale_tile: the online softmax without
    the rescale of earlier key tiles of that width (a sensitivity bug)."""
    s = (q @ k.transpose(-1, -2)) * scale
    if bias is not None:
        s = s + bias
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    o = P @ v
    if no_rescale_tile:
        Lk, t = s.shape[-1], no_rescale_tile
        nt = -(-Lk // t)
        sp = F.pad(s, (0, nt * t - Lk), value=-INF).unflatten(-1, (nt, t))
        m = sp.amax(-1).cummax(-1).values  # the running maximum after each tile
        wgt = torch.exp(sp - m[..., None]).flatten(-2)[..., :Lk]
        l = wgt.sum(-1)
        o, lse = (wgt @ v) / l[..., None], m[..., -1] + torch.log(l)
    if D is None:
        D = (dO * (o if O is None else O)).sum(-1)
    dS = P * (dO @ v.transpose(-1, -2) - D[..., None])
    return dict(o=o, lse=lse, D=D, dq=(dS @ k) * scale, dk=(dS.transpose(-1, -2) @ q) * scale,
                dv=P.transpose(-1, -2) @ dO, dS=dS)


def _heads(t, n, L, parts, nH):
    """[n*L, parts*nH*d] -> [parts, n, nH, L, d]"""
    return t.double().reshape(n, L, parts, nH, -1).permute(2, 0, 3, 1, 4)


def _rows(*ts):
    """[n, nH, L, d] tensors -> [n*L, len(ts)*nH*d] in [part][head][d] channel order"""
    n, nH, L, d = ts[0].shape
    return torch.stack(ts).permute(1, 3, 0, 2, 4).reshape(n * L, len(ts) * nH * d)


def ref_mhsa(c, ins, bug=None, O=None):
    B, L, C, nH = c.B, c.L, c.C, c.nH
    dev = ins["qkv"].device
    out = torch.empty(B * L, C, dtype=F64, device=dev)
    lse = torch.empty(B, nH, L, dtype=F64, device=dev)
    D = torch.empty_like(lse)
    dqkv = torch.empty(B * L, 3 * C, dtype=F64, device=dev)
    for b0, b1 in _slices(B, nH * L * L):
        r = slice(b0 * L, b1 * L)
        q, k, v = _heads(ins["qkv"][r], b1 - b0, L, 3, nH)
        dO = _heads(ins["dout"][r], b1 - b0, L, 1, nH)[0]
        Ob = None if O is None else _heads(O[r], b1 - b0, L, 1, nH)[0]
        if bug == "kv_head_xor1":
            perm = [h ^ 1 if h ^ 1 < nH else h for h in range(nH)]
            k, v = k[:, perm], v[:, perm]
        if bug == "keys_past_L_zero":  # the zero-filled rows of the last key tile scored 0
            k, v = (F.pad(t, (0, 0, 0, (-L) % 64)) for t in (k, v))
        a = _attn(q, k, v, dO, c.scale, O=Ob, no_rescale_tile=64 if bug == "no_rescale" else None)
        dk, dv = a["dk"][..., :L, :], a["dv"][..., :L, :]
        if bug == "dk_no_scale":
            dk = dk / c.scale
        out[r] = _rows(a["o"])
        lse[b0:b1] = a["lse"] * (LOG2E if bug == "lse_log2" else 1.0)
        D[b0:b1] = a["D"]
        dqkv[r] = _rows(a["dq"], dk, dv)
    return dict(out=out, lse=lse, D=D, dqkv=dqkv)


def win_maps(c, swap=False):
    """(prow, crow) [windows, w*w]: the padded-map row (qkv / dqkv) and the cropped-map row (out / dout, -1 on padded
    positions) of every window slot, images then windows row-major then tokens row-major.  swap: the window's row and
    column index exchanged (a sensitivity bug; both maps follow it, as the kernel's gathers and stores would)."""
    B, H, W, w = c.B, c.H, c.W, c.w
    Hp, Wp = _pad(H, w), _pad(W, w)
    nwx = Wp // w
    wi = torch.arange((Hp // w) * nwx)
    wy, wx = wi // nwx, wi % nwx
    if swap:
        wy, wx = wx, wy
    t = torch.arange(w * w)
    y = (wy[:, None] * w + t[None] // w)[None]
    x = (wx[:, None] * w + t[None] % w)[None]
    b = torch.arange(B)[:, None, None]
    prow = (((b * Hp + y) * Wp + x) % (B * Hp * Wp)).reshape(-1, w * w)
    crow = torch.where((y < H) & (x < W), (b * H + y) * W + x, -1).reshape(-1, w * w)
    return prow, crow


def ref_win(c, ins, bug=None, O=None):
    B, C, nH, w = c.B, c.C, c.nH, c.w
    L, hd = w * w, hd_of(c)
    dev = ins["qkv"].device
    prow, crow = (t.to(dev) for t in win_maps(c, swap=bug == "win_transposed"))
    nw = prow.shape[0]
    scale = hd ** -0.5 if bug == "scale_hd" else c.scale
    out = torch.zeros(B * c.H * c.W, C, dtype=F64, device=dev)
    lse = torch.empty(nw, nH, L, dtype=F64, device=dev)
    D = torch.empty_like(lse)
    dqkv = torch.zeros(rows_of(c), 3 * C, dtype=F64, device=dev)
    zero = torch.zeros(1, C, dtype=F64, device=dev)

    def cropped(t, rows):  # cropped-map rows, zero on padded slots
        return torch.cat([zero, t.double()])[(rows + 1).reshape(-1)]

    for s0, s1 in _slices(nw, nH * L * L):
        n = s1 - s0
        q, k, v = _heads(ins["qkv"][prow[s0:s1].reshape(-1)], n, L, 3, nH)
        dO = _heads(cropped(ins["dout"], crow[s0:s1]), n, L, 1, nH)[0]
        Ob = None if O is None else _heads(cropped(O, crow[s0:s1]), n, L, 1, nH)[0]
        bias = None
        if bug == "pad_keys_masked":
            bias = torch.zeros(n, 1, 1, L, dtype=F64, device=dev).masked_fill((crow[s0:s1] < 0)[:, None, None], -INF)
        if bug == "keys_past_L_zero":
            k, v = (F.pad(t, (0, 0, 0, (-L) % 64)) for t in (k, v))
        a = _attn(q, k, v, dO, scale, bias, O=Ob)
        if bug == "prep_head_pairs":  # lanes 16-31 of the head-dim-32 prep kernel read head h, not h + 1
            Dp = a["D"].clone()
            Dp[:, 1::2] = a["D"][:, 0:nH - 1:2]
            a = _attn(q, k, v, dO, scale, bias, D=Dp)
        real = crow[s0:s1] >= 0
        o = _rows(a["o"]).view(n, L, C)
        out[crow[s0:s1][real]] = o[real]
        lse[s0:s1] = a["lse"]
        D[s0:s1] = a["D"]
        dqkv[prow[s0:s1].reshape(-1)] = _rows(a["dq"], a["dk"][..., :L, :], a["dv"][..., :L, :])
    return dict(out=out, lse=lse, D=D, dqkv=dqkv)


def _mirror_mode(mode):
    """the mode whose neighbour chunk is 8 - j for mode's chunk j (mode_dict: chunk = mode if mode > 4 else mode - 1)"""
    if mode <= 0:
        return mode
    j = 8 - (mode if mode > 4 else mode - 1)
    return j if j > 4 else j + 1


def sc_slots(c):
    """[chunks, 49] in-image token index (0-based over the nx*ny map, -1 on padded positions) of every chunk slot"""
    mx, my = _pad(c.nx, VA.W) // VA.W, _pad(c.ny, VA.W) // VA.W
    ch = torch.arange(mx * my)
    l = torch.arange(W2)
    X = (ch // my)[:, None] * VA.W + (l // VA.W)[None]
    Y = (ch % my)[:, None] * VA.W + (l % VA.W)[None]
    return torch.where((X < c.nx) & (Y < c.ny), X * c.ny + Y, -1)


def sc_key_columns(c, mode):
    """[chunks, NB] bool: the bias columns a chunk's queries read (the global key, then the keys of the mode's
    neighbour chunks that lie on the map)"""
    mx, my = _pad(c.nx, VA.W) // VA.W, _pad(c.ny, VA.W) // VA.W
    ch = torch.arange(mx * my)
    r = torch.arange(W2)
    ok = torch.zeros(mx * my, NB, dtype=torch.bool)
    ok[:, 0] = True
    for j in VA.mode_chunks(mode):
        X = ((ch // my) + j // 3 - 1)[:, None] * VA.W + (r // VA.W)[None]
        Y = ((ch % my) + j % 3 - 1)[:, None] * VA.W + (r % VA.W)[None]
        ok[:, 1 + j * W2:1 + (j + 1) * W2] = (X >= 0) & (X < c.nx) & (Y >= 0) & (Y < c.ny)
    return ok


def ref_sc(c, ins, mode, bug=None, O=None):
    B, C, nH, nx, ny = c.B, c.C, c.nH, c.nx, c.ny
    n, N = nx * ny, 1 + nx * ny
    dev = ins["q"].device
    idx = VA.dense_index(nx, ny, _mirror_mode(mode) if bug == "chunk_mirrored" else mode, device=dev)
    bias, bias_g = ins["bias"].double(), ins["bias_g"].double()
    if bug == "no_global_bias":
        bias = bias.clone()
        bias[:, :, 0] = 0
    if bug == "bias_g_shift":
        bias_g = torch.roll(bias_g, 1, -1)
    loc = bias.reshape(nH, -1)[:, idx.clamp_min(0)].masked_fill((idx < 0)[None], -INF)
    bm = torch.cat([bias_g[:, None, :], loc], 1)  # [nH, N, N], as VA.dense_attention builds it
    out = torch.empty(B * N, C, dtype=F64, device=dev)
    lse_rows = torch.empty(B, nH, N, dtype=F64, device=dev)
    D_rows = torch.empty_like(lse_rows)
    dq = torch.empty(B * N, C, dtype=F64, device=dev)
    dkv = torch.empty(B * N, 2 * C, dtype=F64, device=dev)
    dS = torch.zeros(nH, N, N, dtype=F64, device=dev)
    for b0, b1 in _slices(B, nH * N * N):
        r = slice(b0 * N, b1 * N)
        q = _heads(ins["q"][r], b1 - b0, N, 1, nH)[0]
        k, v = _heads(ins["kv"][r], b1 - b0, N, 2, nH)
        dO = _heads(ins["dout"][r], b1 - b0, N, 1, nH)[0]
        Ob = None if O is None else _heads(O[r], b1 - b0, N, 1, nH)[0]
        a = _attn(q, k, v, dO, c.scale, bm[None], O=Ob)
        out[r], dq[r], dkv[r] = _rows(a["o"]), _rows(a["dq"]), _rows(a["dk"], a["dv"])
        lse_rows[b0:b1], D_rows[b0:b1] = a["lse"], a["D"]
        dS += a["dS"].sum(0)
    ok = idx >= 0
    dbias = torch.zeros(nH, W2 * NB, dtype=F64, device=dev)
    dbias.index_add_(1, idx[ok], dS[:, 1:][:, ok])
    # the contract layout [B, nH, chunks, 49]: real slots from their token's row; padded slots see q = 0, so their
    # scores are the bias of the columns their chunk reads
    slots = sc_slots(c).to(dev)
    cols = sc_key_columns(c, mode).to(dev)
    pad_lse = torch.logsumexp(bias[:, None].masked_fill(~cols[None, :, None, :], -INF), -1)  # [nH, chunks, 49]
    lse = pad_lse[None].repeat(B, 1, 1, 1)
    D = torch.zeros_like(lse)
    real = slots >= 0
    lse[:, :, real] = lse_rows[:, :, 1 + slots[real]]
    D[:, :, real] = D_rows[:, :, 1 + slots[real]]
    if bug == "lse_log2":
        lse = lse * LOG2E
    return dict(out=out, lse=lse, lse_g=lse_rows[:, :, 0], D=D, dqkv=torch.cat([dq, dkv], 1),
                dbias=dbias.view(nH, W2, NB), dbias_g=dS[:, 0])


def ref_vd(c, ins, bug=None, O=None):
    B, L, C, nH = c.B, c.L, c.C, c.nH
    dev = ins["qkv"].device
    bias = ins["bias"].double()
    if bug == "bias_transposed":
        bias = bias.transpose(-1, -2)
    out = torch.empty(B * L, C, dtype=F64, device=dev)
    lse = torch.empty(B, nH, L, dtype=F64, device=dev)
    D = torch.empty_like(lse)
    dqkv = torch.empty(B * L, 3 * C, dtype=F64, device=dev)
    dbias = torch.zeros(nH, L, L, dtype=F64, device=dev)
    for b0, b1 in _slices(B, nH * L * L):
        r = slice(b0 * L, b1 * L)
        q, k, v = _heads(ins["qkv"][r], b1 - b0, L, 3, nH)
        dO = _heads(ins["dout"][r], b1 - b0, L, 1, nH)[0]
        Ob = None if O is None else _heads(O[r], b1 - b0, L, 1, nH)[0]
        a = _attn(q, k, v, dO, c.scale, bias[None], O=Ob)
        out[r], dqkv[r] = _rows(a["o"]), _rows(a["dq"], a["dk"], a["dv"])
        lse[b0:b1], D[b0:b1] = a["lse"], a["D"]
        keep = torch.ones(b1 - b0, dtype=torch.bool, device=dev)
        if bug == "dbias_one_part":  # only part 0 (images 0, 16, 32, ...) summed
            keep = (torch.arange(b0, b1, device=dev) % 16) == 0
        dbias += a["dS"][keep].sum(0)
    return dict(out=out, lse=lse, D=D, dqkv=dqkv, dbias=dbias)


def reference(c, ins, mode=None, bug=None, O=None):
    if c.fam == "mhsa":
        return ref_mhsa(c, ins, bug, O)
    if c.fam == "win":
        return ref_win(c, ins, bug, O)
    if c.fam == "sc":
        return ref_sc(c, ins, mode, bug, O)
    return ref_vd(c, ins, bug, O)


# ================================ metrics ==============================================================================
def _rel(a, b):
    a, b = a.double(), b.double().to(a.device)
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _per_group(got, ref, groups, parts, nH, sel=None):
    """largest rel-L2 over (group, part, head) of row-major [R, parts*nH*d] tensors; groups [G, n] rows, -1 absent;
    sel: the parts measured (all by default)"""
    groups = groups.to(got.device)
    ok = (groups >= 0)[:, :, None, None, None]

    def g(t):
        return t.double().to(got.device).reshape(t.shape[0], parts, nH, -1)[groups.clamp_min(0)] * ok

    a, b = g(got), g(ref)
    num = (a - b).pow(2).sum((1, 4)).sqrt()
    den = b.pow(2).sum((1, 4)).sqrt()
    # a group whose reference is below 1 % of the tensor's RMS group norm is measured against that 1 %: there the
    # gradient is a cancellation (one key: dq = dk = 0 exactly; near one-hot rows) below the fp32 rounding of its terms
    floor = 1e-2 * float(den.pow(2).mean().sqrt())
    r = num / den.clamp_min(max(floor, 1e-30))
    return float((r if sel is None else r[:, sel]).max())


def out_groups(c):
    """[groups, n] output rows of each (sequence | window | image chunk) group (-1 absent)"""
    if c.fam in ("mhsa", "vd"):
        return torch.arange(c.B * c.L).view(c.B, c.L)
    if c.fam == "win":
        return win_maps(c)[1]
    N = 1 + c.nx * c.ny
    slots = sc_slots(c)
    b = torch.arange(c.B)[:, None, None] * N
    chunks = torch.where(slots[None] >= 0, b + 1 + slots[None], -1).reshape(-1, W2)
    glob = F.pad((torch.arange(c.B) * N)[:, None], (0, W2 - 1), value=-1)
    return torch.cat([chunks, glob])


def grad_groups(c):
    """[groups, n] dqkv rows of each sequence | window (window mode: every padded-map row) | image"""
    if c.fam == "win":
        return win_maps(c)[0]
    n = rows_of(c) // c.B
    return torch.arange(c.B * n).view(c.B, n)


def errors(c, got, ref, regime="normal", ref_D=None):
    """every metric of GATES, of kernel results `got` against the reference `ref`; ref_D: the reference with D taken
    from the kernel's O (large logits)"""
    e = dict(out=_rel(got["out"], ref["out"]),
             out_seq=_per_group(got["out"], ref["out"], out_groups(c), 1, c.nH),
             lse=float((got["lse"].double() - ref["lse"].to(got["lse"].device)).abs().max()),
             dqkv=_rel(got["dqkv"], ref["dqkv"]),
             dqkv_seq=_per_group(got["dqkv"], ref["dqkv"], grad_groups(c), 3, c.nH))
    if "lse_g" in ref:
        e["lse"] = max(e["lse"], float((got["lse_g"].double() - ref["lse_g"].to(got["lse"].device)).abs().max()))
    for k in ("dbias", "dbias_g"):
        if k in ref:
            for sfx, r in (("", ref), ("_D", ref_D)):
                if r is not None:
                    a, b = got[k].double(), r[k].to(got[k].device)
                    e[k + sfx] = _rel(a, b)
                    e[k + "_head" + sfx] = max(_rel(a[h], b[h]) for h in range(c.nH))
    if ref_D is not None:
        G = grad_groups(c)
        e["dv_seq"] = _per_group(got["dqkv"], ref["dqkv"], G, 3, c.nH, sel=slice(2, 3))
        e["dqk_seq_D"] = _per_group(got["dqkv"], ref_D["dqkv"], G, 3, c.nH, sel=slice(0, 2))
    return e


def failures(c, err, regime):
    gates = GATES[c.fam][gate_class(regime)]
    return {k: (err[k], g) for k, g in gates.items() if not err[k] < g}


def _seed(name):
    return sum(ord(ch) * 31 ** i for i, ch in enumerate(name)) % (1 << 31)


def _fmt(err):
    return " ".join(f"{k} {v:.2e}" for k, v in err.items())


# ================================ 1. the reference (CPU) ===============================================================
def _pin(a, b, what, tol=1e-12):
    """max |a - b| relative to max |b| (absolute where b is exactly 0: one key, whose softmax gradient vanishes)"""
    a, b = a.detach(), b.detach()
    den = float(b.abs().max())
    e = float((a - b).abs().max()) / (den if den > 0 else 1.0)
    assert e < tol, (what, e)


@pytest.mark.parametrize("L,nH", [(1, 2), (37, 3), (65, 2), (130, 1)])
def test_mhsa_reference_is_the_oracle_vit_attention(L, nH):
    """ref_mhsa on the qkv Linear's output against float64 autograd of oracle.vit.attention (identity proj)"""
    from oracle import vit as V
    g = torch.Generator().manual_seed(L * 10 + nH)
    B, C = 2, 64 * nH
    x = torch.randn(B, L, C, generator=g, dtype=F64).requires_grad_()
    wq = (torch.randn(3 * C, C, generator=g, dtype=F64) * C ** -0.5).requires_grad_()
    bq = torch.randn(3 * C, generator=g, dtype=F64).requires_grad_()
    sd = {"a.qkv.weight": wq, "a.qkv.bias": bq, "a.proj.weight": torch.eye(C, dtype=F64),
          "a.proj.bias": torch.zeros(C, dtype=F64)}
    dout = torch.randn(B, L, C, generator=g, dtype=F64)
    o = V.attention(sd, "a.", x, nH)
    dx, dbq = torch.autograd.grad(o, (x, bq), dout)
    c = mhsa(B, L, C, nH)
    ins = dict(qkv=F.linear(x, wq, bq).detach().reshape(B * L, 3 * C), dout=dout.reshape(B * L, C))
    r = ref_mhsa(c._replace(scale=0.125), ins)
    _pin(r["out"], o.reshape(B * L, C), "out")
    _pin((r["dqkv"] @ wq.detach()).view(B, L, C), dx, "dx")
    _pin(r["dqkv"].sum(0), dbq, "dbias")
    s = ins["qkv"].view(B, L, 3, nH, 64)
    _pin(r["lse"], torch.logsumexp(torch.einsum("bqhd,bkhd->bhqk", s[:, :, 0], s[:, :, 1]) * 0.125, -1), "lse")
    _pin(r["D"], (dout.view(B, L, nH, 64) * o.detach().view(B, L, nH, 64)).sum(-1).transpose(1, 2), "D")


def _cvt_attention_lines(t, B, C, H, W, w, heads, hd):
    """the attention lines of oracle.cvt.attention after the qkv projection (t [B, 3C, Hp, Wp], the padded map's pw
    output), with the head dim a parameter (the oracle writes 64)"""
    Hp, Wp = t.shape[-2:]
    sx, sy = Hp // w, Wp // w
    q, k, v = t.chunk(3, dim=1)

    def part(u):
        u = u.reshape(B, heads, hd, sx, w, sy, w).permute(0, 3, 5, 1, 4, 6, 2)
        return u.reshape(B * sx * sy, heads, w * w, hd)

    q, k, v = part(q), part(k), part(v)
    attn = (q @ k.transpose(-1, -2) * C ** -0.5).softmax(dim=-1)
    o = (attn @ v).reshape(B, sx, sy, heads, w, w, hd).permute(0, 3, 6, 1, 4, 2, 5).reshape(B, C, Hp, Wp)
    return o[:, :, :H, :W]


@pytest.mark.parametrize("H,W,w,nH,hd", [(10, 10, 7, 2, 64), (9, 13, 6, 1, 64), (7, 7, 7, 1, 64), (11, 5, 3, 2, 32),
                                         (16, 9, 8, 3, 32)])
def test_window_reference_is_the_oracle_cvt_attention(H, W, w, nH, hd):
    """ref_win on a padded map against float64 autograd of oracle.cvt.attention (head dim 64: the oracle itself, with
    an identity depthwise kernel, eval BatchNorm and identity proj_out; head dim 32: its attention lines, written for
    any head dim).  Padded rows of the qkv map are the pw bias (zero activations), so the pw bias gradient holds the
    padded rows' share, and padded query rows' dq is 0."""
    from oracle import cvt as CV
    g = torch.Generator().manual_seed(H * 100 + W * 10 + w)
    B, C = 2, nH * hd
    Hp, Wp = _pad(H, w), _pad(W, w)
    x = torch.randn(B, C, H, W, generator=g, dtype=F64).requires_grad_()
    wp = (torch.randn(3 * C, C, generator=g, dtype=F64) * C ** -0.5).requires_grad_()
    bp = torch.randn(3 * C, generator=g, dtype=F64).requires_grad_()
    dout = torch.randn(B, C, H, W, generator=g, dtype=F64)
    bn = (1 + CV.BN_EPS) ** -0.5
    if hd == 64:
        dw = torch.zeros(C, 1, 3, 3, dtype=F64)
        dw[:, 0, 1, 1] = 1.0
        sd = {"a.qkv.dw.weight": dw, "a.qkv.bn.weight": torch.ones(C, dtype=F64),
              "a.qkv.bn.bias": torch.zeros(C, dtype=F64), "a.qkv.pw.weight": wp.view(3 * C, C, 1, 1),
              "a.qkv.pw.bias": bp, "a.proj_out.weight": torch.eye(C, dtype=F64).view(C, C, 1, 1),
              "a.proj_out.bias": torch.zeros(C, dtype=F64)}
        bufs = {"a.qkv.bn.running_mean": torch.zeros(C, dtype=F64), "a.qkv.bn.running_var": torch.ones(C, dtype=F64),
                "a.qkv.bn.num_batches_tracked": torch.zeros((), dtype=torch.long)}
        o = CV.attention(sd, bufs, "a.", x, nH, w, False)
    else:
        t = F.conv2d(F.pad(x, (0, Wp - W, 0, Hp - H)) * bn, wp.view(3 * C, C, 1, 1), bp)
        o = _cvt_attention_lines(t, B, C, H, W, w, nH, hd)
    dx, dbp = torch.autograd.grad(o, (x, bp), dout)
    qkv = F.conv2d(F.pad(x.detach(), (0, Wp - W, 0, Hp - H)) * bn, wp.detach().view(3 * C, C, 1, 1), bp.detach())
    c = win(B, H, W, w, C, nH)._replace(scale=C ** -0.5)
    ins = dict(qkv=qkv.permute(0, 2, 3, 1).reshape(-1, 3 * C), dout=dout.permute(0, 2, 3, 1).reshape(-1, C))
    r = ref_win(c, ins)
    _pin(r["out"], o.permute(0, 2, 3, 1).reshape(-1, C), "out")
    dxp = (r["dqkv"] @ wp.detach() * bn).view(B, Hp, Wp, C)[:, :H, :W].permute(0, 3, 1, 2)
    _pin(dxp, dx, "dx")
    _pin(r["dqkv"].sum(0), dbp, "dbias")
    prow, crow = win_maps(c)
    pad = crow < 0
    assert r["lse"].shape == (prow.shape[0], nH, w * w) and torch.isfinite(r["lse"]).all()
    assert (r["dqkv"][prow[pad], :C] == 0).all() and (r["D"].transpose(1, 2)[pad] == 0).all()
    if pad.any():  # padded keys take part: the padded rows' k / v gradients are non-zero
        assert r["dqkv"][prow[pad], C:].abs().amax() > 1e-3


def _sc_sd(g, C, nH, N):
    """the sliding-chunk state of oracle.vil.sc_attention: one table entry per (query slot, key column), so the
    table's gradient is the local bias gradient itself"""
    from oracle import vil as VL
    n_cols = 9 * W2
    return {"a.query.weight": (torch.randn(C, C, generator=g, dtype=F64) * C ** -0.5).requires_grad_(),
            "a.query.bias": torch.randn(C, generator=g, dtype=F64),
            "a.kv.weight": (torch.randn(2 * C, C, generator=g, dtype=F64) * C ** -0.5).requires_grad_(),
            "a.kv.bias": torch.randn(2 * C, generator=g, dtype=F64),
            "a.local_relative_position_bias_table": torch.randn(W2 * n_cols, nH, generator=g,
                                                                dtype=F64).requires_grad_(),
            "a.relative_position_index": torch.arange(W2 * n_cols).view(W2, n_cols),
            "a.g2l_relative_position_bias": torch.randn(2, nH, 1, generator=g, dtype=F64).requires_grad_(),
            "a.g2g_relative_position_bias": torch.randn(nH, 1, 1, generator=g, dtype=F64).requires_grad_(),
            "a.proj.weight": torch.eye(C, dtype=F64), "a.proj.bias": torch.zeros(C, dtype=F64)}, VL


@pytest.mark.parametrize("nx,ny,mode", [(10, 9, 0), (10, 9, 3), (10, 9, 7), (7, 7, -1), (4, 12, 5), (15, 8, 0)])
def test_sliding_chunk_reference_is_the_oracle_vil_attention(nx, ny, mode):
    """ref_sc against float64 autograd of oracle.vil.sc_attention (out, dx, the table / g2l / g2g gradients) and of
    oracle.vil_attn.dense_attention with the bias and global-row bias as leaves (every dbias / dbias_g element)"""
    g = torch.Generator().manual_seed(nx * 100 + ny * 10 + mode + 1)
    B, nH = 2, 2
    C, N = 32 * nH, 1 + nx * ny
    sd, VL = _sc_sd(g, C, nH, N)
    x = torch.randn(B, N, C, generator=g, dtype=F64).requires_grad_()
    dout = torch.randn(B, N, C, generator=g, dtype=F64)
    o = VL.sc_attention(sd, "a.", x, nx, ny, nH, mode)
    tab, g2l, g2g = (sd["a." + k] for k in ("local_relative_position_bias_table", "g2l_relative_position_bias",
                                              "g2g_relative_position_bias"))
    dx, dtab, dg2l, dg2g = torch.autograd.grad(o, (x, tab, g2l, g2g), dout)
    wq, wkv = sd["a.query.weight"].detach(), sd["a.kv.weight"].detach()
    bias = torch.cat([g2l[1][:, :, None].expand(nH, W2, 1), tab.view(W2, 9 * W2, nH).permute(2, 0, 1)], -1).detach()
    bias_g = torch.cat([g2g[:, 0, :], g2l[0].expand(nH, N - 1)], -1).detach()
    ins = dict(q=F.linear(x, wq, sd["a.query.bias"]).detach().reshape(B * N, C),
               kv=F.linear(x, wkv, sd["a.kv.bias"]).detach().reshape(B * N, 2 * C), bias=bias, bias_g=bias_g,
               dout=dout.reshape(B * N, C))
    c = sc(B, nx, ny, nH)._replace(scale=VIL_SCALE)
    r = ref_sc(c, ins, mode)
    _pin(r["out"], o.reshape(B * N, C), "out")
    _pin((r["dqkv"][:, :C] @ wq + r["dqkv"][:, C:] @ wkv).view(B, N, C), dx, "dx")
    _pin(r["dbias"][:, :, 1:].permute(1, 2, 0).reshape(-1, nH), dtab, "dtable")
    _pin(r["dbias"][:, :, 0].sum(1), dg2l[1, :, 0], "dg2l[1]")
    _pin(r["dbias_g"][:, 1:].sum(1), dg2l[0, :, 0], "dg2l[0]")
    _pin(r["dbias_g"][:, 0], dg2g[:, 0, 0], "dg2g")
    # every element: dense_attention with the biases as leaves
    bl, bgl = bias.clone().requires_grad_(), bias_g.clone().requires_grad_()
    o2 = VA.dense_attention(ins["q"], ins["kv"], bl, bgl, VA.dense_index(nx, ny, mode), B, N, nH, VIL_SCALE)
    db, dbg = torch.autograd.grad(o2, (bl, bgl), ins["dout"])
    _pin(r["dbias"], db, "dbias")
    _pin(r["dbias_g"], dbg, "dbias_g")
    skipped = ~sc_key_columns(c, mode).any(0)
    assert (r["dbias"][:, :, skipped] == 0).all()
    # lse: each real token's row of the masked N x N scores; padded slots the bias of the columns their chunk reads
    s = ins["q"].view(B, N, nH, 32).transpose(1, 2) @ ins["kv"][:, :C].reshape(B, N, nH, 32).permute(0, 2, 3, 1)
    loc = bias.reshape(nH, -1)[:, VA.dense_index(nx, ny, mode).clamp_min(0)]
    loc = loc.masked_fill((VA.dense_index(nx, ny, mode) < 0)[None], -INF)
    full = torch.logsumexp(s * VIL_SCALE + torch.cat([bias_g[:, None], loc], 1)[None], -1)
    _pin(r["lse_g"], full[:, :, 0], "lse_g")
    slots = sc_slots(c)
    _pin(r["lse"][:, :, slots >= 0], full[:, :, 1 + slots[slots >= 0]], "lse")
    assert torch.isfinite(r["lse"]).all() and r["lse"].shape == (B, nH, slots.shape[0], W2)


@pytest.mark.parametrize("L0,nglo", [(7, 1), (3, 0), (6, 1), (1, 0)])
def test_dense_reference_is_the_oracle_vil_full_attention(L0, nglo):
    """ref_vd against float64 autograd of oracle.vil.full_attention (one table entry per (query, key) of the map)"""
    from oracle import vil as VL
    g = torch.Generator().manual_seed(L0 * 10 + nglo)
    B, nH = 3, 2
    C, npatch = 32 * nH, L0 * L0
    L = npatch + nglo
    x = torch.randn(B, L, C, generator=g, dtype=F64).requires_grad_()
    wq = (torch.randn(3 * C, C, generator=g, dtype=F64) * C ** -0.5).requires_grad_()
    bq = torch.randn(3 * C, generator=g, dtype=F64)
    tab = torch.randn(npatch * npatch, nH, generator=g, dtype=F64).requires_grad_()
    g2l = torch.randn(2, nH, 1, generator=g, dtype=F64).requires_grad_()
    g2g = torch.randn(nH, 1, 1, generator=g, dtype=F64).requires_grad_()
    sd = {"a.qkv.weight": wq, "a.qkv.bias": bq, "a.relative_position_index": torch.arange(npatch * npatch).view(
        npatch, npatch), "a.local_relative_position_bias_table": tab, "a.g2l_relative_position_bias": g2l,
        "a.g2g_relative_position_bias": g2g, "a.proj.weight": torch.eye(C, dtype=F64),
        "a.proj.bias": torch.zeros(C, dtype=F64)}
    dout = torch.randn(B, L, C, generator=g, dtype=F64)
    o = VL.full_attention(sd, "a.", x, nH, nglo)
    dx, dtab, dg2l, dg2g = torch.autograd.grad(o, (x, tab, g2l, g2g), dout, allow_unused=True)
    bias = tab.detach().view(npatch, npatch, nH).permute(2, 0, 1)
    if nglo:
        top = torch.cat([g2g, g2l[0].unsqueeze(-1).expand(-1, -1, npatch)], -1)
        bias = torch.cat([top, torch.cat([g2l[1].unsqueeze(1).expand(-1, npatch, -1), bias], -1)], 1).detach()
    ins = dict(qkv=F.linear(x, wq, bq).detach().reshape(B * L, 3 * C), bias=bias, dout=dout.reshape(B * L, C))
    c = vd(B, L, C, nH)._replace(scale=VIL_SCALE)
    r = ref_vd(c, ins)
    _pin(r["out"], o.reshape(B * L, C), "out")
    _pin((r["dqkv"] @ wq.detach()).view(B, L, C), dx, "dx")
    _pin(r["dbias"][:, nglo:, nglo:].permute(1, 2, 0).reshape(-1, nH), dtab, "dtable")
    if nglo:
        _pin(r["dbias"][:, 0, 0], dg2g[:, 0, 0], "dg2g")
        _pin(r["dbias"][:, 0, 1:].sum(-1), dg2l[0, :, 0], "dg2l[0]")
        _pin(r["dbias"][:, 1:, 0].sum(-1), dg2l[1, :, 0], "dg2l[1]")


@pytest.mark.parametrize("name", ["mhsa_B2_L129_C192_h3", "win_B2_30x17_w14_C128_h4", "sc_B2_10x17_h3",
                                  "vd_B2_L9_C768_h24"])
def test_regimes_do_what_they_say(name):
    """late: the maximum score of most rows sits on the last key / in a later ViL tile; uniform: the softmax is exactly
    uniform, so lse = log(key count)"""
    c = SYNTHETIC[name]
    for mode in modes_for(c, "late")[:3] if c.fam == "sc" else (None,):
        late = make_inputs(c, "late", "cpu", 1, mode)
        uni = make_inputs(c, "uniform", "cpu", 2, mode)
        ru = reference(c, uni, mode)
        if c.fam == "sc":
            cols = sc_key_columns(c, mode).sum(1).double()  # keys per chunk
            assert torch.allclose(ru["lse"], cols.log()[None, None, :, None].expand_as(ru["lse"]), atol=1e-12)
            assert torch.allclose(ru["lse_g"], torch.full_like(ru["lse_g"], math.log(1 + c.nx * c.ny)), atol=1e-12)
            if mode != -1:  # the later tiles' bias is 5 above the own chunk's
                assert late["bias"][:, :, 1 + 8 * W2:].mean() > late["bias"][:, :, 1 + 4 * W2:1 + 5 * W2].mean() + 4
            continue
        L = c.w * c.w if c.fam == "win" else c.L
        assert torch.allclose(ru["lse"], torch.full_like(ru["lse"], math.log(L)), atol=1e-12)
        q, k, _ = _heads(late["qkv"][:rows_of(c)], 1, rows_of(c), 3, c.nH)
        if c.fam == "win":
            prow = win_maps(c)[0]
            s = q[0][:, prow] @ k[0][:, prow].transpose(-1, -2)
        else:
            s = (q[0].view(c.nH, c.B, c.L, -1) @ k[0].view(c.nH, c.B, c.L, -1).transpose(-1, -2))
            if c.fam == "vd":
                s = s * c.scale + late["bias"][:, None].double()
        assert (s.argmax(-1) == L - 1).double().mean() > 0.5


# each bug must move the reference by >= 5x the gate of the metric named, on the GPU case, regime and mode named
SENSITIVITY = [
    ("keys_past_L_zero", "mhsa_B2_L65_C192_h3", "normal", None, "out"),
    ("keys_past_L_zero", "mhsa_B16_L37_C384_h6", "normal", None, "out"),
    ("keys_past_L_zero", "mhsa_B2_L129_C768_h12", "normal", None, "out_seq"),
    ("no_rescale", "mhsa_B2_L129_C192_h3", "late", None, "out"),
    ("no_rescale", "mhsa_B2_L65_C768_h12", "late", None, "lse"),
    ("lse_log2", "mhsa_B2_L65_C192_h3", "normal", None, "lse"),
    ("kv_head_xor1", "mhsa_B2_L64_C192_h3", "normal", None, "out_seq"),
    ("dk_no_scale", "mhsa_B2_L63_C768_h12", "normal", None, "dqkv_seq"),
    ("prep_head_pairs", "win_B2_12x12_w12_C256_h8", "normal", None, "dqkv_seq"),
    ("prep_head_pairs", "win_B2_26x13_w12_C96_h3", "normal", None, "dqkv_seq"),
    ("pad_keys_masked", "win_B2_30x17_w7_C192_h3", "normal", None, "out_seq"),
    ("pad_keys_masked", "win_B2_17x30_w14_C64_h1", "normal", None, "out_seq"),
    ("scale_hd", "win_B2_7x7_w7_C192_h3", "normal", None, "out"),
    ("scale_hd", "win_B2_30x17_w14_C128_h4", "normal", None, "out"),
    ("win_transposed", "win_B2_30x17_w7_C192_h3", "normal", None, "out"),
    ("win_transposed", "win_B2_17x30_w14_C64_h1", "normal", None, "out"),
    ("keys_past_L_zero", "win_B2_7x7_w7_C192_h3", "normal", None, "out"),
    ("chunk_mirrored", "sc_B2_10x17_h3", "normal", 2, "out_seq"),
    ("chunk_mirrored", "sc_B3_16x9_h6", "normal", 6, "out_seq"),
    ("no_global_bias", "sc_B2_10x17_h3", "normal", 0, "out"),
    ("no_global_bias", "sc_B2_3x5_h3", "normal", -1, "out"),
    ("bias_g_shift", "sc_B2_10x17_h3", "normal", 0, "out_seq"),
    ("bias_g_shift", "sc_B3_16x9_h6", "normal", 4, "dbias_g_head"),
    ("lse_log2", "sc_B3_16x9_h6", "normal", 1, "lse"),
    ("bias_transposed", "vd_B2_L9_C768_h24", "normal", None, "out"),
    ("bias_transposed", "vd_B17_L49_C192_h6", "normal", None, "out"),
    ("dbias_one_part", "vd_B17_L49_C192_h6", "normal", None, "dbias"),
    ("dbias_one_part", "vd_B33_L37_C384_h12", "normal", None, "dbias_head"),
]


def _all_cases():
    d = dict(table_cases())
    d.update(SYNTHETIC)
    return d


@pytest.mark.parametrize("bug,name,regime,mode,metric", SENSITIVITY)
def test_gates_see_plausible_kernel_bugs(bug, name, regime, mode, metric):
    c = _all_cases()[name]
    ins = make_inputs(c, regime, "cpu", _seed(name + regime), mode)
    good = reference(c, ins, mode)
    bad = reference(c, ins, mode, bug)
    assert all(torch.isfinite(t).all() for t in bad.values())
    err = errors(c, bad, good)[metric]
    gate = GATES[c.fam][gate_class(regime)][metric]
    print(f"sensitivity {bug} on {name} ({regime}, mode {mode}): {metric} {err:.3e} = {err / gate:.1f}x gate")
    assert err >= 5 * gate, (bug, name, metric, err, gate)


def test_table_and_synthetic_entries_cover_the_kernels():
    """TABLE holds the nine backbones, each with a fwd and a bwd launch per geometry; the synthetic entries hold the
    edges the kernels branch on"""
    assert set(TABLE) == {"deit_tiny_p16", "deit_small_p16", "deit_small_p8", "vit_base_p16", "cvt_13", "cvt_13_w14",
                          "cvt_s3", "cvt_s3_w14", "vil_2262"}
    for arch, ents in TABLE.items():
        for e in ents:
            fam, d = e[0].rsplit("_", 1)
            assert (fam, d) in ENTRY.values()
            twin = "bwd" if d == "fwd" else "fwd"
            assert any(x[0] == f"{fam}_{twin}" and x[1:] == e[1:] for x in ents), (arch, e)
    syn = list(SYNTHETIC.values())
    assert {c.L for c in syn if c.fam == "mhsa"} >= {1, 63, 64, 65, 128, 129, 256}
    assert {c.nH for c in syn if c.fam == "mhsa"} >= {3, 12}
    assert {c.w for c in syn if c.fam == "win"} >= {1, 3, 6, 7, 12, 14}
    assert any(c.fam == "win" and c.w == c.H for c in syn)
    assert {hd_of(c) for c in syn if c.fam == "win"} == {32, 64}
    assert any(c.fam == "win" and c.H % c.w and c.W % c.w and c.H != c.W for c in syn)
    assert all(c.nx != c.ny and c.nx % 7 and c.ny % 7 for c in syn if c.fam == "sc")
    assert {c.L for c in syn if c.fam == "vd"} >= {1, 9, 256} and {c.B for c in syn if c.fam == "vd"} >= {17, 33}


# ================================ 2. the step's launches (GPU) =========================================================
def signature(name, a):
    """the TABLE tuple of one launch (name, ctypes arguments)"""
    fam, d = ENTRY[name]
    k = f"{fam}_{d}"
    if name == "esvit_mhsa_fwd":
        return (k, int(a[3]), int(a[4]), int(a[5]), int(a[6]), f32(float(a[7])))
    if name == "esvit_mhsa_bwd":
        return (k, int(a[6]), int(a[7]), int(a[8]), int(a[9]), f32(float(a[10])))
    if name == "esvit_mhsa_win_fwd":
        return (k, *(int(x) for x in a[3:9]), f32(float(a[9])))
    if name == "esvit_mhsa_win_bwd":
        return (k, *(int(x) for x in a[6:12]), f32(float(a[12])))
    if name == "esvit_vil_sc_fwd":
        return (k, *(int(x) for x in a[8:12]))
    if name == "esvit_vil_sc_bwd":
        return (k, *(int(x) for x in a[15:19]))
    if name == "esvit_vil_dense_fwd":
        return (k, *(int(x) for x in a[4:8]))
    return (k, *(int(x) for x in a[9:13]))


def record_arch(arch):
    """the set of TABLE tuples of the attention launches of the second eager B = 2 step of an arch (the first
    allocates)"""
    from bench import synthetic_crops
    from esvit_b200 import _lib, engine
    dev = torch.device("cuda:0")
    lr = 5e-4 * TABLE_B / 256.0
    step, student, teacher, _ = engine.make_step(arch=arch, out_dim=65536, ncrops=10, dense=True, device=dev, lr=lr,
                                                 ddp=False, optimizer="fused", cuda_graph=False)
    student.train()
    teacher.train()
    crops = [c.to(dev) for c in synthetic_crops(TABLE_B, 8, 0)]
    step(crops, 1, lr, 0.04, 0.996)
    seen = set()
    plain = _lib._plain_call

    def recording(name, *args):
        if name in ENTRY:
            seen.add(signature(name, args))
        return plain(name, *args)

    _lib._plain_call = recording
    try:
        step(crops, 1, lr, 0.04, 0.996)
        torch.cuda.synchronize()
    finally:
        _lib._plain_call = plain
    del step, student, teacher, crops
    torch.cuda.empty_cache()
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("arch", list(TABLE))
def test_table_matches_the_step(arch):
    """the step launches exactly the table's signatures: no launch outside the table, no table entry without one"""
    seen = record_arch(arch)
    table = set(TABLE[arch])
    print(f"table {arch}: {sorted(seen)}")
    assert not seen - table, ("launched, not in the table", sorted(seen - table))
    assert not table - seen, ("in the table, not launched", sorted(table - seen))


# ================================ 3. kernels against fp64 (GPU) ========================================================
def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    from esvit_b200 import _lib
    _lib.call(name, *args)


def buffers(c):
    """name -> (shape, dtype, row width) of every kernel output and workspace"""
    from esvit_b200 import _lib
    B, C, nH = c.B, c.C, c.nH
    if c.fam in ("mhsa", "vd"):
        L = c.L
        d = dict(out=((B * L, C), BF16, C), lse=((B, nH, L), F32, L), dvec=((B, nH, L), F32, L),
                 dqkv=((B * L, 3 * C), BF16, 3 * C))
        if c.fam == "vd":
            d["part"] = ((_lib.load().esvit_vil_dense_parts(B), nH, L, L), F32, L)
            d["dbias"] = ((nH, L, L), F32, L)
        return d
    if c.fam == "win":
        nw, L = win_maps(c)[0].shape
        return dict(out=((B * c.H * c.W, C), BF16, C), lse=((nw, nH, L), F32, L), dvec=((nw, nH, L), F32, L),
                    dqkv=((rows_of(c), 3 * C), BF16, 3 * C))
    N, nch = 1 + c.nx * c.ny, sc_slots(c).shape[0]
    ws = _lib.load().esvit_vil_sc_ws_floats(B, c.nx, c.ny, nH)
    return dict(out=((B * N, C), BF16, C), lse=((B, nH, nch, W2), F32, W2), lse_g=((B, nH), F32, nH),
                dvec=((B, nH, nch, W2), F32, W2), ws=((ws,), F32, 1), dq=((B * N, C), BF16, C),
                dkv=((B * N, 2 * C), BF16, 2 * C), dbias=((nH, W2, NB), F32, NB), dbias_g=((nH, N), F32, N))


def run(c, ins, mode=None, fill=math.nan, pad=0, bufs=None, fills=None):
    """the entry point's fwd then bwd through the C ABI.  Every output is allocated with `pad` rows past its end, all
    filled with `fill` (fills: per-buffer overrides); bufs: name -> caller-owned flat tensors to write into instead.
    Returns (outputs shaped as the contract, the rows past each end)."""
    dev = next(iter(ins.values())).device
    got, past = {}, {}
    for k, (shape, dt, row) in buffers(c).items():
        n = math.prod(shape)
        if bufs is not None and k in bufs:
            t = bufs[k]
        else:
            t = torch.full((n + pad * row,), (fills or {}).get(k, fill), dtype=dt, device=dev)
        got[k], past[k] = t[:n].view(shape), t[n:]
    P, S, s = _p, _stream(), c.scale
    B, C, nH = c.B, c.C, c.nH
    if c.fam == "mhsa":
        _call("esvit_mhsa_fwd", P(ins["qkv"]), P(got["out"]), P(got["lse"]), B, c.L, C, nH, s, S)
        _call("esvit_mhsa_bwd", P(ins["qkv"]), P(got["out"]), P(ins["dout"]), P(got["lse"]), P(got["dvec"]),
              P(got["dqkv"]), B, c.L, C, nH, s, S)
    elif c.fam == "win":
        geo = (B, c.H, c.W, c.w, C, nH, s, S)
        _call("esvit_mhsa_win_fwd", P(ins["qkv"]), P(got["out"]), P(got["lse"]), *geo)
        _call("esvit_mhsa_win_bwd", P(ins["qkv"]), P(got["out"]), P(ins["dout"]), P(got["lse"]), P(got["dvec"]),
              P(got["dqkv"]), *geo)
    elif c.fam == "sc":
        m = ins["mode"] if "mode" in ins else torch.tensor([mode], dtype=torch.int32, device=dev)
        geo = (B, c.nx, c.ny, nH, s, S)
        _call("esvit_vil_sc_fwd", P(ins["q"]), P(ins["kv"]), P(ins["bias"]), P(ins["bias_g"]), P(m), P(got["out"]),
              P(got["lse"]), P(got["lse_g"]), *geo)
        _call("esvit_vil_sc_bwd", P(ins["q"]), P(ins["kv"]), P(ins["bias"]), P(ins["bias_g"]), P(m), P(got["out"]),
              P(ins["dout"]), P(got["lse"]), P(got["lse_g"]), P(got["dvec"]), P(got["ws"]), P(got["dq"]),
              P(got["dkv"]), P(got["dbias"]), P(got["dbias_g"]), *geo)
        got["dqkv"] = torch.cat([got["dq"], got["dkv"]], 1)
    else:
        geo = (B, c.L, C, nH, s, S)
        _call("esvit_vil_dense_fwd", P(ins["qkv"]), P(ins["bias"]), P(got["out"]), P(got["lse"]), *geo)
        _call("esvit_vil_dense_bwd", P(ins["qkv"]), P(ins["bias"]), P(got["out"]), P(ins["dout"]), P(got["lse"]),
              P(got["dvec"]), P(got["part"]), P(got["dqkv"]), P(got["dbias"]), *geo)
    torch.cuda.synchronize()
    return got, past


def check(c, regime, mode=None, tag=""):
    dev = torch.device("cuda:0")
    name = name_of(c)
    ins = make_inputs(c, regime, dev, _seed(name + regime), 0 if mode is None else mode)
    got, _ = run(c, ins, mode)
    for k in ("out", "lse", "dqkv") + (("lse_g", "dbias", "dbias_g") if c.fam == "sc" else ("dbias",) if c.fam == "vd"
                                        else ()):
        assert torch.isfinite(got[k]).all(), (name, regime, mode, k)
    ref = reference(c, ins, mode)
    ref_D = reference(c, ins, mode, O=got["out"]) if gate_class(regime) == "peaked" else None
    err = errors(c, got, ref, regime, ref_D)
    if ref_D is not None:
        err["dqkv_seq_exact"] = err.pop("dqkv_seq")
    print(f"attn {tag}{regime} {name}" + ("" if mode is None else f" mode {mode}") + f": {_fmt(err)}")
    bad = failures(c, err, regime)
    assert not bad, (name, regime, mode, bad)
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("name", list(table_cases()) + list(SYNTHETIC))
def test_case_matches_fp64(name, regime):
    """a geometry of the step (B = 2) or a synthetic edge, under one input regime, every ViL mode it runs"""
    c = _all_cases()[name]
    for mode in modes_for(c, regime):
        check(c, regime, mode)
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(table_cases(BENCH_B // TABLE_B)))
def test_bench_batch_case_matches_fp64(name):
    """the step's geometries at the bench batch (B = 64): 512 local sequences, 128 ViT p8 sequences of 785 tokens,
    ViL dq segments of several images, 16 dense dq parts of several images each"""
    c = table_cases(BENCH_B // TABLE_B)[name]
    for mode in modes_for(c, "normal", bench=True):
        check(c, "normal", mode, "bench ")
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.xfail(strict=True, reason="the backward's D = rowsum(dO * O) uses the bf16 O; where a row is dominated "
                                       "by one key, its dq / dk are a cancellation that this rounding dominates "
                                       "(DESIGN.md §4.19)")
@pytest.mark.parametrize("name", ["mhsa_B16_L37_C384_h6", "win_B16_24x24_w7_C64_h1"])
def test_large_logit_dq_dk_per_sequence_against_exact_fp64(name):
    c = _all_cases()[name]
    ins = make_inputs(c, "large", torch.device("cuda:0"), _seed(name + "large"))
    got, _ = run(c, ins)
    err = errors(c, got, reference(c, ins))["dqkv_seq"]
    print(f"attn large {name}: dqkv_seq against exact fp64 {err:.2e}")
    assert err < GATES[c.fam]["normal"]["dqkv_seq"]


# ================================ 4. the C-ABI contract (GPU) ==========================================================
CONTRACT = ["mhsa_B4_L197_C384_h6", "mhsa_B2_L65_C192_h3", "win_B16_24x24_w14_C64_h1", "win_B2_30x17_w7_C192_h3",
            "win_B2_26x13_w12_C96_h3", "win_B3_9x20_w6_C160_h5", "sc_B2_10x17_h3", "sc_B16_12x12_h6",
            "vd_B17_L49_C192_h6", "vd_B4_L197_C384_h12"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", CONTRACT)
def test_contract(name):
    """NaN-prefilled outputs, lse, dvec, dqkv, dbias and workspaces come back finite wherever the contract defines
    them (window mode: dqkv over all B*Hp*Wp rows, padded rows' dq exactly 0; ViL: every lse slot of every edge
    chunk); sentinel rows past each buffer are untouched; ViL dbias / dbias_g are written, not accumulated (a prefill of
    3 gives the same bits) and 0 in the columns of skipped chunks; reruns are bit-identical"""
    c = _all_cases()[name]
    dev = torch.device("cuda:0")
    for mode in ((2, -1, 0) if c.fam == "sc" else (None,)):
        ins = make_inputs(c, "normal", dev, _seed(name), mode or 0)
        got, past = run(c, ins, mode, pad=PAD)
        for k, v in got.items():
            if k in ("ws", "part"):
                continue
            assert torch.isfinite(v).all(), (name, mode, k)
        if c.fam == "win":
            prow, crow = win_maps(c)
            pad_rows = prow[crow < 0].to(dev)
            assert (got["dqkv"][pad_rows, :c.C] == 0).all()
        _, past2 = run(c, ins, mode, fill=SENTINEL, pad=PAD)
        for k, v in past2.items():
            assert (v == SENTINEL).all(), (name, mode, k)
        again, _ = run(c, ins, mode, fill=3.0 if c.fam in ("sc", "vd") else math.nan)
        for k in got:
            if k not in ("ws", "part"):
                assert torch.equal(got[k], again[k]), (name, mode, k)
        if c.fam == "sc":
            skipped = ~sc_key_columns(c, mode).any(0).to(dev)
            unread = torch.ones(NB, dtype=torch.bool, device=dev)
            unread[0] = False
            for j in VA.mode_chunks(mode):
                unread[1 + j * W2:1 + (j + 1) * W2] = False
            assert skipped[unread].all()
            assert (got["dbias"][:, :, skipped] == 0).all()


def _offset_groups(cases, ins_list, mode=None):
    """run the cases back to back in shared input / output buffers (the way the resolution-group ops launch them, at
    pointer offsets) and return each case's outputs"""
    dev = torch.device("cuda:0")
    keys = list(ins_list[0])
    big_in = {k: torch.cat([i[k].reshape(-1) for i in ins_list]) for k in keys}
    views, o = [], {k: 0 for k in keys}
    for i in ins_list:
        v = {}
        for k in keys:
            n = i[k].numel()
            v[k] = big_in[k][o[k]:o[k] + n].view(i[k].shape)
            o[k] += n
        views.append(v)
    sizes = [buffers(c) for c in cases]
    big_out = {k: torch.full((sum(math.prod(s[k][0]) for s in sizes),), math.nan, dtype=sizes[0][k][1], device=dev)
               for k in sizes[0] if k not in ("ws", "part")}
    res, o = [], {k: 0 for k in big_out}
    for c, v, s in zip(cases, views, sizes):
        b = {}
        for k in big_out:
            n = math.prod(s[k][0])
            b[k] = big_out[k][o[k]:o[k] + n]
            o[k] += n
        res.append(run(c, v, mode, bufs=b)[0])
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("fam", ["mhsa", "win", "sc", "vd"])
def test_resolution_groups_equal_separate_calls(fam):
    """the global and local geometry of one step launched at pointer offsets into shared buffers (inputs and outputs)
    equal separate calls on their own buffers, bit for bit"""
    pairs = {"mhsa": ("mhsa_B4_L197_C384_h6", "mhsa_B16_L37_C384_h6"),
             "win": ("win_B4_28x28_w7_C192_h3", "win_B16_12x12_w7_C192_h3"),
             "sc": ("sc_B4_28x28_h6", "sc_B16_12x12_h6"),
             "vd": ("vd_B4_L197_C384_h12", "vd_B16_L37_C384_h12")}[fam]
    cases = [_all_cases()[n] for n in pairs]
    dev = torch.device("cuda:0")
    mode = 5 if fam == "sc" else None
    ins = [make_inputs(c, "normal", dev, _seed(name_of(c)), mode or 0) for c in cases]
    together = _offset_groups(cases, ins, mode)
    for c, i, t in zip(cases, ins, together):
        alone, _ = run(c, i, mode)
        for k in t:
            if k not in ("ws", "part"):
                assert torch.equal(t[k], alone[k]), (name_of(c), k)


@pytest.mark.gpu
def test_refusals():
    """arguments the host-side checks refuse return ESVIT_ERR_BAD_ARG (ValueError) and leave every NaN buffer
    untouched: C != nH*64 (whole sequence), a window head dim outside {32, 64}, w > min(H, W), ViL dense L > 256"""
    dev = torch.device("cuda:0")
    S = _stream()

    def nan(n, dt=F32):
        return torch.full((n,), math.nan, dtype=dt, device=dev)

    def refused(name, *args):
        with pytest.raises(ValueError):
            _call(name, *args)

    outs = []
    for B, L, C, nH in ((2, 8, 96, 1), (2, 8, 128, 1), (2, 8, 192, 2)):
        qkv, out, lse, dvec, dqkv = nan(B * L * 3 * C, BF16), nan(B * L * C, BF16), nan(B * nH * L), nan(
            B * nH * L), nan(B * L * 3 * C, BF16)
        refused("esvit_mhsa_fwd", _p(qkv), _p(out), _p(lse), B, L, C, nH, 0.125, S)
        refused("esvit_mhsa_bwd", _p(qkv), _p(out), _p(out), _p(lse), _p(dvec), _p(dqkv), B, L, C, nH, 0.125, S)
        outs += [out, lse, dvec, dqkv]
    for B, H, W, w, C, nH in ((2, 8, 8, 7, 48, 1), (2, 8, 8, 7, 256, 2), (2, 8, 8, 7, 16, 1), (2, 5, 9, 6, 64, 2),
                              (2, 9, 5, 7, 64, 1), (2, 6, 6, 7, 128, 4)):
        Hp, Wp = _pad(H, w), _pad(W, w)
        n = B * Hp * Wp
        qkv, out, lse, dvec, dqkv = nan(n * 3 * C, BF16), nan(B * H * W * C, BF16), nan(n * nH), nan(n * nH), nan(
            n * 3 * C, BF16)
        refused("esvit_mhsa_win_fwd", _p(qkv), _p(out), _p(lse), B, H, W, w, C, nH, C ** -0.5, S)
        refused("esvit_mhsa_win_bwd", _p(qkv), _p(out), _p(out), _p(lse), _p(dvec), _p(dqkv), B, H, W, w, C, nH,
                C ** -0.5, S)
        outs += [out, lse, dvec, dqkv]
    for B, L, C, nH in ((2, 257, 96, 3), (1, 400, 32, 1)):
        qkv, bias, out, lse, dvec = nan(B * L * 3 * C, BF16), nan(nH * L * L), nan(B * L * C, BF16), nan(
            B * nH * L), nan(B * nH * L)
        part, dqkv, dbias = nan(min(B, 16) * nH * L * L), nan(B * L * 3 * C, BF16), nan(nH * L * L)
        refused("esvit_vil_dense_fwd", _p(qkv), _p(bias), _p(out), _p(lse), B, L, C, nH, VIL_SCALE, S)
        refused("esvit_vil_dense_bwd", _p(qkv), _p(bias), _p(out), _p(out), _p(lse), _p(dvec), _p(part), _p(dqkv),
                _p(dbias), B, L, C, nH, VIL_SCALE, S)
        outs += [out, lse, dvec, part, dqkv, dbias]
    torch.cuda.synchronize()
    for t in outs:
        assert torch.isnan(t.float()).all()
