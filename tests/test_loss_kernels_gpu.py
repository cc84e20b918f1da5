"""The DINO / DDINO loss kernels (csrc/loss.cu) against an fp64 reference of their C-ABI contract, at the loss
geometries of the step (the cls term, and the region terms of Swin / CvT / ViL, ViT p16 and ViT p8 at B = 64, 2 + 8
crops), at K from 8 to 65 536, and in the input regimes training meets: normalised heads, wide logits, a near-one-hot
teacher, the uniform teacher of a collapsed run, a large center and a teacher whose mass reaches below the stored-q
flush threshold, over the teacher-temperature warm-up.  Both CE paths run every case: the default one on teacher
probabilities stored once per row (esvit_row_softmax_q, esvit_dino_ce_q_fwd / _bwd) and the ESVIT_CE_Q=0 one that
recomputes them per pairing (esvit_row_lse, esvit_dino_ce_fwd / _bwd); then esvit_weighted_sum, esvit_colsum and
esvit_center_ema.  Every output is NaN-prefilled, so an element that is never written fails.

The reference (CPU tests, not `gpu`-marked) is pinned to a float64 run of `oracle.losses.dino_loss` / `ddino_loss`, and
each plausible kernel bug of a list below is shown to move the reference by at least 5x the gate the GPU test uses."""
import math
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import losses as OL

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
NCROPS = 10                       # 2 global + 8 local crops
N_TERMS = 2 * NCROPS - 2
STUDENT_TEMP = 0.1
Q_SCALE = 4096.0                  # stored teacher probabilities: fp16 q * 2^12
Q12_NORMAL = 2.0 ** -14           # q12 below this (q < 2^-26 = 1.5e-8) is an fp16 subnormal: the flush threshold
LN2 = math.log(2.0)

# Gates per CE path ("q": stored teacher probabilities, "lse": ESVIT_CE_Q=0) and input regime, at about 3x the largest
# error measured on an H100 over every case of the regime (DESIGN.md §4.16 has the measured maxima):
#   lse / lse_s: max |lse - ref| of the teacher / student log-sum-exp (natural log)
#   row_loss: max over rows of |row_loss - ref| / (n_r |lse_s| + |<q, s~>|)
#   ds_row / ds: largest per-row and global rel-L2 of the logit gradient
#   loss: |loss - ref| / sum_r |w_r row_loss_r|
# On the "q" path the CE kernels are measured against the reference on the kernel's own stored q12.  The lse path's
# wide / one-hot ds_row is where a student row puts its softmax peak on the teacher's near-one-hot column: there ds is a
# cancellation n p - q that the fp32 exponent of the recomputed q (|t~| up to 750) dominates.
_G = ("lse", "lse_s", "row_loss", "ds_row", "ds", "loss")
GATES = {
    "q": {
        "normalised": dict(zip(_G, (6e-6, 3.5e-6, 6e-7, 1.2e-2, 5e-3, 2.5e-7))),
        "wide": dict(zip(_G, (1.6e-4, 5e-5, 5e-7, 1e-2, 5e-3, 4e-7))),
        "onehot": dict(zip(_G, (3e-4, 1.8e-5, 4e-7, 1e-2, 5e-3, 2.5e-7))),
        "uniform": dict(zip(_G, (3e-7, 1.8e-5, 5e-7, 1.2e-2, 5.5e-3, 2e-7))),
        "large_center": dict(zip(_G, (2e-5, 1e-4, 5e-7, 1.1e-2, 5.5e-3, 3.5e-6))),
        "tail": dict(zip(_G, (2e-6, 1.8e-5, 5e-7, 1.1e-2, 5e-3, 2e-7))),
    },
    "lse": {
        "normalised": dict(zip(_G, (3e-6, 3e-6, 1e-6, 1.2e-2, 5e-3, 3.5e-7))),
        "wide": dict(zip(_G, (1e-4, 2.5e-5, 3e-5, 4e-2, 5e-3, 4e-7))),
        "onehot": dict(zip(_G, (1.5e-4, 6.5e-6, 4.5e-5, 2.1e-2, 5e-3, 5e-7))),
        "uniform": dict(zip(_G, (3e-7, 6.5e-6, 3.5e-7, 1.2e-2, 5.5e-3, 2e-7))),
        "large_center": dict(zip(_G, (1.5e-5, 1e-4, 7e-6, 1.1e-2, 5.5e-3, 5e-6))),
        "tail": dict(zip(_G, (4e-6, 6.5e-6, 7e-7, 1.1e-2, 5e-3, 2.5e-7))),
    },
}
COLSUM = 6e-8  # max over columns of |colsum - ref| / sum_r |t_rk|
# Two gates of the "q" path follow from the stored format, not from a measurement: every stored q12 within Q12_ULP fp16
# ulp of the exact 2^12 q (0 allowed below the flush threshold), and at most FLUSHED of a row's probability mass lost
# below it.
Q12_ULP = 1.0
FLUSHED = 1e-3

Case = namedtuple("Case", "geom K regime temp gscale B")

# region geometry (Tg, Tl) per backbone: tokens of a 224² global / 96² local crop after the last stage.  CvT-13 (s1, s3
# and their window-14 specs) and ViL 2262 end at stride 32 like Swin, s_npatch [49, 9] (tests/test_cvt_oracle.py,
# tests/test_vil_oracle.py): the Swin table is theirs.
GEOMS = {"cls": None, "swin": (49, 9), "vit16": (196, 36), "vit8": (784, 144)}
REGIMES = ("normalised", "wide", "onehot", "uniform", "large_center", "tail")
TEMPS = (0.04, 0.0555, 0.07)      # the teacher-temperature warm-up 0.04 -> 0.07
GSCALES = (1.0, 2.0, 2.0 ** -16, 0.0)
ALL_K = (8, 384, 1000, 4096, 65528, 65536)
# (ViT rows past 2^31 elements at K = 65 536: test_vit_gpu.py::test_head_and_loss_kernels_past_2_pow_31_elements)
VIT_K = (8, 384, 1000, 4096)


def _name(c):
    return f"{c.geom}_k{c.K}_{c.regime}_t{c.temp}_g{c.gscale:g}"


CASES = {}


def _add(geom, K, regime="normalised", temp=0.04, gscale=1.0, B=64):
    c = Case(geom, K, regime, temp, gscale, B)
    CASES[_name(c)] = c


for _g, _ks in (("cls", ALL_K), ("swin", ALL_K), ("vit16", VIT_K), ("vit8", VIT_K)):
    for _k in _ks:
        _add(_g, _k)
for _i, (_r, _t) in enumerate((r, t) for r in REGIMES for t in TEMPS):
    _add("cls", 65536, _r, _t, GSCALES[_i % 4])                       # every regime through the warm-up, real K
for _i, _r in enumerate(REGIMES):
    _add("swin", 65536, _r, TEMPS[_i % 3], GSCALES[(_i + 1) % 4])     # ... and on the 10 880 region rows
    if _r != "tail":                                                  # (no mass below 1.5e-8 fits in 1000 entries)
        _add("cls", 1000, _r, TEMPS[(_i + 1) % 3], GSCALES[(_i + 2) % 4])
_add("swin", 65528, "tail", 0.07)
for _gs in GSCALES[1:]:
    _add("cls", 4096, gscale=_gs)


def f32(x):
    """the fp32 value a Python float becomes at the C ABI (c_float)"""
    return float(np.float32(x))


# ================================ the fp64 reference ===================================================================
def ref_teacher(t, center, inv_temp_t, bug=None):
    """teacher rows: natural-log LSE of (t - center) * inv_temp, q = softmax, q12 = 2^12 q exactly and its fp16
    rounding"""
    z = t.double() if bug == "no_center" else t.double() - center.double().view(1, -1)
    z = z * inv_temp_t
    lse = torch.logsumexp(z, -1)
    if bug == "lse_log2":
        lse = lse / LN2
    q = torch.exp(z - lse[:, None])
    q12 = q * Q_SCALE
    q12_h = (q.float().half().double() * Q_SCALE) if bug == "q_unscaled" else q12.float().half()
    return dict(lse=lse, q=q, q12=q12, q12_h=q12_h)


def ref_rows(s, q, trow, w, gscale, inv_tau_s, bug=None):
    """student rows paired with the teacher probabilities q [Rt, K] (fp64): lse_s, row_loss, ds and the row_loss scale
    n_r |lse_s| + |<q, s~>|"""
    K = s.shape[1]
    t0, t1 = trow[:, 0].long(), trow[:, 1].long()
    v0, v1 = t0 >= 0, t1 >= 0
    if bug == "skip_second":
        v1 = v1 & v0
    qs = q[t0.clamp_min(0)] * v0[:, None] + q[t1.clamp_min(0)] * v1[:, None]
    n = (v0.double() + v1.double())
    if bug == "n2_single":
        n = torch.where(n == 1, 2.0, n)
    st = s.double() * inv_tau_s
    keep = K - 8 if bug == "drop_last8" else K
    lse_s = torch.logsumexp(st[:, :keep], -1)
    dot = (qs[:, :keep] * (s.double()[:, :keep] if bug == "no_inv_tau_dot" else st[:, :keep])).sum(-1)
    row_loss = n * lse_s - dot
    coef = gscale * w.double() * inv_tau_s
    ds = coef[:, None] * (n[:, None] * torch.exp(st - lse_s[:, None]) - qs)
    if keep < K:
        ds[:, keep:] = 0
    return dict(lse_s=lse_s, row_loss=row_loss, ds=ds, scale=n * lse_s.abs() + dot.abs())


def ref_loss_rows(s, t_or_q, center, trow, w, order, gscale, inv_temp_t, inv_tau_s, bug=None):
    """What the kernels write, in fp64: from teacher logits t (any float dtype but fp16), or from stored probabilities
    (fp16 q12, the esvit_row_softmax_q format).  Returns the teacher's lse / q / q12 / q12_h (logits only), and per
    student row lse_s, row_loss, ds, and the scalar loss = sum_r w_r row_loss_r.  `order` only matters to the
    "order_output_only" bug: row order[i]'s outputs computed from row i's inputs."""
    if t_or_q.dtype == F16:
        out, q = {}, t_or_q.double() / Q_SCALE
    else:
        out = ref_teacher(t_or_q, center, inv_temp_t, bug)
        q = out["q"]
    r = ref_rows(s, q, trow, w, gscale, inv_tau_s, bug)
    if bug == "order_output_only":
        o = order.long()
        for k in ("lse_s", "row_loss", "ds", "scale"):
            x = torch.empty_like(r[k])
            x[o] = r[k]
            r[k] = x
    out.update(r)
    out["loss"] = (w.double() * r["row_loss"]).sum()
    out["loss_scale"] = (w.double() * r["row_loss"]).abs().sum()
    return out


class Errors:
    """every metric the GPU test gates (see GATES), accumulated over chunks of teacher and student rows"""

    def __init__(self):
        self.e = {}
        self.ds_num = self.ds_den = 0.0

    def put(self, k, v):
        v = float(v)
        old = self.e.get(k, 0.0)
        self.e[k] = v if (v != v or v > old) else old  # NaN sticks

    def teacher(self, lse, q12, ref):
        self.put("lse", (lse.double() - ref["lse"]).abs().max())
        if q12 is None:
            return
        g, x = q12.double(), ref["q12"]
        err = (g - x).abs()
        normal = x >= Q12_NORMAL
        ulp = torch.where(normal, torch.exp2(torch.floor(torch.log2(x.clamp_min(Q12_NORMAL))) - 10), 2.0 ** -24)
        units = torch.where(normal | (g != 0), err / ulp, torch.zeros_like(err))  # 0 allowed below the threshold
        self.put("q12_ulp", units.max())
        lost = torch.where(normal, torch.zeros_like(err), err).sum(-1) / Q_SCALE
        self.put("flushed", lost.max())
        self.put("tail_mass", torch.where(normal, torch.zeros_like(x), x).sum(-1).max() / Q_SCALE)

    def rows(self, got, ref):
        self.put("lse_s", (got["lse_s"].double() - ref["lse_s"]).abs().max())
        d = (got["row_loss"].double() - ref["row_loss"]).abs()
        self.put("row_loss", (d / ref["scale"].clamp_min(1e-300)).max())  # an n_r = 0 row must be exactly 0
        diff = (got["ds"].double() - ref["ds"]).pow(2).sum(-1)
        norm = ref["ds"].pow(2).sum(-1)
        self.put("ds_row", (diff.sqrt() / norm.sqrt().clamp_min(1e-300)).max())  # a zero row must be exactly 0
        self.ds_num += float(diff.sum())
        self.ds_den += float(norm.sum())

    def result(self):
        e = dict(self.e)
        num, den = self.ds_num, self.ds_den
        e["ds"] = math.sqrt(num / den) if den > 0 else (0.0 if num == 0 else math.inf)
        if num != num:
            e["ds"] = math.nan
        return e


def errors(got, ref):
    """the metrics of kernel-shaped results `got` against ref_loss_rows output `ref` (whole tensors)"""
    E = Errors()
    if "lse" in ref:
        E.teacher(got["lse"], got.get("q12"), ref)
    E.rows(got, ref)
    e = E.result()
    e["loss"] = abs(float(got["loss"]) - float(ref["loss"])) / max(float(ref["loss_scale"]), 1e-300)
    return e


# ================================ loss tables and inputs ===============================================================
def _modules(K):
    from esvit_b200.losses import DDINOLoss, DINOLoss
    return DINOLoss(K, NCROPS, 0.04, 0.04, 0, 1), DDINOLoss(K, NCROPS, 0.04, 0.04, 0, 1)


def region_trow_oracle(s_fea, t_fea, B, Tg, Tl, ncrops=NCROPS):
    """trow int32 [Rs, 2] as esvit_region_match writes it, from oracle.losses.region_match: student row of (v, b, i) ->
    teacher region row (iq * B + b) * Tg + arg-max, -1 where v == iq"""
    split = [Tg] * 2 + [Tl] * (ncrops - 2)
    s_feas = torch.split(s_fea, [T * B for T in split])
    t_feas = t_fea.chunk(2)
    out = []
    for v, T in enumerate(split):
        rows = torch.full((B, T, 2), -1, dtype=torch.long, device=s_fea.device)
        for iq in range(2):
            if v != iq:
                idx = OL.region_match(s_feas[v].view(B, T, -1), t_feas[iq].view(B, Tg, -1))
                rows[..., iq] = (iq * B + torch.arange(B, device=s_fea.device)[:, None]) * Tg + idx
        out.append(rows.view(-1, 2))
    return torch.cat(out).int()


def _check_pairing(trow, B, Tg, Tl):
    """a global-view region row pairs with the other global view only, a local-view row with both"""
    ng = 2 * B * Tg
    assert (trow[: B * Tg, 0] == -1).all() and (trow[B * Tg: ng, 1] == -1).all()
    assert (trow[: B * Tg, 1] >= B * Tg).all() and (trow[B * Tg: ng, 0] < B * Tg).all()
    assert (trow[ng:, 0] >= 0).all() and (trow[ng:, 0] < B * Tg).all() and (trow[ng:, 1] >= B * Tg).all()


def tables(geom, B, K, g, dev, gpu_match):
    """(trow int32 [R, 2], w fp32 [R], image-major order int32 [R], Rt) of the loss term, as DINOLoss / DDINOLoss build
    them, plus 20 synthetic rows (a, -1), (-1, a), (a, a), (a, b), (-1, -1) at the end"""
    dino, ddino = _modules(K)
    if geom == "cls":
        trow, w = dino._cls_tables(B, 1.0 / (N_TERMS * B), dev)
        order = dino._order(B, [(NCROPS, 1)], dev)
        Rt = 2 * B
    else:
        Tg, Tl = GEOMS[geom]
        Rs, Rt, P = B * (2 * Tg + (NCROPS - 2) * Tl), 2 * B * Tg, 64
        s_fea = torch.randn(Rs, P, generator=g, device=dev)
        t_fea = torch.randn(Rt, P, generator=g, device=dev)
        if gpu_match:
            from esvit_b200 import ops
            trow = ops.region_match(s_fea, t_fea, B, NCROPS, Tg, Tl)[1]
        else:
            trow = region_trow_oracle(s_fea, t_fea, B, Tg, Tl)
        _check_pairing(trow, B, Tg, Tl)
        w = ddino._region_weights(B, Tg, Tl, N_TERMS, dev)
        order = ddino._order(B, [(2, Tg), (NCROPS - 2, Tl)], dev)
    R0 = trow.shape[0]
    a = torch.randint(0, Rt, (4,), generator=g, device=dev)
    b = (a + 1 + torch.randint(0, Rt - 1, (4,), generator=g, device=dev)) % Rt
    m1 = torch.full_like(a, -1)
    syn = torch.cat([torch.stack(p, 1) for p in ((a, m1), (m1, a), (a, a), (a, b), (m1, m1))]).int()
    w_syn = w.mean() * (0.5 + torch.rand(syn.shape[0], generator=g, device=dev))
    trow = torch.cat([trow, syn]).contiguous()
    w = torch.cat([w, w_syn.float()]).contiguous()
    order = torch.cat([order, torch.arange(R0, R0 + syn.shape[0], dtype=torch.int32, device=dev)]).contiguous()
    return trow, w, order, Rt


def logits(regime, R, Rt, K, temp, g, dev):
    """(s bf16 [R, K], t bf16 [Rt, K], center fp32 [K]) of one input regime"""
    def randn(*shape):
        return torch.randn(*shape, generator=g, device=dev)

    if regime == "normalised":  # unit features . unit last-layer rows: |logit| <= 1
        W = F.normalize(randn(K, 256), dim=1)
        s = (F.normalize(randn(R, 256), dim=1) @ W.t()).clamp(-1, 1)
        t = (F.normalize(randn(Rt, 256), dim=1) @ W.t()).clamp(-1, 1)
        c = 0.5 * (F.normalize(randn(1, 256), dim=1) @ W.t())[0]
    elif regime == "wide":  # an un-normalised last layer
        s, t, c = 3 * randn(R, K), 3 * randn(Rt, K), 0.3 * randn(K)
    elif regime == "onehot":  # one teacher logit 30 above the rest
        s, t, c = randn(R, K), 0.5 * randn(Rt, K), 0.1 * randn(K)
        hot = torch.randint(0, K, (Rt,), generator=g, device=dev)
        t[torch.arange(Rt, device=dev), hot] += 30
    elif regime == "uniform":  # a collapsed teacher: t == center, q = 1 / K
        s = randn(R, K)
        row = randn(K).to(BF16)
        t, c = row.expand(Rt, K).float(), row.float()
    elif regime == "large_center":  # t and center around 50 (bf16 spacing 0.25), small differences; student near 50 too
        base = 48 + 4 * torch.rand(K, generator=g, device=dev)
        t, c, s = base + 0.5 * randn(Rt, K), base + 0.1 * randn(K), 50 + randn(R, K)
    elif regime == "tail":  # 16 entries carry the mass; the rest log-uniform in q from 1e-10 to 1e-7
        s, c = randn(R, K), 0.1 * randn(K)
        logq = math.log(1e-10) + math.log(1e3) * torch.rand(Rt, K, generator=g, device=dev)
        head = torch.rand(Rt, K, generator=g, device=dev).argsort(-1)[:, :16]
        logq.scatter_(1, head, math.log(0.999 / 16))
        t = c + temp * (logq - math.log(0.999 / 16))
    else:
        raise ValueError(regime)
    return s.to(BF16).contiguous(), t.to(BF16).contiguous(), c.float().contiguous()


def _seed(name):
    return sum(ord(ch) * 31 ** i for i, ch in enumerate(name)) % (1 << 31)


def make_case(case, dev, gpu_match):
    g = torch.Generator(device=dev).manual_seed(_seed(_name(case)))
    trow, w, order, Rt = tables(case.geom, case.B, case.K, g, dev, gpu_match)
    s, t, c = logits(case.regime, trow.shape[0], Rt, case.K, case.temp, g, dev)
    return dict(s=s, t=t, center=c, trow=trow, w=w, order=order)


# ================================ 1. the reference (CPU) ===============================================================
def _exact(w, runs):
    """the float64 weights [(count, value)] whose fp32 rounding the loss module's table w holds"""
    w64 = torch.cat([torch.full((n,), v, dtype=F64) for n, v in runs])
    assert torch.equal(w64.float(), w)
    return w64


@pytest.mark.parametrize("K", [384, 4096])
def test_reference_matches_oracle_dino(K):
    """ref_loss_rows on DINOLoss's cls tables == a float64 run of oracle.losses.dino_loss, loss and logit gradient"""
    B, ncrops, temp = 3, NCROPS, 0.0555
    g = torch.Generator().manual_seed(K)
    s = (torch.randn(ncrops * B, K, generator=g, dtype=F64) * 2).requires_grad_()
    t = torch.randn(2 * B, K, generator=g, dtype=F64) * 0.5
    center = torch.randn(1, K, generator=g, dtype=F64) * 0.3
    l_o = OL.dino_loss(s, t, center, ncrops, temp, STUDENT_TEMP)
    (g_o,) = torch.autograd.grad(l_o, s)
    dino, _ = _modules(K)
    trow, w = dino._cls_tables(B, 1.0 / (N_TERMS * B), "cpu")
    w64 = _exact(w, [(NCROPS * B, 1.0 / (N_TERMS * B))])
    r = ref_loss_rows(s.detach(), t, center[0], trow, w64, None, 1.0, 1 / temp, 1 / STUDENT_TEMP)
    assert abs(float(r["loss"]) - l_o.item()) < 1e-12 * abs(l_o.item())
    assert float((r["ds"] - g_o).norm() / g_o.norm()) < 1e-12


@pytest.mark.parametrize("K", [384, 4096])
def test_reference_matches_oracle_ddino(K):
    """the cls and region terms of ref_loss_rows on DDINOLoss's tables (region pairs from oracle.losses.region_match,
    laid out as esvit_region_match writes them) == a float64 run of oracle.losses.ddino_loss"""
    B, Tg, Tl, P, temp = 2, 49, 9, 32, 0.07
    g = torch.Generator().manual_seed(K + 1)
    Rs = B * (2 * Tg + (NCROPS - 2) * Tl)
    s_cls = torch.randn(NCROPS * B, K, generator=g, dtype=F64).requires_grad_()
    s_reg = torch.randn(Rs, K, generator=g, dtype=F64).requires_grad_()
    t_cls = torch.randn(2 * B, K, generator=g, dtype=F64) * 0.5
    t_reg = torch.randn(2 * B * Tg, K, generator=g, dtype=F64) * 0.5
    s_fea = torch.randn(Rs, P, generator=g, dtype=F64)
    t_fea = torch.randn(2 * B * Tg, P, generator=g, dtype=F64)
    center = torch.randn(1, K, generator=g, dtype=F64) * 0.1
    center_grid = torch.randn(1, K, generator=g, dtype=F64) * 0.1
    l_o = OL.ddino_loss((s_cls, s_reg, s_fea, [Tg, Tl]), (t_cls, t_reg, t_fea, [Tg]), center, center_grid, NCROPS,
                        temp, STUDENT_TEMP)
    g_cls, g_reg = torch.autograd.grad(l_o, (s_cls, s_reg))
    _, ddino = _modules(K)
    trow_c, w_c = ddino._cls_tables(B, 0.5 / (N_TERMS * B), "cpu")
    trow_r = region_trow_oracle(s_fea, t_fea, B, Tg, Tl)
    _check_pairing(trow_r, B, Tg, Tl)
    w_r = ddino._region_weights(B, Tg, Tl, N_TERMS, "cpu")
    w_c = _exact(w_c, [(NCROPS * B, 0.5 / (N_TERMS * B))])
    w_r = _exact(w_r, [(2 * B * Tg, 0.5 / (N_TERMS * B * Tg)), ((NCROPS - 2) * B * Tl, 0.5 / (N_TERMS * B * Tl))])
    rc = ref_loss_rows(s_cls.detach(), t_cls, center[0], trow_c, w_c, None, 1.0, 1 / temp, 1 / STUDENT_TEMP)
    rr = ref_loss_rows(s_reg.detach(), t_reg, center_grid[0], trow_r, w_r, None, 1.0, 1 / temp, 1 / STUDENT_TEMP)
    loss = float(rc["loss"] + rr["loss"])
    assert abs(loss - l_o.item()) < 1e-12 * abs(l_o.item())
    assert float((rc["ds"] - g_cls).norm() / g_cls.norm()) < 1e-12
    assert float((rr["ds"] - g_reg).norm() / g_reg.norm()) < 1e-12


def test_reference_q12_input_and_empty_rows():
    """from stored fp16 q12 the reference uses q12 / 2^12 as given; (-1, -1) rows give exactly 0 loss and gradient"""
    g = torch.Generator().manual_seed(5)
    s = torch.randn(6, 64, generator=g).to(BF16)
    t = torch.randn(2, 64, generator=g).to(BF16)
    c = torch.randn(64, generator=g)
    trow = torch.tensor([[0, -1], [-1, 1], [0, 0], [0, 1], [-1, -1], [1, -1]], dtype=torch.int32)
    w = torch.rand(6, generator=g) + 0.5
    a = ref_loss_rows(s, t, c, trow, w, None, 1.0, 25.0, 10.0)
    b = ref_loss_rows(s, a["q12_h"], c, trow, w, None, 1.0, 25.0, 10.0)
    assert float((a["ds"] - b["ds"]).norm() / a["ds"].norm()) < 1e-3
    assert a["row_loss"][4] == 0 and (a["ds"][4] == 0).all() and a["scale"][4] == 0
    assert torch.equal(a["row_loss"][2], 2 * (a["lse_s"][2] - (a["q"][0] * s[2].double() * 10).sum()))


# each bug must move the reference by >= 5x the gate of the metric named, on a B = 2 version of the named GPU case's
# geometry, K, regime and temperature (the gates are per regime)
SENSITIVITY = [
    ("no_center", "cls_k4096_normalised_t0.04_g1", "ds_row"),
    ("no_center", "cls_k65536_large_center_t0.04_g1", "lse"),
    ("no_inv_tau_dot", "cls_k4096_normalised_t0.04_g1", "row_loss"),
    ("no_inv_tau_dot", "swin_k65536_wide_t0.0555_g1.52588e-05", "row_loss"),
    ("n2_single", "cls_k4096_normalised_t0.04_g1", "row_loss"),
    ("n2_single", "swin_k4096_normalised_t0.04_g1", "ds_row"),
    ("lse_log2", "cls_k65536_normalised_t0.0555_g2", "lse"),
    ("lse_log2", "cls_k65536_uniform_t0.04_g2", "lse"),
    ("drop_last8", "cls_k1000_normalised_t0.04_g1", "ds_row"),
    ("drop_last8", "swin_k1000_normalised_t0.04_g1", "row_loss"),
    ("order_output_only", "swin_k4096_normalised_t0.04_g1", "row_loss"),
    ("order_output_only", "cls_k384_normalised_t0.04_g1", "ds_row"),
    ("skip_second", "cls_k4096_normalised_t0.04_g1", "row_loss"),
    ("skip_second", "swin_k384_normalised_t0.04_g1", "ds_row"),
    ("q_unscaled", "cls_k65536_wide_t0.0555_g1", "q12_ulp"),
    ("q_unscaled", "cls_k65536_tail_t0.0555_g1", "q12_ulp"),
]


def _gate(regime, metric):
    """the looser of the two paths' gates"""
    return {"q12_ulp": Q12_ULP, "flushed": FLUSHED}.get(metric) or max(GATES[p][regime][metric] for p in GATES)


@pytest.mark.parametrize("bug,name,metric", SENSITIVITY)
def test_gates_see_plausible_kernel_bugs(bug, name, metric):
    case = CASES[name]._replace(B=2)
    d = make_case(case, "cpu", gpu_match=False)
    args =(d["s"], d["t"], d["center"], d["trow"], d["w"], d["order"], case.gscale or 1.0, f32(1 / case.temp),
            f32(1 / STUDENT_TEMP))
    good = ref_loss_rows(*args)
    bad = ref_loss_rows(*args, bug=bug)
    bad["q12"] = bad["q12_h"]
    err = errors(bad, good)[metric]
    gate = _gate(case.regime, metric)
    print(f"sensitivity {bug} on {name}: {metric} {err:.3e} = {err / gate:.1f}x gate")
    assert err >= 5 * gate, (bug, name, metric, err, gate)


def test_cases_cover_the_issue_matrix():
    """every geometry at every K it fits under 2^31 elements, every regime at every warm-up temperature, every gscale"""
    have = set(CASES.values())
    for geom in GEOMS:
        for K in (ALL_K if geom in ("cls", "swin") else VIT_K):
            assert any(c.geom == geom and c.K == K for c in have), (geom, K)
    for r in REGIMES:
        for t in TEMPS:
            assert any(c.regime == r and c.temp == t for c in have), (r, t)
    assert {c.gscale for c in have} == set(GSCALES)


# ================================ 2. kernels vs reference (GPU) ========================================================
def run_kernels(path, s, t, center, trow, w, order, gscale, inv_temp_t, inv_tau_s):
    """one loss term through the C ABI, every output NaN-prefilled: path "q" = esvit_row_softmax_q +
    esvit_dino_ce_q_fwd / _bwd, path "lse" = esvit_row_lse + esvit_dino_ce_fwd / _bwd (ESVIT_CE_Q=0); then
    esvit_weighted_sum"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    R, K = s.shape
    Rt = t.shape[0]
    dev = s.device
    nan = math.nan
    lse = torch.full((Rt,), nan, dtype=F32, device=dev)
    lse_s = torch.full((R,), nan, dtype=F32, device=dev)
    row_loss = torch.full((R,), nan, dtype=F32, device=dev)
    loss = torch.full((), nan, dtype=F32, device=dev)
    ds = torch.full_like(s, nan)
    gs = torch.tensor([gscale], dtype=F32, device=dev)
    q12 = None
    if path == "q":
        q12 = torch.full((Rt, K), nan, dtype=F16, device=dev)
        _lib.call("esvit_row_softmax_q", _p(t), _p(center), inv_temp_t, _p(lse), _p(q12), Rt, K, _stream())
        _lib.call("esvit_dino_ce_q_fwd", _p(s), _p(q12), _p(lse_s), _p(trow), _p(order), inv_tau_s, _p(row_loss), R, K,
                  _stream())
        _lib.call("esvit_dino_ce_q_bwd", _p(s), _p(q12), _p(lse_s), _p(trow), _p(order), _p(w), _p(gs), inv_tau_s,
                  _p(ds), R, K, _stream())
    else:
        _lib.call("esvit_row_lse", _p(t), _p(center), inv_temp_t, _p(lse), Rt, K, _stream())
        _lib.call("esvit_dino_ce_fwd", _p(s), _p(t), _p(center), _p(lse_s), _p(lse), _p(trow), _p(order), inv_temp_t,
                  inv_tau_s, _p(row_loss), R, K, _stream())
        _lib.call("esvit_dino_ce_bwd", _p(s), _p(t), _p(center), _p(lse_s), _p(lse), _p(trow), _p(order), _p(w), _p(gs),
                  inv_temp_t, inv_tau_s, _p(ds), R, K, _stream())
    _lib.call("esvit_weighted_sum", _p(row_loss), _p(w), R, _p(loss), _stream())
    torch.cuda.synchronize()
    return dict(lse=lse, q12=q12, lse_s=lse_s, row_loss=row_loss, ds=ds, loss=loss)


def _chunks(n, K, elems=1 << 24):
    step = max(1, elems // K)
    return [slice(i, min(n, i + step)) for i in range(0, n, step)]


def measure(got, d, case, path):
    """the gated metrics of one case, the fp64 reference in chunks of whole rows (no row is sampled).  On the "q" path
    the CE kernels are measured against the reference on the kernel's own stored q12, which the q12 metric measures
    against the exact 2^12 q."""
    inv_t, inv_s = f32(1 / case.temp), f32(1 / STUDENT_TEMP)
    t, s = d["t"], d["s"]
    Rt, K = t.shape
    E = Errors()
    q = torch.empty(Rt, K, dtype=F64, device=t.device)
    for c in _chunks(Rt, K):
        ref = ref_teacher(t[c], d["center"], inv_t)
        E.teacher(got["lse"][c], got["q12"][c] if got["q12"] is not None else None, ref)
        q[c] = ref["q"] if got["q12"] is None else got["q12"][c].double() / Q_SCALE
        del ref
    loss = loss_scale = 0.0
    for c in _chunks(s.shape[0], K):
        r = ref_rows(s[c], q, d["trow"][c], d["w"][c], case.gscale, inv_s)
        E.rows({k: got[k][c] for k in ("lse_s", "row_loss", "ds")}, r)
        wl = d["w"][c].double() * r["row_loss"]
        loss += float(wl.sum())
        loss_scale += float(wl.abs().sum())
        del r
    e = E.result()
    e["loss"] = abs(float(got["loss"]) - loss) / loss_scale
    return e


_DATA = {}


def _gpu_data(name):
    """inputs of a case on the GPU (kept for the next test of the same case only)"""
    if name not in _DATA:
        _DATA.clear()
        torch.cuda.empty_cache()
        _DATA[name] = make_case(CASES[name], "cuda", gpu_match=True)
    return _DATA[name]


PATHS = ("q", "lse")


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", list(CASES))
def test_kernels_match_fp64(name, path):
    case = CASES[name]
    d = _gpu_data(name)
    got = run_kernels(path, d["s"], d["t"], d["center"], d["trow"], d["w"], d["order"], case.gscale, 1 / case.temp,
                      1 / STUDENT_TEMP)
    err = measure(got, d, case, path)
    print(f"loss-kernels {name} {path}: " + " ".join(f"{k} {v:.2e}" for k, v in err.items()))
    gates = dict(GATES[path][case.regime])
    if path == "q":
        gates.update(q12_ulp=Q12_ULP, flushed=FLUSHED)
    bad = {k: (err[k], g) for k, g in gates.items() if k in err and not err[k] < g}
    # the (-1, -1) rows: exactly 0 loss and gradient at w != 0
    none = (d["trow"] < 0).all(-1)
    assert (got["row_loss"][none] == 0).all() and (got["ds"][none] == 0).all()
    if case.gscale == 0:
        assert (got["ds"] == 0).all()
    if case.regime == "tail" and path == "q":  # the case puts a measurable share of mass below the threshold
        assert err["tail_mass"] > 1e-5, err["tail_mass"]
    assert not bad, (name, path, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cls_k65536_normalised_t0.04_g1", "swin_k4096_normalised_t0.04_g1",
                                  "vit8_k1000_normalised_t0.04_g1", "swin_k65536_wide_t0.0555_g1.52588e-05"])
def test_colsum_and_center_ema(name):
    """colsum per column against the fp64 sum; the center EMA bit-exact with the reference's three fp32 ATen ops
    center * m + (colsum / rows) * (1 - m) on the kernel's own colsum (main_esvit.py:657-660)"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    d = _gpu_data(name)
    t, center = d["t"], d["center"]
    Rt, K = t.shape
    ws = torch.full((_lib.load().esvit_colsum_workspace_rows() * K,), math.nan, dtype=F32, device=t.device)
    cs = torch.full((K,), math.nan, dtype=F32, device=t.device)
    _lib.call("esvit_colsum", _p(t), Rt, K, _p(ws), _p(cs), _stream())
    ref = t.double().sum(0)
    err = float(((cs.double() - ref).abs() / t.double().abs().sum(0)).max())
    print(f"loss-kernels {name}: colsum {err:.2e}")
    assert err < COLSUM, err
    for m in (0.9, 0.996):
        out = torch.full_like(center, math.nan)
        _lib.call("esvit_center_ema", _p(center), _p(cs), float(Rt), m, _p(out), K, _stream())
        want = center * m + (cs / torch.full_like(cs, float(Rt))) * (1 - m)  # (true division, see DESIGN.md §4.16)
        assert torch.equal(out, want), (m, int((out != want).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("name", ["swin_k4096_normalised_t0.04_g1", "cls_k65536_wide_t0.0555_g1",
                                  "vit16_k1000_normalised_t0.04_g1"])
def test_row_order_and_reruns_are_bit_identical(name, path):
    """each row belongs to one CTA: no order, the image-major order and a random permutation give bit-identical
    row_loss, lse_s and ds; two runs are bit-identical in every output"""
    case = CASES[name]
    d = _gpu_data(name)
    R = d["s"].shape[0]
    g = torch.Generator(device="cuda").manual_seed(7)
    perm = torch.randperm(R, generator=g, device="cuda").int()

    def run(order):
        return run_kernels(path, d["s"], d["t"], d["center"], d["trow"], d["w"], order, case.gscale, 1 / case.temp,
                           1 / STUDENT_TEMP)

    a, b, c, a2 = run(None), run(d["order"]), run(perm), run(None)
    for k in ("row_loss", "lse_s", "ds"):
        assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), k
    for k in ("lse", "q12", "row_loss", "lse_s", "ds", "loss"):
        if a[k] is not None:
            assert torch.equal(a[k], a2[k]), k


@pytest.mark.gpu
def test_bad_arguments_are_rejected():
    """K % 8 != 0, R <= 0 and (stored-q path) K > esvit_row_softmax_q_max_k() are refused before any launch (the
    buffers are large enough for the launch regardless)"""
    from esvit_b200 import _lib
    from esvit_b200.ops import _p, _stream
    dev = "cuda"
    st = _stream()

    def bufs(R, K):
        return dict(x=torch.zeros(max(R, 1), K, dtype=BF16, device=dev), c=torch.zeros(K, dtype=F32, device=dev),
                    q=torch.zeros(max(R, 1), K, dtype=F16, device=dev), v=torch.zeros(max(R, 1), dtype=F32, device=dev),
                    v2=torch.zeros(max(R, 1), dtype=F32, device=dev), tr=torch.zeros(max(R, 1), 2, dtype=torch.int32,
                                                                                      device=dev),
                    ws=torch.zeros(32 * K, dtype=F32, device=dev), o=torch.zeros(K, dtype=F32, device=dev),
                    gs=torch.ones(1, dtype=F32, device=dev))

    def calls(R, K, b):
        return {
            "esvit_row_lse": (_p(b["x"]), _p(b["c"]), 25.0, _p(b["v"]), R, K, st),
            "esvit_row_softmax_q": (_p(b["x"]), _p(b["c"]), 25.0, _p(b["v"]), _p(b["q"]), R, K, st),
            "esvit_dino_ce_fwd": (_p(b["x"]), _p(b["x"]), _p(b["c"]), _p(b["v"]), _p(b["v2"]), _p(b["tr"]), None, 25.0,
                                  10.0, _p(b["v"]), R, K, st),
            "esvit_dino_ce_bwd": (_p(b["x"]), _p(b["x"]), _p(b["c"]), _p(b["v"]), _p(b["v2"]), _p(b["tr"]), None,
                                  _p(b["v"]), _p(b["gs"]), 25.0, 10.0, _p(b["x"]), R, K, st),
            "esvit_dino_ce_q_fwd": (_p(b["x"]), _p(b["q"]), _p(b["v"]), _p(b["tr"]), None, 10.0, _p(b["v2"]), R, K, st),
            "esvit_dino_ce_q_bwd": (_p(b["x"]), _p(b["q"]), _p(b["v"]), _p(b["tr"]), None, _p(b["v2"]), _p(b["gs"]),
                                    10.0, _p(b["x"]), R, K, st),
            "esvit_colsum": (_p(b["x"]), R, K, _p(b["ws"]), _p(b["o"]), st),
        }

    for R, K in ((2, 12), (0, 64), (-1, 64)):
        b = bufs(R, K)
        for name, args in calls(R, K, b).items():
            with pytest.raises(ValueError):
                _lib.call(name, *args)
    b = bufs(1, 64)
    for R in (0, -1):
        with pytest.raises(ValueError):
            _lib.call("esvit_weighted_sum", _p(b["v"]), _p(b["v2"]), R, _p(b["o"]), st)
    for K in (0, -8):
        with pytest.raises(ValueError):
            _lib.call("esvit_center_ema", _p(b["c"]), _p(b["o"]), 1.0, 0.9, _p(b["ws"]), K, st)
    kmax = _lib.load().esvit_row_softmax_q_max_k()
    K = kmax + 8
    b = dict(x=torch.zeros(1, K, dtype=BF16, device=dev), c=torch.zeros(K, dtype=F32, device=dev),
             q=torch.zeros(1, K, dtype=F16, device=dev), v=torch.zeros(1, dtype=F32, device=dev))
    with pytest.raises(ValueError):
        _lib.call("esvit_row_softmax_q", _p(b["x"]), _p(b["c"]), 25.0, _p(b["v"]), _p(b["q"]), 1, K, st)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("ce_q", ["1", "0"])
@pytest.mark.parametrize("dense", [False, True])
def test_module_inside_teacher_temp_warmup(dense, ce_q, monkeypatch):
    """DINOLoss / DDINOLoss at an epoch inside the 0.04 -> 0.07 warm-up (teacher_temp_schedule) against the oracle at
    the schedule's temperature"""
    monkeypatch.setenv("ESVIT_CE_Q", ce_q)
    from esvit_b200.losses import DDINOLoss, DINOLoss
    K, B, ncrops, Tg, Tl, P, epoch = 4096, 2, 6, 49, 9, 64, 11
    sched = OL.teacher_temp_schedule(0.04, 0.07, 30, 100)
    temp = float(sched[epoch])
    assert 0.045 < temp < 0.065
    g = torch.Generator().manual_seed(11 + dense)
    s_cls = torch.randn(ncrops * B, K, generator=g).to(BF16)
    t_cls = torch.randn(2 * B, K, generator=g).to(BF16)
    center = torch.randn(1, K, generator=g) * 0.1
    mod = (DDINOLoss if dense else DINOLoss)(K, ncrops, 0.04, 0.07, 30, 100).cuda()
    mod.center.copy_(center)
    sc = s_cls.cuda().requires_grad_()
    scr = s_cls.double().requires_grad_()
    if dense:
        Rs = B * (2 * Tg + (ncrops - 2) * Tl)
        s_reg = torch.randn(Rs, K, generator=g).to(BF16)
        t_reg = torch.randn(2 * B * Tg, K, generator=g).to(BF16)
        s_fea, t_fea = torch.randn(Rs, P, generator=g), torch.randn(2 * B * Tg, P, generator=g)
        cg = torch.randn(1, K, generator=g) * 0.1
        mod.center_grid.copy_(cg)
        sg, sgr = s_reg.cuda().requires_grad_(), s_reg.double().requires_grad_()
        l = mod((sc, sg, s_fea.cuda(), [Tg, Tl]), (t_cls.cuda(), t_reg.cuda(), t_fea.cuda(), [Tg]), epoch)
        l_r = OL.ddino_loss((scr, sgr, s_fea.double(), [Tg, Tl]),
                            (t_cls.double(), t_reg.double(), t_fea.double(), [Tg]),
                            center.double(), cg.double(), ncrops, temp, STUDENT_TEMP)
        leaves, refs = (sc, sg), (scr, sgr)
    else:
        l = mod(sc, t_cls.cuda(), epoch)
        l_r = OL.dino_loss(scr, t_cls.double(), center.double(), ncrops, temp, STUDENT_TEMP)
        leaves, refs = (sc,), (scr,)
    l.backward()
    l_r.backward()
    assert abs(l.item() - l_r.item()) < 1e-5 * abs(l_r.item()), (l.item(), l_r.item())
    for a, b in zip(leaves, refs):
        r = float((a.grad.double().cpu() - b.grad).norm() / b.grad.norm())
        assert r < 5e-3, r
    c_r = OL.center_update(center, t_cls.float(), 0.9)
    assert float((mod.center.cpu() - c_r).norm() / c_r.norm()) < 1e-5
