"""Generate tests/golden/esvit_cvt_s3.pt and esvit_cvt_s3_w14.pt by RUNNING THE UNMODIFIED REFERENCE's CvT
(models/cvt_v4_transformer.py) at head dim 32, the head dim of experiments/imagenet/cvt_v4/s3.yaml and win_size/s3.yaml.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_cvt_s3

s3 at reduced width: dims 64/128/192/256, heads 2/4/6/8 (head dim 32 in every stage), depths 1/1/2/1, s3's kernels /
strides, crops 2 x 224^2 + 2 x 96^2 at B = 2, K = 4096, run twice: with s3's windows 7 ("w7", esvit_cvt_s3.pt) and with
win_size/s3's [14, 14, 14, 7] ("w14", esvit_cvt_s3_w14.pt).  Each run stores make_golden_cvt.py's cases: the
train-mode dense forward and BatchNorm running statistics, n_last, and the training sequence with every parameter
gradient, with DDINOLoss and DINOLoss at windows 7 and with DDINOLoss at windows 14 (the DINO view-only loss path does
not depend on the windows).  oracle/cvt.py, run at head dim 32 inside `oracle()`, + oracle/losses.py are asserted
against every stored value while the files are written.
"""
from __future__ import annotations

import contextlib
import os
import sys

import torch
import torch.nn.functional as F

from . import cvt as O
from . import make_golden_cvt as M
from . import make_golden_cvt_w14 as MW
from . import reference_import as R

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
OUTS = {"w7": os.path.join(GOLDEN, "esvit_cvt_s3.pt"), "w14": os.path.join(GOLDEN, "esvit_cvt_s3_w14.pt")}

HEAD_DIM = 32
SPEC = dict(M.SPEC, NUM_HEADS=[2, 4, 6, 8])                  # s3.yaml's windows 7
SPEC_W14 = dict(SPEC, WINDOW_SIZE=[14, 14, 14, 7])         # win_size/s3.yaml's windows
SPECS = {"w7": SPEC, "w14": SPEC_W14}


def layout(sd: dict):
    """oracle/cvt.py's layout with heads = dim / HEAD_DIM"""
    return [(dim, dim // HEAD_DIM, depth, k, s, p) for dim, _, depth, k, s, p in _ORIG["layout"](sd)]


def attention(sd, bufs, pre, x, heads, window, train):
    """oracle/cvt.py's attention (Attention.forward :165-220, no rel-pos bias, no mask) at head dim C / heads; x
    [B, C, H, W]"""
    B, C, H, W = x.shape
    hd = C // heads
    w = min(window, H, W)
    pad_r, pad_b = (w - W % w) % w, (w - H % w) % w
    x = F.pad(x, (0, pad_r, 0, pad_b))
    Hp, Wp = x.shape[-2:]
    sx, sy = Hp // w, Wp // w
    t = F.conv2d(x, sd[pre + "qkv.dw.weight"], None, padding=1, groups=C)          # DepthWiseConv2d :101-105
    t = O.batch_norm(t, sd, bufs, pre + "qkv.bn.", train)
    O.bn_step(bufs, pre + "qkv.bn.", train)
    t = F.conv2d(t, sd[pre + "qkv.pw.weight"], sd.get(pre + "qkv.pw.bias"))
    q, k, v = t.chunk(3, dim=1)

    def part(u):  # 'b (h d) (s_x w_x) (s_y w_y) -> (b s_x s_y) h (w_x w_y) d'
        u = u.reshape(B, heads, hd, sx, w, sy, w).permute(0, 3, 5, 1, 4, 6, 2)
        return u.reshape(B * sx * sy, heads, w * w, hd)

    q, k, v = part(q), part(k), part(v)
    attn = (q @ k.transpose(-1, -2) * C ** -0.5).softmax(dim=-1)     # scale = dim_out ** -0.5 (:126)
    o = (attn @ v).reshape(B, sx, sy, heads, w, w, hd).permute(0, 3, 6, 1, 4, 2, 5).reshape(B, C, Hp, Wp)
    o = o[:, :, :H, :W]
    return F.conv2d(o, sd[pre + "proj_out.weight"], sd[pre + "proj_out.bias"])


_ORIG = {"layout": O.layout, "attention": O.attention}


@contextlib.contextmanager
def head_dim32():
    """oracle/cvt.py's forward functions at head dim 32: its layout and attention (which assume head dim 64) replaced
    by the ones above for the duration"""
    O.layout, O.attention = layout, attention
    try:
        yield
    finally:
        O.layout, O.attention = _ORIG["layout"], _ORIG["attention"]


@contextlib.contextmanager
def oracle(spec):
    """oracle/cvt.py with spec's windows at head dim 32"""
    with head_dim32(), MW.windows(spec["WINDOW_SIZE"]):
        yield


@contextlib.contextmanager
def s3(spec):
    """make_golden_cvt's reference model and oracle with spec"""
    old = M.SPEC
    M.SPEC = spec
    try:
        with oracle(spec):
            yield
    finally:
        M.SPEC = old


def load() -> dict:
    """both fixtures as one: {"runs": {"w7": ..., "w14": ...}, "n_last", "K", "temps", "head_dim"}, each case's seeded
    weights and crops rebuilt"""
    G = None
    for name, path in OUTS.items():
        g = torch.load(path, map_location="cpu", weights_only=False)
        assert list(g["runs"]) == [name], (path, list(g["runs"]))
        if G is None:
            G = g
        else:
            assert all(G[k] == g[k] for k in ("n_last", "K", "temps", "head_dim")), path
            G["runs"].update(g["runs"])
    for run in G["runs"].values():
        for C in [run["features"]] + list(run["train"].values()):
            C["state_dict"] = M.seeded(C["state_recipe"], C["weight_seed"])
            C["crops"] = M.crops(C["crop_seed"])
    return G


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    for i, (name, spec) in enumerate(SPECS.items()):
        with s3(spec):
            train = {"ddino": M.train_case(True, 61 + 3 * i)}
            if name == "w7":
                train["dino"] = M.train_case(False, 62 + 3 * i)
            run = dict(spec=spec, features=M.features_case(60 + 3 * i), train=train)
        out = dict(runs={name: run}, n_last=M.N_LAST, K=M.K, temps=(M.TEMP, M.STUDENT_TEMP), head_dim=HEAD_DIM,
                   generator="oracle/make_golden_cvt_s3.py (reference run on CPU fp32, torch %s)" % torch.__version__)
        torch.save(out, OUTS[name])
        print("wrote", OUTS[name], os.path.getsize(OUTS[name]) // 1024, "KiB")
