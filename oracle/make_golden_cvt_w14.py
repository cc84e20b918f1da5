"""Generate tests/golden/esvit_cvt_w14.pt by RUNNING THE UNMODIFIED REFERENCE's CvT (models/cvt_v4_transformer.py) with
the windows of experiments/imagenet/cvt_v4/win_size/s1.yaml.

TEST INFRASTRUCTURE.  Usage (ESVIT_REFERENCE = a reference checkout, else oracle/_ref/):

    python -m oracle.make_golden_cvt_w14

The cases, storage and checks are make_golden_cvt.py's (head-dim-64 CvT, dims 64/128/192/256, heads 1/2/3/4, depths
1/1/2/1, crops 2 x 224^2 + 2 x 96^2 at B = 2, K = 4096), run with WINDOW_SIZE [14, 14, 14, 7].  The per-stage windows
w = min(14, H, W) and tokens L = w^2 are: 224^2: 14 / 196 (stages 0-2), 7 / 49; 96^2: stage 0 padded 24 -> 28 at 14 /
196, then 12 / 144, 6 / 36, 3 / 9.  oracle/cvt.py + oracle/losses.py are asserted against every stored value while the
file is written (inside `w14()`, which gives the oracle's stage_blocks the per-stage window).
"""
from __future__ import annotations

import contextlib
import os
import sys

import torch

from . import cvt as O
from . import make_golden_cvt as M
from . import reference_import as R

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "esvit_cvt_w14.pt")

SPEC = dict(M.SPEC, WINDOW_SIZE=[14, 14, 14, 7])


@contextlib.contextmanager
def windows(ws):
    """oracle/cvt.py's forward functions with window ws[i] in stage i: its stage_blocks takes the window, and
    forward_features / n_last_blocks call it with the default 7"""
    orig = O.stage_blocks

    def stage_blocks(sd, bufs, i, x, heads, depth, train, window=7, keeps=None):
        return orig(sd, bufs, i, x, heads, depth, train, ws[i], keeps)

    O.stage_blocks = stage_blocks
    try:
        yield
    finally:
        O.stage_blocks = orig


@contextlib.contextmanager
def w14():
    """make_golden_cvt's reference model and oracle with SPEC's windows"""
    spec = M.SPEC
    M.SPEC = SPEC
    try:
        with windows(SPEC["WINDOW_SIZE"]):
            yield
    finally:
        M.SPEC = spec


def load(path: str = OUT) -> dict:
    """the fixture with each case's seeded weights and crops rebuilt"""
    return M.load(path)


if __name__ == "__main__":
    if not R.available():
        sys.exit("reference tree not found: set ESVIT_REFERENCE to a checkout of microsoft/esvit")
    torch.manual_seed(0)
    with w14():
        out = dict(spec=SPEC, features=M.features_case(50), n_last=M.N_LAST,
                   train={"ddino": M.train_case(True, 51), "dino": M.train_case(False, 52)}, K=M.K,
                   temps=(M.TEMP, M.STUDENT_TEMP),
                   generator="oracle/make_golden_cvt_w14.py (reference run on CPU fp32, torch %s)" % torch.__version__)
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")
