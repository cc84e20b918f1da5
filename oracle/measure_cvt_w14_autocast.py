"""oracle/measure_cvt_autocast.py for the win_size/s1 windows [14, 14, 14, 7]: how far the UNMODIFIED reference CvT's
own gradients move under bf16 autocast from its fp32 gradients, the yardstick for the gradient gates of
tests/test_cvt_w14_gpu.py.

TEST INFRASTRUCTURE (needs a CUDA device and the reference under oracle/_ref/):

    python -m oracle.measure_cvt_w14_autocast

Two cases, as in measure_cvt_autocast.py: fixture (the spec, seeded weights and crops of tests/golden/esvit_cvt_w14.pt,
train case "ddino", K = 4096) and real (CvT-13 win_size/s1, K = 65 536, 2 + 8 crops at B = 2, the same seeds).
"""
from __future__ import annotations

import json
import sys

import torch

from . import make_golden_cvt_w14 as MW
from . import measure_cvt_autocast as MA
from . import reference_import as R


def main():
    if not (torch.cuda.is_available() and R.available()):
        sys.exit("needs a CUDA device and the reference under oracle/_ref/")
    from esvit_b200.cvt_v4_transformer import S1_W14_SPEC
    G = MW.load()
    C = G["train"]["ddino"]
    print(json.dumps(dict(case="fixture", **MA._case(MW.SPEC, G["K"], C["weight_seed"], C["crops"]))))
    g = torch.Generator().manual_seed(5)
    crops = [torch.randn(2, 3, 224, 224, generator=g) for _ in range(2)] + \
            [torch.randn(2, 3, 96, 96, generator=g) for _ in range(8)]
    print(json.dumps(dict(case="real", **MA._case(S1_W14_SPEC, 65536, 11, crops))))


if __name__ == "__main__":
    main()
