"""oracle/measure_cvt_autocast.py at head dim 32 (experiments/imagenet/cvt_v4/s3.yaml and win_size/s3.yaml): how far the
UNMODIFIED reference CvT's own gradients move under bf16 autocast from its fp32 gradients, the yardstick for the gradient
gates of tests/test_cvt_s3_gpu.py.

TEST INFRASTRUCTURE (needs a CUDA device and the reference under oracle/_ref/):

    python -m oracle.measure_cvt_s3_autocast

Four cases, as in measure_cvt_autocast.py: fixture_w7 / fixture_w14 (the specs, seeded weights and crops of
tests/golden/esvit_cvt_s3.pt, train case "ddino", K = 4096) and real_s3 / real_s3_w14 (the full specs, K = 65 536,
2 + 8 crops at B = 2, the same seeds as the other measurements).
"""
from __future__ import annotations

import json
import sys

import torch

from . import make_golden_cvt_s3 as M3
from . import measure_cvt_autocast as MA
from . import reference_import as R


def main():
    if not (torch.cuda.is_available() and R.available()):
        sys.exit("needs a CUDA device and the reference under oracle/_ref/")
    from esvit_b200.cvt_v4_transformer import S3_SPEC, S3_W14_SPEC
    G = M3.load()
    for name, run in G["runs"].items():
        C = run["train"]["ddino"]
        print(json.dumps(dict(case=f"fixture_{name}", **MA._case(run["spec"], G["K"], C["weight_seed"], C["crops"]))))
    for name, spec in (("real_s3", S3_SPEC), ("real_s3_w14", S3_W14_SPEC)):
        g = torch.Generator().manual_seed(5)
        crops = [torch.randn(2, 3, 224, 224, generator=g) for _ in range(2)] + \
                [torch.randn(2, 3, 96, 96, generator=g) for _ in range(8)]
        print(json.dumps(dict(case=name, **MA._case(spec, 65536, 11, crops))))


if __name__ == "__main__":
    main()
