import os

import torch

from oracle import golden as _golden

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_small.pt")


def rel(a: torch.Tensor, b: torch.Tensor) -> float:
    """||a - b|| / ||b|| in fp64 on CPU."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def assert_close(a, b, tol, name=""):
    r = rel(a, b)
    assert r < tol, f"{name}: rel l2 error {r:.3e} >= {tol:.1e}"


def load_golden(path: str = GOLDEN):
    """the fixture with its seeded weights and crops rebuilt (oracle/golden.py)"""
    return _golden.load(path)


# (actual, golden) restricted to the elements a fixture stores (large tensors are stored as a seeded sample)
at_golden = _golden.at_golden


# tolerances (documented in DESIGN.md §parity): the CUDA path runs its GEMMs and branch activations in bf16
# (8-bit mantissa, like the reference under autocast) against an fp32 CPU oracle.
TOL_FP32_KERNEL = 2e-5   # kernels that are fp32 end to end (LN stats, patch embed, EMA/clip scalars)
TOL_BF16_ACT = 2e-2      # forward activations through bf16 GEMMs
TOL_BF16_GRAD = 6e-2     # parameter gradients through the bf16 backward
