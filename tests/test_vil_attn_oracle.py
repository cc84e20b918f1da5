"""CPU: oracle/vil_attn.py's dense restatement (the yardstick of tests/test_vil_attn_gpu.py) against the unmodified
reference Long2DSCSelfAttention in fp64, modes -1, 0 and 1..8, with and without zero padding (10^2 and 12^2 maps).
Needs the reference under oracle/_ref/ and `einops`, which the reference imports."""
import pytest

from oracle import reference_import as RI


def test_dense_restatement_matches_reference():
    pytest.importorskip("einops")
    if not RI.available():
        pytest.skip(f"reference tree not found at {RI.REF_ROOT}")
    from oracle import vil_attn as O
    for key, err in O.compare_with_reference().items():
        assert err < 1e-12, f"(side, heads, mode) {key}: max abs difference {err:.3e}"
