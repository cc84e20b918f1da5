"""The ws-7 backward stages dQ / dK / dV in the dead tiles of a pipeline stage and lets each thread's next gather
overwrite what that thread just stored from, with no block barrier in between.  A race there would show as dqkv changing
with the schedule: between two runs, or between the full grid and a forced small one (ESVIT_ATTN_GY), where a CTA walks
many windows and every stage is reused.  Checked where the staging meets padding: the 24² map (windows hanging over the
map's edge) shifted and unshifted, and the 3² stage-3 local map, where 40 of the 49 slots of every window are padding."""
import pytest
import torch

from test_window_attn_gpu import CASES, _run_kernel, _seed, make_inputs


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w7_c96_m24_s3", "w7_c96_m24_s0", "w7_c768_m3_s0"])
def test_dqkv_is_independent_of_the_schedule(monkeypatch, name):
    monkeypatch.delenv("ESVIT_ATTN_DBG", raising=False)
    monkeypatch.delenv("ESVIT_ATTN_GY", raising=False)
    case = CASES[name]
    inp = make_inputs(case, _seed(name), "cuda")
    base = _run_kernel(inp, case, nan_fill=True)
    real = base["dqkv"].float()
    assert torch.isfinite(real).all()  # every real token's row is written
    again = _run_kernel(inp, case, nan_fill=True)
    assert torch.equal(again["dqkv"], base["dqkv"])
    for gy in ("1", "2", "5"):
        monkeypatch.setenv("ESVIT_ATTN_GY", gy)
        got = _run_kernel(inp, case, nan_fill=True)
        assert torch.equal(got["dqkv"], base["dqkv"]), gy
