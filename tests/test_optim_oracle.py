"""The fp32 SGD / LARS oracle (oracle/optim.py) against the reference's own optimiser steps
(tests/golden/esvit_optim.pt, written by oracle/make_golden_optim.py from torch.optim.SGD and the unmodified
utils.LARS over utils.get_params_groups)."""
import os

import pytest
import torch

from oracle import make_golden_optim as MG
from oracle import optim as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_optim.pt")


def _golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.mark.parametrize("kind", MG.KINDS)
def test_oracle_reproduces_reference_optimizer_steps(kind):
    G = _golden()
    assert tuple(G["meta"]["steps"]) == MG.STEPS and G["meta"]["clip"] == MG.CLIP
    orc = MG.oracle_run(kind)
    ref = G["runs"][kind]
    assert len(orc) == len(ref) == len(MG.STEPS)
    for it, (o, r) in enumerate(zip(orc, ref)):
        assert o["buffers"].keys() == r["buffers"].keys(), (kind, it)
        for part in ("student", "teacher", "buffers"):
            assert o[part].keys() == r[part].keys()
            for n, v in r[part].items():
                assert torch.allclose(o[part][n], v, rtol=1e-6, atol=1e-7), (kind, it, part, n)


@pytest.mark.parametrize("kind", MG.KINDS)
def test_fixture_covers_cancel_zero_norms_and_clip(kind):
    """step 0 cancels the last layer (no buffer, unchanged weights), the zero-valued weight and the zero-gradient 2-D
    bias get buffers, and the clip fires on the large-gradient steps"""
    G = _golden()
    r0 = G["runs"][kind][0]
    init = {n: p.detach() for n, p in MG.toy().named_parameters()}
    assert "last_layer.weight" not in r0["buffers"]
    assert torch.equal(r0["student"]["last_layer.weight"], init["last_layer.weight"])
    assert float(init["z.weight"].abs().max()) == 0 and float(r0["student"]["z.weight"].abs().max()) > 0
    assert float(r0["buffers"]["tok.bias"].abs().max()) == 0
    assert torch.equal(r0["student"]["tok.bias"], init["tok.bias"])  # group 1 (wd 0), zero gradient
    for it, s in enumerate(MG.STEPS):
        norms = [float(g.norm()) for g in MG.step_grads(MG.toy(), it).values()]
        assert (max(norms) > MG.CLIP) == (s[4] > 1), (it, max(norms))


def test_lars_trust_ratio_is_by_dimension():
    """a 2-D parameter of group 1 (wd 0) still gets the trust ratio; a 1-D one never does"""
    torch.manual_seed(0)
    w2 = torch.nn.Parameter(torch.randn(4, 3))
    w1 = torch.nn.Parameter(torch.randn(5))
    opt = O.LARS([{"params": [w2, w1], "weight_decay": 0.0}], lr=1.0, eta=0.01)
    g2, g1 = torch.randn(4, 3), torch.randn(5)
    w2.grad, w1.grad = g2.clone(), g1.clone()
    a2, a1 = w2.detach().clone(), w1.detach().clone()
    opt.step()
    q = 0.01 * a2.norm() / g2.norm()
    assert torch.allclose(w2.detach(), a2 - q * g2, rtol=1e-6, atol=1e-7)
    assert torch.allclose(w1.detach(), a1 - g1, rtol=1e-6, atol=1e-7)
