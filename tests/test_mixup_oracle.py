"""The fp32 mixup DINOLoss oracle against the reference's own values (tests/golden/esvit_mixup.pt, written by
oracle/make_golden_mixup.py from the unmodified reference DINOLoss)."""
import os

import pytest
import torch

from oracle import golden as GD
from oracle import losses as L
from oracle import mixup as M
from oracle import make_golden_mixup as MG

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_mixup.pt")


def _golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.mark.parametrize("name", sorted(MG.CASES))
def test_oracle_reproduces_reference_mixup_loss(name):
    G = _golden()
    c = G["cases"][name]
    wt, tt, wte, ne, st, cm = G["meta"]["schedule"]
    sched = L.teacher_temp_schedule(wt, tt, wte, ne)
    targets = list(c["targets"])
    center = torch.zeros(1, c["K"])
    for rec in c["steps"]:
        s, t = MG.case_inputs(c["B"], c["K"], c["ncrops"], c["seed"], rec["epoch"])
        s = s.requires_grad_(True)
        loss = M.dino_loss_mixup(s, t, center, c["ncrops"], float(sched[rec["epoch"]]), targets, st)
        loss.backward()
        assert abs(float(loss) - rec["loss"]) <= 2e-5 * max(1.0, abs(rec["loss"])), (float(loss), rec["loss"])
        g, ref = GD.at_golden(s.grad, rec["grad"])
        assert torch.allclose(g, ref, rtol=1e-4, atol=1e-6 * float(ref.abs().max())), name
        center = L.center_update(center, t, cm)
        assert torch.allclose(center, rec["center"], atol=1e-7), name


@pytest.mark.parametrize("name", sorted(MG.CASES))
def test_fixture_targets_are_the_documented_recipe(name):
    """The stored targets are timm's mixup_target for the first num_mixup_views views and eye(B) after."""
    c = _golden()["cases"][name]
    B, n_mix = c["B"], c["num_mixup_views"]
    assert torch.equal(c["targets"], torch.stack(MG.case_targets(B, c["ncrops"], c["kind"], n_mix, c["smoothing"],
                                                                 c["seed"])))
    for v in range(c["ncrops"]):
        T = c["targets"][v]
        if v >= n_mix:
            assert torch.equal(T, torch.eye(B))
        elif c["kind"] == "arbitrary":
            assert float(T.min()) >= 0 and float(T[:, (v + 1) % B].abs().max()) == 0
        else:  # each row is a distribution over the B samples; label smoothing makes every entry positive
            assert torch.allclose(T.sum(1), torch.ones(B), atol=1e-6)
            if c["smoothing"] > 0:
                assert float(T.min()) > 0


def test_timm_targets_per_row_lambda_are_not_symmetric():
    lam = torch.tensor([0.9, 0.2, 0.6, 0.3])
    T = M.timm_mixup_target(4, lam, 0.0)
    assert not torch.equal(T, T.t())
    assert torch.allclose(T[0], torch.tensor([0.9, 0.0, 0.0, 0.1]))


@pytest.mark.parametrize("ncrops", [2, 4])
def test_identity_targets_give_the_plain_loss(ncrops):
    g = torch.Generator().manual_seed(ncrops)
    B, K = 5, 96
    s, t = torch.randn(ncrops * B, K, generator=g) * 2, torch.randn(2 * B, K, generator=g)
    center = torch.randn(1, K, generator=g) * 0.1
    eye = [torch.eye(B)] * ncrops
    a = M.dino_loss_mixup(s, t, center, ncrops, 0.05, eye)
    b = L.dino_loss(s, t, center, ncrops, 0.05)
    assert abs(float(a) - float(b)) <= 1e-5 * abs(float(b)), (float(a), float(b))
