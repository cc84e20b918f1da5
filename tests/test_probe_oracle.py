"""CPU: oracle/probe.py reproduces what the UNMODIFIED reference's linear probe produced (tests/golden/esvit_probe.pt,
written by oracle/make_golden_probe.py), CosineAnnealingLR's lr sequence bit for bit, and esvit_b200.probe's
LinearClassifier initialises and names its parameters like the reference's."""
import os

import pytest
import torch

from oracle import golden as GD
from oracle import make_golden_probe as MG
from oracle import probe as PR
from oracle import reference_import as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_probe.pt")


@pytest.fixture(scope="module")
def G():
    return MG.load(GOLDEN)


def test_fixture_is_small():
    assert os.path.getsize(GOLDEN) < 512 << 10


def test_oracle_reproduces_reference_trajectory(G):
    p = G["params"]
    x, y = G["train"]
    w, b, bw, bb = PR.init_classifier(p["D"], p["C"], p["init_seed"]) + (None, None)
    batches = [(x[r:r + p["batch"]], y[r:r + p["batch"]]) for r in range(0, x.shape[0], p["batch"])]
    assert batches[-1][0].shape[0] % 8 != 0  # the ragged last batch
    lrs = PR.cosine_lrs(p["lr"], p["epochs"])
    assert lrs == G["lrs"]
    for s, (xb, yb) in enumerate(batches * p["epochs"]):
        loss, w, b, bw, bb = PR.train_step(w, b, bw, bb, xb, yb, lrs[s // len(batches)])
        ref = G["steps"][s]
        assert abs(loss - ref["loss"]) <= 1e-5 * abs(ref["loss"]), s
        for name, o in (("weight", w), ("bias", b), ("buf_w", bw), ("buf_b", bb)):
            a, r = GD.at_golden(o, ref[name])
            assert torch.allclose(a, r, rtol=1e-4, atol=2e-6), (s, name, float((a - r).abs().max()))
        assert abs(float(w.double().norm()) - ref["weight_norm"]) <= 1e-5 * ref["weight_norm"]
        assert abs(float(bw.double().norm()) - ref["buf_w_norm"]) <= 1e-5 * ref["buf_w_norm"]
    v = PR.validate(w, b, *G["val"], p["batch"])
    for k in ("loss", "acc1", "acc5"):
        assert abs(v[k] - G["validation"][k]) <= 1e-6 * abs(G["validation"][k]), (k, v, G["validation"])
    # every validation outcome stays decided within the margin the fixture was made with
    xv, yv = G["val"]
    assert bool(PR.decided(PR.forward(w, b, xv), yv, p["margin"] * PR.logit_bound(w, xv)).all())


def test_cosine_lrs_equal_torch_scheduler():
    for base, epochs in ((0.003, 2), (0.001 * 1024 / 256, 100), (0.05, 7)):
        w = torch.nn.Parameter(torch.zeros(1))
        opt = torch.optim.SGD([w], base, momentum=0.9, weight_decay=0)
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, epochs, eta_min=0)
        got = []
        for _ in range(epochs):
            got.append(opt.param_groups[0]["lr"])
            opt.step()
            sched.step()
        assert got == PR.cosine_lrs(base, epochs)


def test_classifier_init_and_keys_match_reference():
    from esvit_b200.probe import LinearClassifier
    torch.manual_seed(5)
    m = LinearClassifier(2304, 1000)
    w, b = PR.init_classifier(2304, 1000, 5)
    assert list(m.state_dict()) == ["linear.weight", "linear.bias"]
    assert torch.equal(m.linear.weight, w) and torch.equal(m.linear.bias, b)
    if R.available():  # the reference's own class, AST-extracted
        ref = PR.reference_probe()["LinearClassifier"]
        torch.manual_seed(5)
        r = ref(2304, 1000)
        assert list(r.state_dict()) == list(m.state_dict())
        assert all(torch.equal(a, c) for a, c in zip(r.state_dict().values(), m.state_dict().values()))
