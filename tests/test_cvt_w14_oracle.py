"""The CvT oracle (oracle/cvt.py) with the win_size/s1.yaml windows [14, 14, 14, 7] against the reference fixture
tests/golden/esvit_cvt_w14.pt (CPU)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import cvt as O  # noqa: E402
from oracle import losses as LO  # noqa: E402
from oracle import make_golden_cvt_w14 as MW  # noqa: E402
from oracle.golden import at_golden  # noqa: E402

G = MW.load()


def _close(a, ref, atol=2e-5):
    a, r = at_golden(a, ref)
    assert torch.allclose(a, r, atol=atol, rtol=0), float((a - r).abs().max())


def test_fixture_spec_is_win_size_s1_at_reduced_width():
    assert G["spec"]["WINDOW_SIZE"] == [14, 14, 14, 7]
    assert G["spec"] == MW.SPEC


def test_features_running_stats_and_n_last():
    F_ = G["features"]
    sd = F_["state_dict"]
    bufs = O.buffers(sd)
    with MW.windows(G["spec"]["WINDOW_SIZE"]), torch.no_grad():
        pooled, region, npatch = O.forward_dense(sd, bufs, F_["crops"], True)
        nl = O.n_last_blocks(sd, {k: v.clone() for k, v in bufs.items()}, torch.cat(F_["crops"][:2]), G["n_last"])
    assert npatch == F_["npatch"] == [49, 9]
    _close(pooled, F_["pooled"])
    _close(region, F_["region"])
    for k, v in F_["buffers"].items():
        assert torch.allclose(bufs[k].double(), v.double(), atol=1e-6, rtol=0), k
    _close(nl, F_["n_last"])


def test_window_size_matters():
    """the fixture is not reproduced with the s1 windows (7 everywhere)"""
    F_ = G["features"]
    sd = F_["state_dict"]
    with torch.no_grad():
        pooled, _, _ = O.forward_dense(sd, O.buffers(sd), F_["crops"], True)
    a, r = at_golden(pooled, F_["pooled"])
    assert float((a - r).abs().max()) > 1e-3


def test_train_steps():
    T0, TS = G["temps"]
    for name, C in G["train"].items():
        sd = C["state_dict"]
        x = C["crops"]
        osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running_" not in k
                                           and not k.endswith("weight_g")) for k, v in sd.items()}
        with MW.windows(G["spec"]["WINDOW_SIZE"]):
            with torch.no_grad():
                ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, O.buffers(sd), x[:2], C["dense"])
            os_ = O.multicrop_forward(osd, O.buffers(sd), x, C["dense"])
        zero = torch.zeros(1, G["K"])
        loss = LO.ddino_loss(os_, ot, zero, zero, len(x), T0, TS) if C["dense"] else \
            LO.dino_loss(os_, ot, zero, len(x), T0, TS)
        loss.backward()
        assert abs(float(loss) - C["loss"]) <= 1e-5 * abs(C["loss"]), name
        for k, ref in C["grads"].items():
            a, r = at_golden(osd[k].grad, ref)
            assert torch.allclose(a, r, atol=1e-6, rtol=1e-4), (name, k)
