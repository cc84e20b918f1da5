"""CPU checks of the DINOHead(use_bn=True) oracle (oracle/bnhead.py) against tests/golden/esvit_bnhead.pt, which the
unmodified reference wrote (oracle/make_golden_bnhead.py), and of the esvit_b200 head's module layout."""
import pytest
import torch

from helpers import at_golden, rel
from oracle import bnhead as BH
from oracle import make_golden_bnhead as MB

CASES = ("swin_dense", "swin_view", "vit_dense")


@pytest.fixture(scope="module")
def golden():
    return MB.load()


@pytest.mark.parametrize("name", CASES)
def test_oracle_steps_match_reference_fixture(golden, name):
    C = golden["cases"][name]
    orc = BH.OracleBnStep(C["state_dict"], C["arch"], C["dense"], C["ncrops"], golden["out_dim"], **golden["hp"])
    for it, ref in enumerate(C["steps"]):
        loss, s_out, t_out, grads = orc.step(C["crops"], epoch=0)
        tol = 2e-5 if it == 0 else 2e-3   # later steps: the oracle's own AdamW updates
        assert abs(loss - ref["loss"]) < tol * abs(ref["loss"]), (it, loss, ref["loss"])
        outs = (list(s_out[:2]) + list(t_out[:2])) if C["dense"] else [s_out, t_out]
        for a, b in zip(outs, ref["student_outputs"] + ref["teacher_outputs"]):
            assert rel(*at_golden(a.detach(), b)) < tol * 50
        assert set(grads) == set(ref["grads_stats"])
        gmax = max(n for _, n in ref["grads_stats"].values())
        for k, (_, nrm) in ref["grads_stats"].items():
            assert abs(float(grads[k].double().norm()) - nrm) < 2e-2 * nrm + MB.GRAD_ATOL * gmax, (it, k)
        for k, g in ref["grads_head"].items():
            a, b = at_golden(grads[k], g)
            assert float((a - b).double().norm()) < 2e-2 * float(b.double().norm()) + MB.GRAD_ATOL * gmax, (it, k)
        run = {f"{net}.{k}": v for net, d in (("student", orc.student), ("teacher", orc.teacher))
               for k, v in BH.running_stats(d).items()}
        assert set(run) == set(ref["running"])
        for k, v in ref["running"].items():
            if v.dtype == torch.long:
                assert torch.equal(run[k], v), k
            else:
                assert rel(run[k], v) < tol * 50, (it, k)


@pytest.mark.parametrize("name", CASES)
def test_oracle_eval_head_matches_reference_fixture(golden, name):
    C = golden["cases"][name]
    sd = {k: v.clone() for k, v in C["state_dict"].items() if k.startswith("head.")}
    for k in sd:
        if k.endswith(BH.BUFFERS):
            sd[k] = C["steps"][-1]["running"]["student." + k].clone()
    before = {k: v.clone() for k, v in sd.items()}
    out = BH.dino_head_bn(C["eval_input"], sd, "head", train=False)
    assert rel(*at_golden(out, C["eval_output"])) < 1e-5
    assert all(torch.equal(sd[k], before[k]) for k in sd)   # eval mode leaves the running statistics alone


def test_train_mode_rejects_a_single_row():
    G = MB.load()
    sd = {k: v.clone() for k, v in G["cases"]["swin_view"]["state_dict"].items()}
    with pytest.raises(ValueError):
        BH.dino_head_bn(torch.randn(1, sd["head.mlp.0.weight"].shape[1]), sd, "head", train=True)


@pytest.mark.parametrize("name", CASES)
def test_reference_state_dict_loads_strict(golden, name):
    """esvit_b200's DINOHead(use_bn=True) holds the reference's parameters and buffers under the reference's keys"""
    from esvit_b200.vision_transformer import DINOHead
    C = golden["cases"][name]
    for prefix in ("head.", "head_dense.") if C["dense"] else ("head.",):
        sd = {k[len(prefix):]: v for k, v in C["state_dict"].items() if k.startswith(prefix)}
        h = DINOHead(sd["mlp.0.weight"].shape[1], golden["out_dim"], use_bn=True, **golden["head"])
        h.load_state_dict(sd, strict=True)
        bns = [m for m in h.modules() if isinstance(m, torch.nn.BatchNorm1d)]
        assert len(bns) == 2 and all(m.momentum == 0.1 and m.eps == 1e-5 for m in bns)
        want = [f"mlp.{i}.{b}" for i in (0, 3, 6) for b in ("weight", "bias")]
        want += [f"mlp.{i}.{b}" for i in (1, 4) for b in ("weight", "bias", "running_mean", "running_var",
                                                          "num_batches_tracked")]
        assert sorted(k for k in sd if k.startswith("mlp.")) == sorted(want)


def test_sync_batchnorm_conversion_keeps_the_layout():
    from esvit_b200.vision_transformer import DINOHead
    h = DINOHead(32, 64, use_bn=True, hidden_dim=64, bottleneck_dim=16)
    keys = list(h.state_dict())
    s = torch.nn.SyncBatchNorm.convert_sync_batchnorm(h)
    assert sum(isinstance(m, torch.nn.SyncBatchNorm) for m in s.modules()) == 2
    assert list(s.state_dict()) == keys
    plain = DINOHead(32, 64, hidden_dim=64, bottleneck_dim=16)
    assert not any(isinstance(m, torch.nn.BatchNorm1d) for m in plain.modules())
