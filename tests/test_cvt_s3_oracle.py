"""The CvT oracle (oracle/cvt.py, run at head dim 32 through oracle/make_golden_cvt_s3.py's layout and attention), the
head dim of experiments/imagenet/cvt_v4/s3.yaml and win_size/s3.yaml, against the reference fixtures
tests/golden/esvit_cvt_s3.pt (windows 7) and esvit_cvt_s3_w14.pt (windows 14 / 14 / 14 / 7); the S3 specs against the
reference's yaml files and state_dict; the n-last tap plumbing at s3's depths (CPU)."""
import os
import sys
import types
import warnings

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import cvt as O  # noqa: E402
from oracle import losses as LO  # noqa: E402
from oracle import make_golden_cvt_s3 as M3  # noqa: E402
from oracle.golden import at_golden  # noqa: E402

G = M3.load()
RUNS = sorted(G["runs"])


def _close(a, ref, atol=2e-5):
    a, r = at_golden(a, ref)
    assert torch.allclose(a, r, atol=atol, rtol=0), float((a - r).abs().max())


def test_fixture_spec_is_s3_at_reduced_width():
    from esvit_b200.cvt_v4_transformer import S3_SPEC
    assert RUNS == ["w14", "w7"] and G["head_dim"] == 32
    for name, spec in M3.SPECS.items():
        assert G["runs"][name]["spec"] == spec
        assert [d // h for d, h in zip(spec["DIM_EMBED"], spec["NUM_HEADS"])] == [32] * 4
        for k in ("PATCH_SIZE", "PATCH_STRIDE", "PATCH_PADDING", "KERNEL_QKV", "PADDING_QKV", "QKV_BIAS", "SHIFT",
                  "REL_POS_EMBED", "MLP_RATIO"):
            assert spec[k] == S3_SPEC[k], k
    assert G["runs"]["w7"]["spec"]["WINDOW_SIZE"] == [7] * 4
    assert G["runs"]["w14"]["spec"]["WINDOW_SIZE"] == [14, 14, 14, 7]


@pytest.mark.parametrize("run", RUNS)
def test_features_running_stats_and_n_last(run):
    R_ = G["runs"][run]
    F_ = R_["features"]
    sd = F_["state_dict"]
    bufs = O.buffers(sd)
    with M3.oracle(R_["spec"]), torch.no_grad():
        pooled, region, npatch = O.forward_dense(sd, bufs, F_["crops"], True)
        nl = O.n_last_blocks(sd, {k: v.clone() for k, v in bufs.items()}, torch.cat(F_["crops"][:2]), G["n_last"])
    assert npatch == F_["npatch"] == [49, 9]
    _close(pooled, F_["pooled"])
    _close(region, F_["region"])
    for k, v in F_["buffers"].items():
        assert torch.allclose(bufs[k].double(), v.double(), atol=1e-6, rtol=0), k
    _close(nl, F_["n_last"])


def test_head_dim_matters():
    """the fixture is not reproduced at the oracle's default head dim 64"""
    R_ = G["runs"]["w7"]
    F_ = R_["features"]
    sd = F_["state_dict"]
    with torch.no_grad():
        pooled, _, _ = O.forward_dense(sd, O.buffers(sd), F_["crops"], True)
    a, r = at_golden(pooled, F_["pooled"])
    assert float((a - r).abs().max()) > 1e-3


@pytest.mark.parametrize("run", RUNS)
def test_train_steps(run):
    R_ = G["runs"][run]
    T0, TS = G["temps"]
    assert sorted(R_["train"]) == (["ddino", "dino"] if run == "w7" else ["ddino"])
    for name, C in R_["train"].items():
        sd = C["state_dict"]
        x = C["crops"]
        osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running_" not in k
                                           and not k.endswith("weight_g")) for k, v in sd.items()}
        with M3.oracle(R_["spec"]):
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


def test_specs_and_engine_entries():
    from esvit_b200 import engine
    from esvit_b200.cvt_v4_transformer import S3_SPEC, S3_W14_SPEC
    assert S3_SPEC["DIM_EMBED"] == [64, 128, 256, 512] and S3_SPEC["NUM_HEADS"] == [2, 4, 8, 16]
    assert S3_SPEC["DEPTH"] == [2, 2, 10, 4] and S3_SPEC["DROP_PATH_RATE"] == 0.2
    assert S3_SPEC["WINDOW_SIZE"] == [7] * 4 and S3_W14_SPEC["WINDOW_SIZE"] == [14, 14, 14, 7]
    assert {k: v for k, v in S3_W14_SPEC.items() if k != "WINDOW_SIZE"} == \
        {k: v for k, v in S3_SPEC.items() if k != "WINDOW_SIZE"}
    assert engine.CVT_SPECS["cvt_s3"] == dict(cvt_spec=S3_SPEC, drop_path_rate=0.2)
    assert engine.CVT_SPECS["cvt_s3_w14"] == dict(cvt_spec=S3_W14_SPEC, drop_path_rate=0.2)


def test_parameter_count():
    """the s3 backbone (no classification head, as in pre-training): 22.6 M parameters"""
    from esvit_b200 import cvt_v4_transformer as CV
    m = CV.cvt(CV.S3_SPEC)
    assert round(sum(p.numel() for p in m.parameters()) / 1e6, 1) == 22.6


@pytest.mark.parametrize("spec", [dict(NUM_HEADS=[2, 2, 3, 4]), dict(NUM_HEADS=[4, 8, 12, 16]),
                                  dict(NUM_HEADS=[1, 1, 1, 1])])
def test_head_dims_other_than_one_of_32_or_64_raise(spec):
    """mixed head dims (32 / 64 / 64 / 64), head dim 16, and head dims 64 / 128 / 192 / 256"""
    from esvit_b200 import cvt_v4_transformer as CV
    from oracle import make_golden_cvt as MG
    with pytest.raises(NotImplementedError, match="one head dim per model, 32 or 64"):
        CV.cvt(dict(MG.SPEC, **spec))


@pytest.mark.parametrize("yaml_name", ["s3.yaml", "win_size/s3.yaml"])
def test_reference_yaml_and_state_dict_load_strict(yaml_name):
    """get_cls_model serves the reference's s3 yaml files unchanged, and the reference CvT built from them loads with
    strict=True"""
    from functools import partial

    import yaml

    from esvit_b200 import cvt_v4_transformer as CV
    from oracle import reference_import as R
    path = os.path.join(R.REF_ROOT, "experiments", "imagenet", "cvt_v4", yaml_name)
    if not (R.available() and os.path.isfile(path)):
        pytest.skip("the reference is not installed under oracle/_ref/")
    with open(path) as f:
        cfg = yaml.safe_load(f)
    spec = cfg["MODEL"]["SPEC"]
    assert spec == (CV.S3_SPEC if yaml_name == "s3.yaml" else CV.S3_W14_SPEC)
    config = types.SimpleNamespace(MODEL=types.SimpleNamespace(SPEC=spec, NUM_CLASSES=0))
    net = CV.get_cls_model(config)
    R.load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import cvt_v4_transformer as ref_cvt
        ref = ref_cvt.CvT(num_classes=0, act_layer=ref_cvt.QuickGELU, norm_layer=partial(ref_cvt.LayerNorm, eps=1e-5),
                          init="trunc_norm", use_dense_prediction=False, spec=dict(spec))
    sd = ref.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(sd, strict=True)
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert net.num_features == 512
    assert net._stage(2)[1].window_size == spec["WINDOW_SIZE"][2]


def test_n_last_tap_plumbing_at_s3_depths(monkeypatch):
    """forward_return_n_last_blocks(x, n, avgpool, depth=[2, 2, 10, 4]) with every C-ABI call a no-op: the probe widths
    of s3's last n blocks, and the depth check"""
    from esvit_b200 import _lib, engine, ops
    monkeypatch.setattr(_lib, "call", lambda name, *a: None)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_chk", lambda t, dtype, name: None if t is None else t.contiguous())
    torch.manual_seed(0)
    for arch in ("cvt_s3", "cvt_s3_w14"):
        net = engine.build_network(dict(engine.CVT_SPECS[arch]), 256, True, False, True, 224, None).eval()
        depth = [2, 2, 10, 4]
        x = torch.randn(2, 3, 224, 224)
        for n, w in ((1, 512), (4, 4 * 512), (5, 256 + 4 * 512), (18, 2 * 64 + 2 * 128 + 10 * 256 + 4 * 512)):
            assert net.forward_return_n_last_blocks(x, n, False, depth).shape == (2, w), (arch, n)
        for n in (0, 19):
            with pytest.raises(ValueError):
                net.forward_return_n_last_blocks(x, n, False, depth)
        with pytest.raises(ValueError):
            net.forward_return_n_last_blocks(x, 1, False, [2, 2, 6, 2])
