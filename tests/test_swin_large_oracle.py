"""CPU: the Swin-L / Swin-T W14 specs.  The oracle reproduces what the unmodified reference computed at Swin-L widths
(tests/golden/esvit_large.pt, written by oracle/make_golden_large.py), and engine.build_network holds the reference
SwinTransformer's parameters under its keys for both specs."""
import os
import warnings

import pytest
import torch

from helpers import GOLDEN, at_golden, load_golden
from oracle import losses as L
from oracle import step as ST
from oracle import make_golden_large as MGL
from oracle import swin as S

GOLDEN_LARGE = os.path.join(os.path.dirname(GOLDEN), "esvit_large.pt")


@pytest.fixture(scope="module")
def D():
    return load_golden(GOLDEN_LARGE)["dense"]


def test_oracle_matches_reference_at_swin_l_widths(D):
    """forward outputs, region indices, loss, gradients and centers of one DDINO step"""
    M = D["meta"]
    spec = S.SwinSpec(**M["spec"])
    assert spec.num_features == 1536 and tuple(spec.num_heads) == (6, 12, 24, 48)
    with torch.no_grad():
        s = S.multicrop_forward(D["crops"], D["state_dict"], spec)
        t = S.multicrop_forward(D["crops"][:2], D["state_dict"], spec)
    assert s[3] == D["s_npatch"] == [49, 9] and t[3] == D["t_npatch"]
    for a, k in zip(list(s[:3]) + list(t[:3]), ("s_cls", "s_region", "s_fea", "t_cls", "t_region", "t_fea")):
        assert torch.allclose(*at_golden(a, D[k]), atol=2e-5, rtol=1e-4), k
    B, ncrops = M["batch"], M["ncrops"]
    sf = torch.split(s[2], [49 * B] * 2 + [9 * B] * (ncrops - 2))
    tf = t[2].chunk(2)
    for (iq, v), ref in D["indices"].items():
        T = 49 if v < 2 else 9
        assert torch.equal(L.region_match(sf[v].view(B, T, -1), tf[iq].view(B, 49, -1)), ref), (iq, v)
    orc = ST.OracleStep(D["state_dict"], spec, ncrops, M["out_dim"], **M["hp"])
    loss = orc.step(D["crops"], epoch=0, keep_grads=True)
    assert abs(loss - D["losses"][0]) < 2e-5 * max(1.0, abs(D["losses"][0]))
    for k, g in D["grads_step0_full"].items():
        a, g = at_golden(orc.grads_step[k], g)
        assert torch.allclose(a, g, atol=1e-7 + 1e-4 * float(g.abs().max()), rtol=1e-3), k
    for k, (_, nrm) in D["grads_step0_stats"].items():
        assert abs(float(orc.grads_step[k].double().norm()) - nrm) < 1e-3 * nrm + 1e-9, k
    assert torch.allclose(orc.center, D["center_after"], atol=1e-6)
    assert torch.allclose(orc.center_grid, D["center_grid_after"], atol=1e-6)


@pytest.mark.parametrize("arch,ospec", [("swin_large_w7", MGL.SWIN_L_W7), ("swin_tiny_w14", MGL.SWIN_T_W14)])
def test_specs_match_oracle(arch, ospec):
    from esvit_b200 import engine
    spec = dict(engine.SWIN_SPECS[arch])
    spec.pop("drop_path_rate")
    assert spec == {k: list(v) if isinstance(v, tuple) else v for k, v in ospec.items()}


@pytest.mark.parametrize("arch", ["swin_large_w7", "swin_tiny_w14"])
def test_reference_state_dict_loads_strict(arch):
    """the reference SwinTransformer built from the spec's yaml values loads into engine.build_network's backbone with
    strict=True, and the DDINO heads sit on num_features"""
    from esvit_b200 import engine
    from oracle import reference_import as R
    if not R.available():
        pytest.skip("the reference is not installed under oracle/_ref/")
    spec = dict(engine.SWIN_SPECS[arch])
    ospec = S.SwinSpec(img_size=224, use_dense_prediction=True,
                       **{k: v for k, v in spec.items() if k != "drop_path_rate"})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = R.build_swin(ospec, 256, drop_path_rate=spec["drop_path_rate"])
    net = engine.build_network(spec, 256, True)
    sd = ref.state_dict()
    assert set(sd) == set(net.state_dict())
    net.load_state_dict(sd, strict=True)
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert ref.num_features == net.num_features == ospec.num_features
    if arch == "swin_large_w7":
        assert ospec.num_features == 1536 and sd["patch_embed.proj.weight"].shape == (192, 3, 4, 4)
        assert sd["layers.2.downsample.norm.weight"].shape == (3072,)
        assert sd["layers.3.blocks.1.attn.relative_position_bias_table"].shape == (169, 48)
    else:
        assert sd["layers.0.blocks.0.attn.relative_position_bias_table"].shape == (27 * 27, 3)
