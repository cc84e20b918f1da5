"""CPU: the fp32 oracle (oracle/vil.py) against the reference fixture tests/golden/esvit_vil.pt, and the Vision
Longformer host-side pieces (esvit_b200.vision_longformer): the bicubic weight matrices against F.interpolate, the
relative-position bias plans against the reference's gather + interpolate, the configuration checks, a strict load of a
reference-shaped state_dict, and the same against the unmodified reference (skipped without the tree or einops)."""
import sys
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F

from esvit_b200 import vision_longformer as V
from oracle import losses as LO
from oracle import make_golden_vil as MG
from oracle import vil as O
from oracle.golden import at_golden, recipe

G = MG.load()


def _close(a, ref, atol=2e-5):
    a, r = at_golden(a, ref)
    assert torch.allclose(a, r, atol=atol, rtol=0), float((a - r).abs().max())


def test_oracle_forward_and_n_last_against_fixture():
    F_ = G["features"]
    with torch.no_grad():
        cls, region, npatch = O.forward_dense(F_["state_dict"], F_["crops"], iter(F_["modes"]), True)
        nl = O.n_last_blocks(F_["state_dict"], torch.cat(F_["crops"][:2]), G["n_last"])
    assert npatch == F_["npatch"] == [49, 9]
    _close(cls, F_["x_cls"])
    _close(region, F_["region"])
    _close(nl, F_["n_last"])


def test_oracle_training_steps_against_fixture():
    T0, TS = G["temps"]
    for name, C in G["train"].items():
        sd, x, nt = C["state_dict"], C["crops"], C["n_teacher_modes"]
        osd = {k: v.clone().requires_grad_(v.dtype.is_floating_point and not k.endswith("weight_g")) for k, v in sd.items()}
        with torch.no_grad():
            ot = O.multicrop_forward({k: v.detach() for k, v in osd.items()}, x[:2], C["dense"], iter(C["modes"][:nt]))
        os_ = O.multicrop_forward(osd, x, C["dense"], iter(C["modes"][nt:]))
        zero = torch.zeros(1, G["K"])
        loss = LO.ddino_loss(os_, ot, zero, zero, len(x), T0, TS) if C["dense"] else \
            LO.dino_loss(os_, ot, zero, len(x), T0, TS)
        loss.backward()
        assert abs(float(loss) - C["loss"]) <= 1e-5 * abs(C["loss"]), name
        for k, ref in C["grads"].items():
            a, r = at_golden(osd[k].grad, ref)
            assert torch.allclose(a, r, atol=1e-6, rtol=1e-4), (name, k)


def test_reference_shaped_state_dict_loads_strict():
    """the fixture's state_dict (recorded from the reference's MsViT: 241 keys for vil_2262, here the reduced arch) and
    one recorded in the layout of vil_2262 load into MsViT with strict=True"""
    m = V.msvit(dict(MG.ARGS), use_dense_prediction=True)
    m.head = m.head_dense = torch.nn.Identity()
    sd = G["features"]["state_dict"]
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    full = V.msvit()
    rec = recipe(full.state_dict())
    assert len(rec) == 241
    full.load_state_dict(O.seeded(rec, 0), strict=True)


@pytest.mark.parametrize("n_in,n_out", [(196, 36), (49, 9)])
def test_bicubic_matrix_matches_interpolate(n_in, n_out):
    A = V.bicubic_matrix(n_in, n_out / n_in)
    assert A.shape == (n_out, n_in)
    X = torch.randn(4, n_in, n_in)
    want = F.interpolate(X[None], scale_factor=n_out / n_in, mode='bicubic')[0].double()
    At = torch.from_numpy(A)
    got = At @ X.double() @ At.T
    assert float((got - want).abs().max()) < 5e-6


def _apply(plan, params):
    (rp, col, val), _, nrows = plan
    M = sp.csr_matrix((val.numpy().astype(np.float64), col.numpy(), rp.numpy()), shape=(nrows, sum(p.numel() for p in params)))
    return torch.from_numpy(M @ torch.cat([p.reshape(-1) for p in params]).double().numpy())


def test_dense_bias_plan_matches_gather_and_interpolate():
    torch.manual_seed(0)
    for m, Ns in ((V.Attention(384, 12, True, rpe=True, wx=14, wy=14, nglo=1), (197, 37)),
                  (V.Attention(768, 24, True, rpe=True, wx=7, wy=7, nglo=0), (49, 9))):
        params = [p for p in (m.local_relative_position_bias_table, getattr(m, "g2l_relative_position_bias", None),
                              getattr(m, "g2g_relative_position_bias", None)) if p is not None]
        (plan, offs) = V.bias_plan(m, Ns, "cpu")
        y = _apply(plan, [p.detach() for p in params])
        nH = m.num_heads
        for N, off in zip(Ns, offs):
            npatch = N - m.nglo
            loc = m.local_relative_position_bias_table.detach()[m.relative_position_index.view(-1)].view(
                m.wx * m.wy, m.wx * m.wy, nH)
            if npatch != m.wx * m.wy:
                loc = F.interpolate(loc.reshape(1, m.wx * m.wy, m.wx * m.wy, nH).permute(0, 3, 1, 2),
                                    scale_factor=npatch / (m.wx * m.wy), mode='bicubic').permute(0, 2, 3, 1)[0]
            b = loc.permute(2, 0, 1)
            if m.nglo:
                g2l, g2g = m.g2l_relative_position_bias.detach(), m.g2g_relative_position_bias.detach()
                top = torch.cat([g2g, g2l[0].unsqueeze(-1).expand(-1, -1, npatch)], -1)
                b = torch.cat([top, torch.cat([g2l[1].unsqueeze(1).expand(-1, npatch, -1), b], -1)], 1)
            got = y[off:off + b.numel()].view(b.shape)
            assert float((got - b.double()).abs().max()) < 1e-6


def test_sliding_chunk_index_and_plan():
    from oracle import vil_attn as OV
    torch.manual_seed(1)
    m = V.Long2DSCSelfAttention(96, 3, True, sharew=True, nglo=1, rpe=True, mode=1)
    assert m.relative_position_index.shape == (49, 441)
    Ns = (1 + 56 * 56, 1 + 24 * 24)
    (plan, offs) = V.bias_plan(m, Ns, "cpu")
    params = [m.local_relative_position_bias_table.detach(), m.g2l_relative_position_bias.detach(),
              m.g2g_relative_position_bias.detach()]
    y = _apply(plan, params)
    for N, (bo, bgo) in zip(Ns, offs):
        b, bg = OV.module_biases(m, N)
        assert torch.equal(y[bo:bo + b.numel()].view(b.shape).float(), b.detach())
        assert torch.equal(y[bgo:bgo + bg.numel()].view(bg.shape).float(), bg.detach())


@pytest.mark.parametrize("change,key", [
    (dict(arch=V.VIL_2262['arch'].replace('a0', 'a1', 1)), "ape"),
    (dict(arch=V.VIL_2262['arch'].replace('h3,d96', 'h2,d96')), "head dim"),
    (dict(arch=V.VIL_2262['arch'].replace('f7', 'f5', 1)), "key f"),
    (dict(arch=V.VIL_2262['arch'].replace('g1', 'g2', 1)), "key g"),
    (dict(arch=V.VIL_2262['arch'].replace('f7,a0', 'f7,a0,r1', 1)), "add_pooled"),
    (dict(arch=V.VIL_2262['arch'].rsplit('_', 1)[0]), "3-stage"),
    (dict(only_glo=True), "only_glo"),
    (dict(sharew=False), "sharew"),
    (dict(sw_exact=1), "sw_exact"),
    (dict(with_se='SE'), "with_se"),
    (dict(attn_type='performer'), "performer"),
])
def test_unserved_configurations_raise(change, key):
    with pytest.raises(NotImplementedError, match=key):
        V.msvit(dict(V.VIL_2262, **change))


def test_reference_state_dict_loads_strict():
    from oracle import reference_import as R
    if not R.available():
        pytest.skip("the reference is not installed under oracle/_ref/")
    pytest.importorskip("einops")
    R._install_shims()
    if R.REF_ROOT not in sys.path:
        sys.path.insert(0, R.REF_ROOT)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from models import vision_longformer as RV
        ref = RV.MsViT(num_classes=0, **V.VIL_2262)
    mine = V.msvit()
    sd = ref.state_dict()
    assert len(sd) == 241 and set(sd) == set(mine.state_dict())
    mine.load_state_dict(sd, strict=True)
    for k, v in mine.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert mine.layer_cfgs == ref.layer_cfgs and mine.out_planes == ref.out_planes == 768
    assert mine.Nglos == ref.Nglos and mine.num_layers == ref.num_layers
