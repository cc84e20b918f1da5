"""CPU: oracle.attn.selfattention reproduces what the UNMODIFIED reference's SwinTransformer.forward_selfattention
produced (tests/golden/esvit_attn.pt, written by oracle/make_golden_attn.py): list structure, shapes and values."""
import os

import pytest
import torch

from oracle import attn as A
from oracle import golden as GD
from oracle import swin as S

GOLDEN_ATTN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_attn.pt")


@pytest.fixture(scope="module")
def G():
    return A.load_golden_attn(GOLDEN_ATTN)


def test_fixture_is_small():
    assert os.path.getsize(GOLDEN_ATTN) < 1 << 20


def test_fixture_covers_the_geometries(G):
    assert sorted(G["cases"]) == ["w14_112", "w14_96", "w7_112", "w7_96"]
    for C in G["cases"].values():
        assert sorted(C["maps"]) == [1, 2]
        assert len(C["maps"][1]) == 1 and len(C["maps"][2]) == sum(C["spec"]["depths"])


@pytest.mark.parametrize("name", ["w7_112", "w7_96", "w14_112", "w14_96"])
def test_oracle_selfattention_matches_reference(G, name):
    C = G["cases"][name]
    spec = S.SwinSpec(**C["spec"])
    with torch.no_grad():
        for n, refs in C["maps"].items():
            o = A.selfattention(C["images"], C["state_dict"], spec, n)
            outs = [o] if n == 1 else o
            assert len(outs) == len(refs), n
            for i, (a, ref) in enumerate(zip(outs, refs)):
                a, r = GD.at_golden(a, ref)
                assert a.shape == r.shape, (n, i)
                assert torch.allclose(a, r, atol=2e-5, rtol=0), (n, i, float((a - r).abs().max()))
