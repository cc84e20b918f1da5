"""CPU: oracle/eval.py reproduces what the UNMODIFIED reference's evaluation code produced (tests/golden/esvit_eval.pt,
written by oracle/make_golden_eval.py): forward_return_n_last_blocks features and eval_knn.knn_classifier accuracies."""
import os

import pytest
import torch

from oracle import eval as E
from oracle import swin as S

GOLDEN_EVAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "esvit_eval.pt")


@pytest.fixture(scope="module")
def G():
    return E.load_golden_eval(GOLDEN_EVAL)


def test_fixture_is_small():
    assert os.path.getsize(GOLDEN_EVAL) < 1 << 20


def test_oracle_n_last_blocks_matches_reference(G):
    P = G["probe"]
    spec = S.SwinSpec(**P["spec"])
    assert sorted(P["features"]) == [1, 2, 3, 6]
    with torch.no_grad():
        for n, ref in P["features"].items():
            o = E.n_last_blocks(P["images"], P["state_dict"], spec, n)
            assert o.shape == ref.shape, n
            assert torch.allclose(o, ref, atol=2e-5, rtol=0), (n, float((o - ref).abs().max()))


def test_oracle_knn_classifier_matches_reference(G):
    K = G["knn"]
    xtr, ytr, xte, yte = K["features"]
    for k in K["ks"]:
        assert E.knn_classifier(xtr, ytr, xte, yte, k, K["T"], K["params"]["num_classes"]) == K["accuracy"][k], k


def test_oracle_knn_indices_match_reference(G):
    K = G["knn"]
    xtr, _, xte, _ = K["features"]
    _, idx = E.knn_topk(xtr, xte, K["idx"].shape[1])
    assert torch.equal(idx, K["idx"])
