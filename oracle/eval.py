"""Functional fp32 oracle of the evaluation entry points.

TEST INFRASTRUCTURE — see ``oracle/__init__.py``.  Citations are into the reference repository.

  * ``n_last_blocks``: SwinTransformer.forward_return_n_last_blocks (models/swin_transformer.py:799-837) over
    BasicLayer.forward_with_features (:483-490), built on ``oracle.swin``;
  * ``knn_topk`` / ``knn_vote`` / ``knn_classifier``: eval_knn.py:193-232, with the neighbour order made explicit
    (fp32 similarity descending, ties to the lower train index) and the class order of the reference's
    ``probs.sort(1, True)`` as a stable descending sort;
  * ``clustered_features``: the seeded, L2-normalised synthetic features of the k-NN fixture and tests.
"""
from __future__ import annotations

import ast
import os

import torch
import torch.nn.functional as F

from . import golden as GD
from . import reference_import as R
from . import swin as S

Tensor = torch.Tensor


def n_last_blocks(x: Tensor, sd, spec: S.SwinSpec, n: int, prefix: str = "") -> Tensor:
    """[B, sum C_i]: token means of the last n block outputs in execution order; last-stage outputs pass through the
    final norm first (:825-829)."""
    x = S.patch_embed(x, sd, prefix + "patch_embed", spec.patch_size)
    last = len(spec.depths) - 1
    start = sum(spec.depths) - n
    out, b = [], 0
    for i, depth in enumerate(spec.depths):
        for j in range(depth):
            ws, shift = spec.block_window_shift(i, j)
            x = S.swin_block(x, sd, f"{prefix}layers.{i}.blocks.{j}", spec.num_heads[i], ws, shift)
            if b >= start:
                y = S.layer_norm(x, sd, prefix + "norm") if i == last else x
                out.append(y.mean(dim=1))  # AdaptiveAvgPool1d(1) over tokens (:831)
            b += 1
        if i < last:
            x = S.patch_merging(x, sd, f"{prefix}layers.{i}.downsample")
    return torch.cat(out, dim=-1)


def knn_topk(train: Tensor, test: Tensor, k: int, chunk: int = 256):
    """(sims [M, k], idx [M, k]) of test @ train.T (eval_knn.py:209-210): fp32 descending, ties to the lower index."""
    sims, idx = [], []
    for r0 in range(0, test.shape[0], chunk):
        s = torch.mm(test[r0:r0 + chunk], train.t())
        v, i = torch.sort(s, dim=1, descending=True, stable=True)
        sims.append(v[:, :k])
        idx.append(i[:, :k])
    return torch.cat(sims), torch.cat(idx)


def knn_vote(sims: Tensor, idx: Tensor, train_labels: Tensor, test_labels: Tensor, T: float, num_classes: int):
    """(top1 hits, top5 hits) of the weighted vote (eval_knn.py:211-227): each neighbour adds exp(s / T) to its class."""
    w = sims.div(T).exp()
    probs = torch.zeros(sims.shape[0], num_classes, dtype=w.dtype, device=w.device)
    probs.scatter_add_(1, train_labels[idx], w)
    pred = torch.sort(probs, dim=1, descending=True, stable=True).indices
    correct = pred[:, :5].eq(test_labels.view(-1, 1))
    return int(correct[:, 0].sum()), int(correct.sum())


def knn_classifier(train_features, train_labels, test_features, test_labels, k, T, num_classes=1000):
    """eval_knn.knn_classifier -> (top1, top5) in percent."""
    sims, idx = knn_topk(train_features, test_features, k)
    top1, top5 = knn_vote(sims, idx, train_labels, test_labels, T, num_classes)
    M = test_labels.shape[0]
    return top1 * 100.0 / M, top5 * 100.0 / M


def clustered_features(seed: int, n_train: int, n_test: int, dim: int, num_classes: int, noise: float = 1.0,
                       device="cpu"):
    """L2-normalised features around num_classes seeded unit centres (eval_knn.py:132-133 normalises them):
    (train fp32 [n_train, dim], train labels int64, test fp32 [n_test, dim], test labels int64)."""
    g = torch.Generator(device=device).manual_seed(seed)
    centres = F.normalize(torch.randn(num_classes, dim, generator=g, device=device), dim=1)

    def draw(n):
        y = torch.randint(0, num_classes, (n,), generator=g, device=device)
        x = centres[y] + torch.randn(n, dim, generator=g, device=device) * (noise / dim ** 0.5)
        return F.normalize(x, dim=1), y

    xtr, ytr = draw(n_train)
    xte, yte = draw(n_test)
    return xtr, ytr, xte, yte


def reference_knn_classifier():
    """The UNMODIFIED eval_knn.knn_classifier, AST-extracted (the module imports torchvision datasets).  It calls .cuda()
    on a scratch tensor (eval_knn.py:198): on CPU, run it under ``cpu_cuda_shim``."""
    path = os.path.join(R.REF_ROOT, "eval_knn.py")
    tree = ast.parse(open(path).read())
    env = {"torch": torch}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name == "knn_classifier":
            exec(compile(ast.Module([node], []), path, "exec"), env)
    return env["knn_classifier"]


class cpu_cuda_shim:
    """Tensor.cuda -> identity for a CPU run of the reference's knn_classifier."""

    def __enter__(self):
        self.saved = torch.Tensor.cuda
        torch.Tensor.cuda = lambda t, *a, **kw: t
        return self

    def __exit__(self, *exc):
        torch.Tensor.cuda = self.saved


def probe_images(batch: int, size: int, seed: int) -> Tensor:
    return torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(seed))


def load_golden_eval(path: str) -> dict:
    """tests/golden/esvit_eval.pt with its seeded weights, images and k-NN features rebuilt"""
    G = torch.load(path, map_location="cpu", weights_only=False)
    P, K = G["probe"], G["knn"]
    P["state_dict"] = GD.seeded_state_dict(P["state_recipe"], P["weight_seed"])
    P["images"] = probe_images(P["batch"], P["spec"]["img_size"], P["image_seed"])
    K["features"] = clustered_features(**K["params"])
    K["idx"] = K["idx"].long()
    return G
