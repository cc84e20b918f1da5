"""Exact weighted k-NN classification of frozen features on the esvit_b200 kernels (csrc/knn.cu).

``knn_classifier`` is a drop-in for ``eval_knn.knn_classifier`` (eval_knn.py:193-232): same arguments, top-1 / top-5
accuracy in percent as Python floats.  ``knn_topk`` is the neighbour search on its own.

The neighbours are the exact fp32 top-k of ``test @ train.T`` (ties to the lower train index) although the similarities
run on bf16 tensor cores: per chunk of test rows the bf16 GEMM writes S, the select kernel finds the k-th largest bf16
value tau of each row, rescores every column with S >= tau - 2 delta in fp32 and keeps the fp32 top-k.  delta bounds
the bf16 error (DESIGN.md §4.4), so no true neighbour can fall outside the candidates.  A row whose candidates overflow
the scratch buffer is rerun with a buffer of the size it reported; nothing is approximated.
"""
from __future__ import annotations

import math

import torch

from . import _lib, ops
from .ops import _p, _stream

Tensor = torch.Tensor

MAX_CLASSES = 11264            # class scores of one test row live in shared memory (csrc/knn.cu)
_CHUNK_BYTES = 1 << 30         # bf16 similarity chunk [rows, N_pad]
_SCRATCH_BYTES = 1 << 28       # candidate scratch (int32 index + fp32 value per slot)
_CAP_SLACK = 4096              # candidate slots per row beyond k before a row is rerun

# candidate statistics of the last knn_topk / knn_classifier call
last_stats = {"max_candidates": 0, "rerun_rows": 0, "chunks": 0}


def _features(name: str, t) -> Tensor:
    if not isinstance(t, Tensor) or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if t.dim() != 2 or t.shape[0] == 0:
        raise ValueError(f"{name} must be a non-empty [rows, dim] matrix, got {tuple(t.shape)}")
    return t.contiguous()


def _prep(x: Tensor, rows_pad: int):
    """bf16 copy zero-padded to rows_pad rows, fp32 row norms and their maximum"""
    R, D = x.shape
    xb = torch.empty(rows_pad, D, dtype=torch.bfloat16, device=x.device)
    norm = torch.empty(R, dtype=torch.float32, device=x.device)
    mx = torch.zeros(1, dtype=torch.float32, device=x.device)
    _lib.call("esvit_knn_prep", _p(x), _p(xb), _p(norm), _p(mx), R, rows_pad, D, _stream())
    return xb, norm, mx


def _select(S, a, b, a_norm, b_max, rows, nrows, k, cap, count, sims, idx):
    N, D = b.shape
    ci = torch.empty(nrows * cap, dtype=torch.int32, device=a.device)
    cv = torch.empty(nrows * cap, dtype=torch.float32, device=a.device)
    _lib.call("esvit_knn_select", _p(S), S.shape[1], _p(a), _p(b), _p(a_norm), _p(b_max), _p(rows), nrows, N, D, k, cap,
              _p(ci), _p(cv), _p(count), _p(sims), _p(idx), _stream())


@torch.no_grad()
def knn_topk(train_features: Tensor, test_features: Tensor, k: int):
    """-> (sims fp32 [M, k] sorted descending, idx int64 [M, k]): the exact fp32 top-k of test @ train.T per test row,
    ties broken by the lower train index."""
    train = _features("train_features", train_features)
    test = _features("test_features", test_features)
    N, D = train.shape
    M = test.shape[0]
    if test.shape[1] != D:
        raise ValueError(f"feature dims differ: train {D}, test {test.shape[1]}")
    if D % 8:
        raise ValueError(f"feature dim must be a multiple of 8, got {D}")
    if test.device != train.device:
        raise ValueError("train and test features must be on the same device")
    k = int(k)
    if not 1 <= k <= N:
        raise ValueError(f"k must be in [1, {N}] (number of train rows), got {k}")
    if N >= 2 ** 31:
        raise ValueError("more than 2^31 - 1 train rows")
    dev = train.device
    n_pad = -(-N // 8) * 8  # the GEMM's N % 8 == 0
    with torch.cuda.device(dev):
        bb, _, b_max = _prep(train, n_pad)
        ab, a_norm, _ = _prep(test, M)
        cap = min(N, k + _CAP_SLACK)
        mc = max(1, min(M, _CHUNK_BYTES // (2 * n_pad), _SCRATCH_BYTES // (8 * cap)))
        sims = torch.empty(M, k, dtype=torch.float32, device=dev)
        idx = torch.empty(M, k, dtype=torch.int64, device=dev)
        count = torch.empty(M, dtype=torch.int32, device=dev)
        max_cand, rerun, chunks = 0, 0, 0
        for r0 in range(0, M, mc):
            r1 = min(M, r0 + mc)
            S = ops.gemm(ab[r0:r1], bb)  # bf16 [r1 - r0, n_pad], the nn.Linear forward form
            args = (test[r0:r1], train, a_norm[r0:r1], b_max)
            outs = (count[r0:r1], sims[r0:r1], idx[r0:r1])
            _select(S, *args, None, r1 - r0, k, cap, *outs)
            cmax = int(count[r0:r1].max())  # one sync per chunk
            if cmax > cap:
                rows = torch.nonzero(count[r0:r1] > cap).view(-1).to(torch.int32)
                rerun += rows.numel()
                _select(S, *args, rows, rows.numel(), k, cmax, *outs)
            max_cand = max(max_cand, cmax)
            chunks += 1
    last_stats.update(max_candidates=max_cand, rerun_rows=rerun, chunks=chunks)
    return sims, idx


def _labels(name: str, t, n: int, dev) -> Tensor:
    if not isinstance(t, Tensor) or t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f"{name} must be an integer tensor")
    if t.numel() != n:
        raise ValueError(f"{name} has {t.numel()} entries for {n} feature rows")
    return t.reshape(-1).to(device=dev, dtype=torch.int64).contiguous()


@torch.no_grad()
def knn_classifier(train_features: Tensor, train_labels: Tensor, test_features: Tensor, test_labels: Tensor, k: int,
                   T: float, num_classes: int = 1000):
    """Weighted k-NN accuracy of eval_knn.py:193-232 -> (top1, top5) in percent.  Each of the k nearest train rows votes
    exp(similarity / T) for its class; a test row counts as a top-n hit when its class is among the n best scores, equal
    scores ordered by class (a stable descending sort).  The reference's unstable sort leaves the order of equal scores
    unspecified; it matters only when the true class has score 0 and fewer than 5 classes have a positive score."""
    train = _features("train_features", train_features)
    test = _features("test_features", test_features)
    num_classes = int(num_classes)
    if not 1 <= num_classes <= MAX_CLASSES:
        raise ValueError(f"num_classes must be in [1, {MAX_CLASSES}], got {num_classes}")
    T = float(T)
    if not (T > 0 and math.isfinite(T)):
        raise ValueError(f"temperature must be positive and finite, got {T}")
    dev = train.device
    ytr = _labels("train_labels", train_labels, train.shape[0], dev)
    yte = _labels("test_labels", test_labels, test.shape[0], dev)
    lo_hi = torch.stack([torch.stack(torch.aminmax(ytr)), torch.stack(torch.aminmax(yte))]).tolist()
    if min(lo_hi[0][0], lo_hi[1][0]) < 0 or max(lo_hi[0][1], lo_hi[1][1]) >= num_classes:
        raise ValueError(f"labels must lie in [0, {num_classes})")
    sims, idx = knn_topk(train, test, k)
    M = test.shape[0]
    with torch.cuda.device(dev):
        hits = torch.zeros(2, dtype=torch.int64, device=dev)
        _lib.call("esvit_knn_vote", _p(sims), _p(idx), _p(ytr), _p(yte), M, int(k), T, num_classes, _p(hits), _stream())
        top1, top5 = hits.tolist()
    return top1 * 100.0 / M, top5 * 100.0 / M
