"""2-rank NCCL parity of the linear probe: LinearProbeStep AVG-all-reduces the classifier gradient when a process group
is initialised (DDP's semantics in eval_linear.py), so two ranks on the two halves of each batch reproduce one process on
the whole batch.  Skipped on a 1-GPU box."""
import os
import socket
import tempfile

import pytest
import torch

from helpers import rel

pytestmark = pytest.mark.gpu

D, C, B, STEPS = 2304, 1000, 64, 3


class _Features:
    def forward_return_n_last_blocks(self, x, n, avgpool, depths):
        return x.reshape(x.shape[0], -1)


def _data():
    g = torch.Generator().manual_seed(31)
    centres = torch.randn(16, D, generator=g)
    y = torch.randint(0, 16, (STEPS, B), generator=g)
    return centres[y] + torch.randn(STEPS, B, D, generator=g), y


def _train(rows, device):
    from esvit_b200 import probe
    x, y = _data()
    torch.manual_seed(0)
    clf = probe.LinearClassifier(D, C).to(device)
    opt = probe.ProbeSGD(clf.parameters(), 0.01, momentum=0.9, weight_decay=0)
    step = probe.LinearProbeStep(_Features(), clf, opt, 4, False, [])
    for s in range(STEPS):
        step(x[s, rows].to(device).reshape(-1, D, 1, 1).contiguous(), y[s, rows])
    torch.cuda.synchronize()
    return clf.linear.weight.detach().cpu(), clf.linear.bias.detach().cpu()


def _worker(rank, world, port, path):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        w0, b0 = torch.load(path)
        half = B // world
        w, b = _train(slice(rank * half, (rank + 1) * half), dev)
        d0 = (w0 - _init()[0]).double()
        assert rel(w - _init()[0], d0) < 1e-4, rel(w - _init()[0], d0)
        assert rel(b, b0) < 1e-4, rel(b, b0)
    finally:
        dist.destroy_process_group()


def _init():
    from oracle import probe as PR
    return PR.init_classifier(D, C, 0)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_probe_equals_single_process():
    import torch.multiprocessing as mp
    want = _train(slice(0, B), "cuda:0")
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "want.pt")
        torch.save(want, path)
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        mp.spawn(_worker, args=(2, port, path), nprocs=2, join=True)
