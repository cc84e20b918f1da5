"""2-rank NCCL parity of the SyncBatchNorm DINO head: after nn.SyncBatchNorm.convert_sync_batchnorm, DINOHead(use_bn=True)
on each rank's half of the rows gives the outputs, running statistics and (summed over ranks) gradients of one process
running all rows.  Skipped on a 1-GPU box."""
import os
import socket
import tempfile

import pytest
import torch
import torch.nn as nn

from helpers import rel

pytestmark = pytest.mark.gpu

ROWS, IN_DIM, OUT_DIM = 640, 256, 1024
HEAD = dict(hidden_dim=512, bottleneck_dim=128)


def _inputs():
    from esvit_b200.vision_transformer import DINOHead
    torch.manual_seed(0)
    h = DINOHead(IN_DIM, OUT_DIM, use_bn=True, **HEAD)
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for m in h.modules():
            if isinstance(m, nn.BatchNorm1d):
                m.weight.copy_(1 + 0.1 * torch.randn(m.num_features, generator=g))
                m.bias.copy_(0.1 * torch.randn(m.num_features, generator=g))
    x = torch.randn(ROWS, IN_DIM, generator=g)
    go = torch.randn(ROWS, OUT_DIM, generator=g).to(torch.bfloat16)
    return h, x, go


def _run(h, x, go, device):
    h = h.to(device).train()
    out = h(x.to(device))
    out.backward(go.to(device))
    return {"out": out.detach().cpu(),
            "grads": {k: p.grad.detach().cpu() for k, p in h.named_parameters() if p.grad is not None},
            "buffers": {k: b.detach().cpu() for k, b in h.named_buffers()}}


def _worker(rank, world, port, path):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        h, x, go = _inputs()
        h = nn.SyncBatchNorm.convert_sync_batchnorm(h)
        assert sum(isinstance(m, nn.SyncBatchNorm) for m in h.modules()) == 2
        half = ROWS // world
        r = _run(h, x[rank * half:(rank + 1) * half], go[rank * half:(rank + 1) * half], dev)
        want = torch.load(path, map_location="cpu", weights_only=False)
        assert rel(r["out"], want["out"][rank * half:(rank + 1) * half]) < 1e-2
        for k, v in want["buffers"].items():
            if v.dtype == torch.long:
                assert torch.equal(r["buffers"][k], v), k
            else:
                assert rel(r["buffers"][k], v) < 1e-4, k
        # parameter gradients are local sums (DDP averages them afterwards): their sum over ranks is the full gradient
        for k, v in want["grads"].items():
            t = r["grads"][k].to(dev)
            dist.all_reduce(t)
            if k.endswith("mlp.0.bias") or k.endswith("mlp.3.bias"):   # removed by the BN that follows: about 0
                assert float(t.norm()) < 1e-3 * float(want["grads"]["mlp.0.weight"].norm()), k
            else:
                assert rel(t.cpu(), v) < 2e-2, k
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_sync_batchnorm_head_equals_single_process():
    import torch.multiprocessing as mp
    h, x, go = _inputs()
    want = _run(h, x, go, "cuda:0")
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "want.pt")
        torch.save(want, path)
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        mp.spawn(_worker, args=(2, port, path), nprocs=2, join=True)
