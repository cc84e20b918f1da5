"""2-rank NCCL parity of CvT's SyncBatchNorm path: after nn.SyncBatchNorm.convert_sync_batchnorm, the depthwise + BN op
(ops.DwBnFn) on each rank's half of two resolution groups gives the outputs, running statistics and (summed over ranks)
gradients of one process running the concatenated batch.  Skipped on a 1-GPU box."""
import os
import socket
import tempfile

import pytest
import torch
import torch.nn as nn

from helpers import rel

pytestmark = pytest.mark.gpu

C = 64
GEOS = [(4, 56, 56, 7), (6, 24, 24, 7)]   # (B, H, W, w) of the concatenated batch; rank r holds images [r*B/2, (r+1)*B/2)


def _groups(shard):
    from esvit_b200 import ops
    groups, r0, p0 = [], 0, 0
    for B, H, W, w in GEOS:
        B = B // 2 if shard else B
        Hp, Wp = ops.win_padded(H, W, w)
        groups.append((B, H, W, w, r0, p0))
        r0 += B * H * W
        p0 += B * Hp * Wp
    return tuple(groups)


def _inputs(device):
    g = torch.Generator().manual_seed(3)
    ys = [(torch.randn(B * H * W, C, generator=g) * 0.7 + 0.2).to(torch.bfloat16) for B, H, W, _ in GEOS]
    gos = []
    for B, H, W, w in GEOS:
        Hp, Wp = -(-H // w) * w, -(-W // w) * w
        gos.append(torch.randn(B * Hp * Wp, C, generator=g).to(torch.bfloat16))
    bn = nn.BatchNorm2d(C)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.1 * torch.randn(C, generator=g))
        bn.bias.copy_(0.1 * torch.randn(C, generator=g))
        bn.running_var.copy_(1 + torch.rand(C, generator=g))
    w = torch.randn(C, 1, 3, 3, generator=g) * 0.3
    return ys, gos, bn.to(device), w.to(device)


def _shard(ts, geos_rows, rank):
    """rows of this rank's half of every group"""
    out = []
    for t, (B, rows) in zip(ts, geos_rows):
        half = B // 2 * rows
        out.append(t[rank * half:(rank + 1) * half])
    return out


def _run(ys, gos, bn, w, groups, pg, device):
    from esvit_b200 import ops
    y = torch.cat(ys).to(device).requires_grad_(True)
    wp = w.detach().clone().requires_grad_(True)
    out = ops.DwBnFn.apply(y, wp, bn.weight, bn.bias, bn, groups, True, pg)
    out.backward(torch.cat(gos).to(device))
    return {"out": out.detach().cpu(), "dy": y.grad.cpu(), "dw": wp.grad.cpu(), "dgamma": bn.weight.grad.cpu(),
            "dbeta": bn.bias.grad.cpu(), "rm": bn.running_mean.cpu(), "rv": bn.running_var.cpu(),
            "nbt": int(bn.num_batches_tracked)}


def _worker(rank, world, port, path):
    import torch.distributed as dist
    from esvit_b200.cvt_v4_transformer import _sync_group
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        ys, gos, bn, w = _inputs(dev)
        sbn = nn.SyncBatchNorm.convert_sync_batchnorm(nn.Sequential(bn))[0].to(dev).train()
        pg = _sync_group(sbn)
        assert pg is not None
        padded = [-(-H // ww) * ww * -(-W // ww) * ww for _, H, W, ww in GEOS]
        r = _run(_shard(ys, [(B, H * W) for B, H, W, _ in GEOS], rank),
                 _shard(gos, [(B, p) for (B, _, _, _), p in zip(GEOS, padded)], rank), sbn, w, _groups(True), pg, dev)
        want = torch.load(path, map_location="cpu", weights_only=False)
        # this rank's rows of the output and of the input gradient
        for key, rows in (("out", padded), ("dy", [H * W for _, H, W, _ in GEOS])):
            parts, o = [], 0
            for (B, _, _, _), n in zip(GEOS, rows):
                parts.append(want[key][o + rank * (B // 2) * n:o + (rank + 1) * (B // 2) * n])
                o += B * n
            assert rel(r[key], torch.cat(parts)) < 1e-2, key
        for key in ("rm", "rv"):
            assert rel(r[key], want[key]) < 1e-5, key
        assert r["nbt"] == want["nbt"] == len(GEOS)
        # parameter gradients are local sums (DDP averages them afterwards): their sum over ranks is the full gradient
        for key in ("dw", "dgamma", "dbeta"):
            t = r[key].to(dev)
            dist.all_reduce(t)
            assert rel(t.cpu(), want[key]) < 1e-3, key
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_sync_batchnorm_equals_single_process():
    import torch.multiprocessing as mp
    ys, gos, bn, w = _inputs("cuda:0")
    want = _run(ys, gos, bn.train(), w, _groups(False), None, "cuda:0")
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "want.pt")
        torch.save(want, path)
        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        mp.spawn(_worker, args=(2, port, path), nprocs=2, join=True)
