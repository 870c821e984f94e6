"""Global-batch TCCALoss across real processes: two ranks, each with a row shard of the batch.

On one GPU both ranks share ``cuda:0`` and exchange through gloo (which reduces CUDA tensors; the NCCL-style pack /
all-reduce / unpack of the moment exchange runs, CCAB_EXCHANGE=nccl, then the all-reduce of the tensor buffer).  With
two GPUs the same checks run on NCCL, the second step under ``torch.cuda.set_sync_debug_mode("error")``.  Checked
against one process holding the whole batch: the losses (bit for bit across ranks), each rank's gradient rows, and a
DDP step whose parameter gradient is (1/2) of the full-batch gradient."""
import datetime
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

pytestmark = pytest.mark.gpu

N_ROWS = 300
SPLIT = 140           # rank 0 holds rows [0, 140), rank 1 the rest: both at least as many as the widths + 1

CASES = [[5, 4], [6, 5, 4], [16, 12, 8, 4]]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _data(widths, seed):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(N_ROWS, 3, generator=g, dtype=torch.float64)
    return [lat @ torch.randn(3, w, generator=g, dtype=torch.float64) + torch.randn(N_ROWS, w, generator=g,
                                                                                  dtype=torch.float64)
            for w in widths]


def _make(glob):
    from cca_zoo_b200.deep import TCCALoss

    return TCCALoss(eps=1e-5, precision="exact", global_batch=glob)


class _Encoders(nn.Module):
    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.a = nn.Linear(12, 5).double()
        self.b = nn.Linear(9, 4).double()
        self.c = nn.Linear(7, 3).double()
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64))

    def forward(self, x1, x2, x3):
        return [self.a(x1), self.b(x2), self.c(x3)]


def _inputs():
    g = torch.Generator().manual_seed(1)
    return [torch.randn(N_ROWS, d, generator=g, dtype=torch.float64) for d in (12, 9, 7)]


def _worker(rank, world, port, backend, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      CCAB_EXCHANGE="nccl")
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120), **kw)
    try:
        lo, hi = (0, SPLIT) if rank == 0 else (SPLIT, N_ROWS)
        res = {}
        for widths in CASES:
            zs = [z[lo:hi].to(dev).requires_grad_(True) for z in _data(widths, sum(widths))]
            fn = _make(True)
            for it in range(2):                  # the second step runs with the status recycled (and sync-checked)
                for z in zs:
                    z.grad = None
                if it == 1 and backend == "nccl":
                    torch.cuda.set_sync_debug_mode("error")
                try:
                    loss = fn(zs)
                    loss.backward()
                finally:
                    torch.cuda.set_sync_debug_mode(0)
            fn.check()
            res[str(widths)] = (loss.detach().cpu(), [z.grad.cpu() for z in zs])
        model = nn.parallel.DistributedDataParallel(_Encoders().to(dev), device_ids=[dev.index])
        xs = [x[lo:hi].to(dev) for x in _inputs()]
        _make(True)(model(*xs)).backward()
        res["ddp"] = [p.grad.cpu() for p in model.parameters()]
        torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _single_process():
    ref = {}
    for widths in CASES:
        zs = [z.cuda().requires_grad_(True) for z in _data(widths, sum(widths))]
        loss = _make(False)(zs)
        loss.backward()
        ref[str(widths)] = (loss.detach().cpu(), [z.grad.cpu() for z in zs])
    model = _Encoders().cuda()
    _make(False)(model(*(x.cuda() for x in _inputs()))).backward()
    ref["ddp"] = [p.grad.cpu() for p in model.parameters()]
    return ref


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


def _spawn_and_check(tmp_path, backend):
    mp.spawn(_worker, args=(2, _free_port(), backend, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt") for r in range(2))
    ref = _single_process()
    for widths in CASES:
        key = str(widths)
        (l0, g0), (l1, g1) = r0[key], r1[key]
        lref, gref = ref[key]
        assert torch.equal(l0, l1), f"{key}: the ranks' losses differ"
        assert abs(float(l0) - float(lref)) <= 1e-10 * abs(float(lref)), key
        for a, b, r in zip(g0, g1, gref):
            assert a.shape[0] == SPLIT and b.shape[0] == N_ROWS - SPLIT
            assert _rel(a, r[:SPLIT]) <= 1e-10 and _rel(b, r[SPLIT:]) <= 1e-10, key
    # the loss is shift invariant, so the bias gradients are 0 up to rounding: compare against the largest gradient
    scale = max(float(r.abs().max()) for r in ref["ddp"])
    for a, b, r in zip(r0["ddp"], r1["ddp"], ref["ddp"]):
        assert torch.equal(a, b)
        assert float((a - 0.5 * r).abs().max()) <= 1e-10 * scale, "DDP averages: (1/W) of the global-batch gradient"


def test_two_processes_on_one_gpu_gloo(tmp_path):
    _spawn_and_check(tmp_path, "gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_nccl(tmp_path):
    _spawn_and_check(tmp_path, "nccl")
