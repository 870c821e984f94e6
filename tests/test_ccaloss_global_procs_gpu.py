"""Global-batch deep objectives across real processes: two ranks, each with a row shard of the batch.

On one GPU both ranks share ``cuda:0`` and exchange through gloo (which reduces CUDA tensors; the NCCL-style
pack / all-reduce / unpack of ``parallel.allreduce_moments_lazy`` runs, CCAB_EXCHANGE=nccl).  With two GPUs the same
checks run on NCCL, and on the NVLS exchange kernel where the machine offers multicast, with the steps also run under
``torch.cuda.set_sync_debug_mode("error")``.  Checked against one process holding the whole batch: the losses (bit
for bit across ranks), each rank's gradient rows, and a DDP step whose parameter gradient is (1/2) of the full-batch
gradient."""
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


# (loss class, widths): the narrow fused kernels, the wide path, and the Python-assembled MCCA / GCCA stages
CASES = [("CCALoss", [5, 4]), ("CCALoss", [130, 96]), ("MCCALoss", [6, 5, 4]), ("GCCALoss", [4, 4, 4])]


def _make(kind, glob):
    from cca_zoo_b200 import deep

    return getattr(deep, kind)(eps=1e-5, precision="exact", global_batch=glob)


class _Encoders(nn.Module):
    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.a = nn.Linear(12, 5).double()
        self.b = nn.Linear(9, 4).double()
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64))

    def forward(self, x1, x2):
        return [self.a(x1), self.b(x2)]


def _inputs():
    g = torch.Generator().manual_seed(1)
    return torch.randn(N_ROWS, 12, generator=g, dtype=torch.float64), torch.randn(N_ROWS, 9, generator=g,
                                                                                   dtype=torch.float64)


def _worker(rank, world, port, backend, exchange, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      CCAB_EXCHANGE=exchange)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    kw = dict(device_id=dev) if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120), **kw)
    try:
        lo, hi = (0, SPLIT) if rank == 0 else (SPLIT, N_ROWS)
        res = {}
        for kind, widths in CASES:
            zs = [z[lo:hi].to(dev).requires_grad_(True) for z in _data(widths, len(widths) + sum(widths))]
            fn = _make(kind, True)
            for it in range(2):                  # the second step runs with the status recycled (and sync-checked)
                for z in zs:
                    z.grad = None
                if it == 1 and backend == "nccl" and kind != "GCCALoss":     # GCCALoss reads back by design
                    torch.cuda.set_sync_debug_mode("error")
                try:
                    loss = fn(zs)
                    loss.backward()
                finally:
                    torch.cuda.set_sync_debug_mode(0)
            if hasattr(fn, "check"):
                fn.check()
            res[f"{kind}{widths}"] = (loss.detach().cpu(), [z.grad.cpu() for z in zs])
        model = nn.parallel.DistributedDataParallel(_Encoders().to(dev), device_ids=[dev.index])
        x1, x2 = (x[lo:hi].to(dev) for x in _inputs())
        _make("CCALoss", True)(model(x1, x2)).backward()
        res["ddp"] = [p.grad.cpu() for p in model.parameters()]
        torch.save(res, os.path.join(out, f"rank{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _single_process():
    ref = {}
    for kind, widths in CASES:
        zs = [z.cuda().requires_grad_(True) for z in _data(widths, len(widths) + sum(widths))]
        loss = _make(kind, False)(zs)
        loss.backward()
        ref[f"{kind}{widths}"] = (loss.detach().cpu(), [z.grad.cpu() for z in zs])
    model = _Encoders().cuda()
    _make("CCALoss", False)(model(*(x.cuda() for x in _inputs()))).backward()
    ref["ddp"] = [p.grad.cpu() for p in model.parameters()]
    return ref


def _rel(a, b):
    return float((a - b).abs().max()) / float(b.abs().max())


def _spawn_and_check(tmp_path, backend, exchange):
    mp.spawn(_worker, args=(2, _free_port(), backend, exchange, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(tmp_path / f"rank{r}.pt") for r in range(2))
    ref = _single_process()
    for kind, widths in CASES:
        key = f"{kind}{widths}"
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
    _spawn_and_check(tmp_path, "gloo", "nccl")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("exchange", ["nccl", "auto"])
def test_two_gpus_nccl_and_nvls(tmp_path, exchange):
    _spawn_and_check(tmp_path, "nccl", exchange)
