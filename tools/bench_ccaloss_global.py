"""Time the global-batch CCALoss step against the per-replica one, float32, at bench.py's ccaloss64 and ccaloss512
shapes (n = 4096 rows per rank, widths [64, 64] and [512, 512], eps 1e-5).

    python tools/bench_ccaloss_global.py [--out results/bench_ccaloss_global.json]

One GPU: the fused local step (ccab_ccaloss_fwd + ccab_ccaloss_bwd) against the split global stages (moment pass ->
ccab_ccaloss_fwd_moments -> ccab_ccaloss_bwd_global) with the exchange left out -- the overhead a multi-GPU user pays
besides the exchange itself.  Two GPUs (when present): the per-step time of CCALoss forward + backward, per-replica
against global_batch=True, with the exchange on NCCL and on the NVLS kernel.  Times are CUDA-event medians of 50
steps after 10 warm-up steps; the card's name and power limit are printed with them.
"""
from __future__ import annotations

import argparse
import datetime
import json
import os
import socket
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cca_zoo_b200 import ops  # noqa: E402
from cca_zoo_b200.deep import CCALoss  # noqa: E402
from cca_zoo_b200.deep.objectives import _resolve_precision  # noqa: E402

SHAPES = {"ccaloss64": [64, 64], "ccaloss512": [512, 512]}
N, EPS = 4096, 1e-5


def timed(fn, reps=50, warm=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def views(dims, device, seed=0):
    g = torch.Generator(device=device).manual_seed(seed)
    return [torch.randn(N, d, generator=g, device=device) for d in dims]


def one_gpu(dims):
    z1, z2 = views(dims, "cuda")
    prec = _resolve_precision("auto", [z1, z2])
    go = torch.ones(1, device="cuda")
    n_dev = torch.tensor([float(N)], dtype=torch.float64, device="cuda")

    def local():
        _, saved, _ = ops.ccaloss_fwd(z1, z2, EPS, prec)
        ops.ccaloss_bwd(z1, z2, saved, go)

    def split():
        mom = ops.moments([z1, z2], precision=prec)
        _, saved, _ = ops.ccaloss_fwd_moments(mom, n_dev, dims[0], dims[1], EPS, torch.float32)
        ops.ccaloss_bwd_global(z1, z2, saved, go)

    return {"precision": prec, "local_fused_ms": timed(local), "global_split_ms": timed(split)}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, exchange, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2",
                      CCAB_EXCHANGE=exchange)
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=dev, timeout=datetime.timedelta(seconds=120))
    try:
        res = {}
        for name, dims in SHAPES.items():
            zs = [z.requires_grad_(True) for z in views(dims, dev, seed=rank)]
            row = {}
            for route, glob in (("local_ms", False), ("global_ms", True)):
                fn = CCALoss(eps=EPS, global_batch=glob)
                row[route] = timed(lambda: fn(zs).backward())
                fn.check()
            res[name] = row
        if rank == 0:
            with open(out, "w") as f:
                json.dump(res, f)
    finally:
        dist.destroy_process_group()


def two_gpus(exchange, tmp):
    import torch.multiprocessing as mp

    out = os.path.join(tmp, f"two_gpu_{exchange}.json")
    mp.spawn(_worker, args=(_free_port(), exchange, out), nprocs=2, join=True)
    with open(out) as f:
        return json.load(f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {"gpu": gpu[0] if gpu else "unknown", "n_per_rank": N, "one_gpu": {}, "two_gpus": {}}
    print(f"# {result['gpu']}")
    for name, dims in SHAPES.items():
        r = one_gpu(dims)
        result["one_gpu"][name] = r
        print(f"{name:11s} 1 GPU  local fused {r['local_fused_ms']:.3f} ms  global split stages "
              f"{r['global_split_ms']:.3f} ms  ({r['precision']})")
    if torch.cuda.device_count() >= 2:
        import tempfile

        with tempfile.TemporaryDirectory() as tmp:
            for exchange in ("nccl", "nvls"):
                try:
                    r = two_gpus(exchange, tmp)
                except Exception as err:  # noqa: BLE001 -- NVLS needs multicast: report what could not run
                    result["two_gpus"][exchange] = f"not measured: {err}"
                    print(f"2 GPUs {exchange}: not measured ({err})")
                    continue
                result["two_gpus"][exchange] = r
                for name, row in r.items():
                    print(f"{name:11s} 2 GPUs {exchange}: per-replica {row['local_ms']:.3f} ms  global batch "
                          f"{row['global_ms']:.3f} ms per step")
    else:
        result["two_gpus"] = "not measured: fewer than 2 GPUs"
        print("2 GPUs: not measured (fewer than 2 GPUs)")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
