"""Time the global-batch and 16-bit TCCALoss steps (forward + backward) at n = 4096 rows per rank, widths [64, 64, 64]
and [32, 32, 32, 32], eps 1e-5.

    python tools/bench_tccaloss_global.py [--out results/bench_tccaloss_global.json]

One GPU: the per-replica float32 step against the global-batch stages on the same float32 representations with both
exchanges left out (the body ``_TCCALossGlobalFn`` runs in a single process for 16-bit input) -- the overhead a
multi-GPU user pays besides the exchanges themselves; and bfloat16 representations against float32 ones.  Two GPUs
(when present): the per-step time of TCCALoss per-replica against global_batch=True over NCCL.  Times are CUDA-event
medians of 50 steps after 10 warm-up steps, the routes alternated over 3 rounds (the median of the round medians); the
card's name and power limit are printed with them.
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

from cca_zoo_b200.deep import TCCALoss  # noqa: E402
from cca_zoo_b200.deep.objectives import _LazyStatus, _TCCALossGlobalFn  # noqa: E402

SHAPES = {"tcca64x3": [64, 64, 64], "tcca32x4": [32, 32, 32, 32]}
N, EPS, ROUNDS = 4096, 1e-5, 3


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


def alternated(routes):
    """{name: fn} -> {name: median over ROUNDS of the per-round medians}, the routes alternated within each round."""
    runs = {k: [] for k in routes}
    for _ in range(ROUNDS):
        for k, fn in routes.items():
            runs[k].append(timed(fn))
    return {k: sorted(v)[len(v) // 2] for k, v in runs.items()}


def views(dims, device, seed=0, dtype=torch.float32):
    g = torch.Generator(device=device).manual_seed(seed)
    lat = torch.randn(N, 4, generator=g, device=device)
    return [(lat @ torch.randn(4, d, generator=g, device=device) + torch.randn(N, d, generator=g, device=device))
            .to(dtype).requires_grad_(True) for d in dims]


def one_gpu(dims):
    z32 = views(dims, "cuda")
    z16 = [z.detach().to(torch.bfloat16).requires_grad_(True) for z in z32]
    local = TCCALoss(eps=EPS)
    half = TCCALoss(eps=EPS)
    status = _LazyStatus("TCCALoss")

    def per_replica():
        local(z32).backward()

    def global_stages():                     # the global body, float32 input, no exchange
        _TCCALossGlobalFn.apply(EPS, "auto", status, False, None, False, *z32).backward()

    def bf16():
        half(z16).backward()

    res = alternated({"per_replica_f32_ms": per_replica, "global_stages_f32_ms": global_stages, "bf16_ms": bf16})
    local.check()
    half.check()
    status.check()
    return res


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, out):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2",
                      CCAB_EXCHANGE="nccl")
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=dev, timeout=datetime.timedelta(seconds=120))
    try:
        res = {}
        for name, dims in SHAPES.items():
            zs = views(dims, dev, seed=rank)
            fns = {"local_ms": TCCALoss(eps=EPS), "global_ms": TCCALoss(eps=EPS, global_batch=True)}
            res[name] = {k: timed(lambda fn=fn: fn(zs).backward()) for k, fn in fns.items()}
            for fn in fns.values():
                fn.check()
        if rank == 0:
            with open(out, "w") as f:
                json.dump(res, f)
    finally:
        dist.destroy_process_group()


def two_gpus(tmp):
    import torch.multiprocessing as mp

    out = os.path.join(tmp, "two_gpu_nccl.json")
    mp.spawn(_worker, args=(_free_port(), out), nprocs=2, join=True)
    with open(out) as f:
        return json.load(f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tccaloss_global: no CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {"gpu": gpu[0] if gpu else "unknown", "n_per_rank": N, "one_gpu": {}, "two_gpus": {}}
    print(f"# {result['gpu']}")
    for name, dims in SHAPES.items():
        r = one_gpu(dims)
        result["one_gpu"][name] = r
        print(f"{name:9s} 1 GPU  per-replica f32 {r['per_replica_f32_ms']:.3f} ms  global stages f32 (no exchange) "
              f"{r['global_stages_f32_ms']:.3f} ms  bf16 {r['bf16_ms']:.3f} ms")
    if torch.cuda.device_count() >= 2:
        import tempfile

        with tempfile.TemporaryDirectory() as tmp:
            r = two_gpus(tmp)
        result["two_gpus"]["nccl"] = r
        for name, row in r.items():
            print(f"{name:9s} 2 GPUs nccl: per-replica {row['local_ms']:.3f} ms  global batch {row['global_ms']:.3f} ms "
                  f"per step")
    else:
        result["two_gpus"] = "not measured: fewer than 2 GPUs"
        print("2 GPUs: not measured (fewer than 2 GPUs)")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
