"""Time TCCALoss forward and forward + backward on the GPU against a torch-eager restatement of the reference
(eigh whitening, the n x k_1 x ... x k_m outer-product array through einsum, autograd), float64.

    python tools/bench_tccaloss.py [--out results/bench_tccaloss.json]

Shapes (n, m, k): (1024, 3, 16), (4096, 3, 64) and (4096, 4, 32).  The eager restatement keeps its n x k^m array
for the backward, so it runs only where that array takes at most 8 GB.  Times are CUDA-event medians of 20 calls
after 3 warm-up calls; the card's name and power limit are printed with them.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cca_zoo_b200.deep import TCCALoss  # noqa: E402

SHAPES = [(1024, 3, 16), (4096, 3, 64), (4096, 4, 32)]
EAGER_LIMIT = 8 << 30


def eager_loss(zs, eps):
    n = zs[0].shape[0]
    H = []
    for z in zs:
        zc = z - z.mean(0)
        S = zc.T @ zc / (n - 1) + eps * torch.eye(z.shape[1], dtype=z.dtype, device=z.device)
        lam, V = torch.linalg.eigh(S)
        H.append(zc @ (V @ torch.diag(lam.clamp(min=eps).rsqrt()) @ V.T))
    letters = "abcdefgh"[:len(H)]
    M = torch.einsum(",".join("z" + c for c in letters) + "->z" + letters, *H).mean(0)
    return -torch.linalg.norm(M.reshape(-1))


def timed(fn, reps=20, warm=3):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = []
    for n, m, k in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(n + m + k)
        zs = [torch.randn(n, k, device="cuda", dtype=torch.float64, generator=g).requires_grad_(True) for _ in range(m)]
        fn = TCCALoss(eps=1e-5)

        def fwd():
            with torch.no_grad():
                fn(zs)

        def fwd_bwd():
            fn(zs).backward()

        row = dict(n=n, m=m, k=k, flop_fwd=2.0 * n * k ** m, flop_bwd=2.0 * m * n * k ** m,
                   fwd_ms=timed(fwd), fwd_bwd_ms=timed(fwd_bwd))
        fn.check()
        row["gflops_fwd_bwd"] = (row["flop_fwd"] + row["flop_bwd"]) / row["fwd_bwd_ms"] / 1e6
        if n * k ** m * 8 <= EAGER_LIMIT:
            def efwd():
                with torch.no_grad():
                    eager_loss(zs, 1e-5)

            def efwd_bwd():
                eager_loss(zs, 1e-5).backward()

            row["eager_fwd_ms"] = timed(efwd, reps=5, warm=1)
            row["eager_fwd_bwd_ms"] = timed(efwd_bwd, reps=5, warm=1)
            with torch.no_grad():
                row["loss_rel_diff"] = abs(float(fn(zs)) - float(eager_loss(zs, 1e-5))) / abs(float(eager_loss(zs, 1e-5)))
            fn.check()
        rows.append(row)
        print(json.dumps(row))
    res = {"gpu": gpu, "rows": rows}
    print(json.dumps({"gpu": gpu}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
