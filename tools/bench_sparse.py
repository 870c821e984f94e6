"""Benchmark of the sparse / ALS path: SCCA_PMD(tau=0.3, latent_dimensions=4) on n = 1e5 samples of two 1024-wide
float32 views that live in HBM.  Prints one JSON line per tolerance: tol = 0 (a fixed max_iter = 500 sweeps per
dimension) and the default tol = 1e-6.  Then one line each for ElasticCCA(alpha=0.01, l1_ratio=0.5),
SCCA_IPLS(alpha=0.01) and SCCA_IPLS() (alpha = 0: the eigendecomposition route) at the default tol: fit_ms and
ms_per_view_update = fit_ms / (2 x the sweeps of all dimensions), which includes the moment pass and the eigensolves.

    python tools/bench_sparse.py [--reps 10] [--warmup 3] [--no-cpu-baseline]

fit_ms: whole fit (moment pass, covariance, ALS call, result copy), median over reps after warm-up.
als_ms: CUDA events around ops.als_fit (the ccab_als_fit call: Gram copy, the persistent kernels and deflations, and
the 64 KB copy of the result), median.  g_bytes: bytes of G the kernels read (one read per sweep, the full passes at the
start and end of each dimension, the deflation's read and write), g_gbps against the 3.35 TB/s of HBM3 (G is 32 MB and
may stay in the 50 MB L2, so the rate can exceed it).  parity: max |W - W_restated| against
oracle.sparse.cov_als_fit on the same covariance.  cpu_baseline_ms: oracle.sparse.ref_als_fit (the reference algorithm
in data space, numpy) at the full size, default tol only.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    args = ap.parse_args()

    import numpy as np
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.datasets import joint_data_device
    from cca_zoo_b200.linear import SCCA_PMD
    from oracle import sparse as S

    if not torch.cuda.is_available():
        raise SystemExit("bench_sparse needs a CUDA device")
    n, dims, k = 100_000, [1024, 1024], 4
    views = joint_data_device(n_views=2, n_samples=n, n_features=dims, latent_dimensions=4, signal_to_noise=0.2,
                              random_state=0, dtype=torch.float32)
    name, power = card()
    D = sum(dims)
    for tol in (0.0, 1e-6):
        est = SCCA_PMD(tau=0.3, latent_dimensions=k, tol=tol, max_iter=500, random_state=0)
        fit_ms = []
        for r in range(args.warmup + args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            est.fit(views)
            torch.cuda.synchronize()
            if r >= args.warmup:
                fit_ms.append(1e3 * (time.perf_counter() - t0))
        C, dims_, n_total = est._fit_device(views)
        rng = np.random.default_rng(0)
        init = np.empty((k, D))
        for d in range(k):
            ws = [rng.standard_normal(p) for p in dims]
            init[d] = np.concatenate([w / np.linalg.norm(w) for w in ws])
        params = est._view_params(dims)
        als_ms = []
        for r in range(args.warmup + args.reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            W, iters = ops.als_fit(C, dims, n_total, "pmd", params, init, 500, tol)
            e.record()
            e.synchronize()
            if r >= args.warmup:
                als_ms.append(s.elapsed_time(e))
        sweeps = int(sum(iters))
        g_bytes = 8 * D * D * (sweeps + 2 * k + 2 * (k - 1))
        G = C.cpu().numpy() * (n_total - 1)
        W_ref, iters_ref = S.cov_als_fit(G, dims, n_total, "pmd", k, params=params, init=[
            [init[d, :dims[0]], init[d, dims[0]:]] for d in range(k)], max_iter=500, tol=tol)
        parity = float(np.abs(W - np.vstack(W_ref)).max())
        am = statistics.median(als_ms)
        line = {"workload": "SCCA_PMD(tau=0.3, k=4) n=1e5 d=[1024,1024] fp32 in HBM", "tol": tol,
                "fit_ms": round(statistics.median(fit_ms), 3), "als_ms": round(am, 3), "sweeps": iters,
                "sweeps_match_restatement": iters == iters_ref, "g_bytes": g_bytes,
                "g_gbps": round(g_bytes / (am * 1e-3) / 1e9, 1),
                "g_share_of_3350_gbps": round(g_bytes / (am * 1e-3) / 3.35e12, 3), "parity_max_abs": parity,
                "gpu": name, "power_limit": power}
        if tol > 0 and not args.no_cpu_baseline:
            host = [v.cpu().numpy() for v in views]
            t0 = time.perf_counter()
            _, it_cpu = S.ref_als_fit(host, "pmd", k, params=params, max_iter=500, tol=tol, random_state=0)
            line["cpu_baseline_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
            line["cpu_baseline"] = ("oracle.sparse.ref_als_fit (reference algorithm in data space, numpy, "
                                    "this host's CPUs)")
            line["cpu_baseline_sweeps"] = it_cpu
        print(json.dumps(line), flush=True)

    # ElasticCCA / SCCA_IPLS: the regression kinds, default tol
    from cca_zoo_b200.linear import SCCA_IPLS, ElasticCCA

    for est in (ElasticCCA(alpha=0.01, l1_ratio=0.5, latent_dimensions=k, random_state=0),
                SCCA_IPLS(alpha=0.01, l1_ratio=1.0, latent_dimensions=k, random_state=0),
                SCCA_IPLS(latent_dimensions=k, random_state=0)):
        fit_ms = []
        for r in range(args.warmup + args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            est.fit(views)
            torch.cuda.synchronize()
            if r >= args.warmup:
                fit_ms.append(1e3 * (time.perf_counter() - t0))
        iters = est._fit_info["iters"]
        fm = statistics.median(fit_ms)
        line = {"workload": f"{type(est).__name__}(alpha={est.alpha}, l1_ratio={est.l1_ratio}, k=4) n=1e5 "
                            "d=[1024,1024] fp32 in HBM", "tol": est.tol, "fit_ms": round(fm, 3), "sweeps": iters,
                "ms_per_view_update": round(fm / (2 * sum(iters)), 3), "gpu": name, "power_limit": power}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
