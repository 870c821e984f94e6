"""Time the CCAR3 fit stage by stage: CCAR3(lambda_=0.05) on standardised float32 JointData.

    python tools/bench_ccar3.py                # the GPU fit of both workloads, stage by stage
    python tools/bench_ccar3.py --reference    # the reference on the host CPUs at the same shapes (needs the
                                               # reference tree; its ADMM capped at --ref-iters iterations)

Workloads: "wide" n = 1e5, widths [2048, 256], k = 8 (the moment pass dominates the data, the ADMM the solve) and
"p_gt_n" n = 2000, widths [8192, 128], k = 8 (the regime the row-sparse penalty is for).  Prints one JSON line per
measurement.  Each stage ends in a device synchronise and is timed on the host clock, warm, median of ``--reps``
runs: the moment pass, the fourth-power pass, Sy^-1/2, M and B0, the ADMM (total and per iteration; its rate is
2 p^2 q flop per iteration over the per-iteration time), and the SVD with the thin products and the host tail.
The whole ``fit`` is timed as well.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"wide": dict(n=100_000, dims=[2048, 256], k=8), "p_gt_n": dict(n=2000, dims=[8192, 128], k=8)}
LAMBDA = 0.05


def host_views(n, dims):
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=2, n_samples=n, n_features=dims, latent_dimensions=4, signal_to_noise=1.0,
                       random_state=0, dtype=np.float32)
    return [((v - v.mean(axis=0)) / v.std(axis=0, ddof=1)).astype(np.float32) for v in views]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def stages(views, k, device):
    """The fit's device stages in order, each ending in a synchronise; returns (stage -> seconds, ADMM info)."""
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.linear import CCAR3
    from cca_zoo_b200.linear._ccar3 import SQRT_INV_CUT, ledoit_wolf_shrinkage, rrr_tail

    est = CCAR3(latent_dimensions=k, lambda_=LAMBDA)
    t, out = time.perf_counter, {}

    def mark(name, t0):
        torch.cuda.synchronize()
        out[name] = t() - t0
        return t()

    t0 = t()
    dev = [torch.from_numpy(v).to(device) for v in views]
    mom, n, dims, in_dtype = est._local_moments(dev, device)
    C, dims, n = est._covariance_stage(mom, n, dims, in_dtype, True)
    t0 = mark("moments", t0)
    p, q = dims
    S = C * ((n - 1) / n)
    Sx, Sxy, Syy = S[:p, :p], S[:p, p:], S[p:, p:]
    Cc, mean = ops.covariance(mom, dims, n, center=True)
    Sc = (Cc[p:, p:] * ((n - 1) / n)).contiguous()
    norm4 = ops.row_norm4_sum(dev[1], mean[p:])
    h = torch.cat([ops.frobenius_norm(Sc), norm4, Sc.diagonal()]).cpu().numpy()
    s, mu = ledoit_wolf_shrinkage(float(h[0]) ** 2, float(h[2:].sum()), float(h[1]), n, q)
    t0 = mark("fourth_power", t0)
    Sy = Sc * (1.0 - s)
    Sy.diagonal().add_(s * mu)
    lam, Vt = ops.syevj(Sy)
    f = torch.where(lam > SQRT_INV_CUT, lam.abs().rsqrt(), torch.zeros_like(lam))
    Sinv = ops.gemm(Vt, ops.scale(Vt, rows=f), transa=True)
    t0 = mark("sy_inv_sqrt", t0)
    A = Sx.contiguous().clone()
    A.diagonal().add_(1.0 + 1e-8)
    Linv, _ = ops.potrf_inv_(A)
    M = ops.gemm(Linv, Linv, transa=True)
    B0 = ops.gemm(M, ops.gemm(Sxy, Sinv))
    t0 = mark("m_and_b0", t0)
    B, _, info = ops.ccar3_admm(M, B0, LAMBDA, 1.0, 1e-4, 10_000)
    t0 = mark("admm", t0)
    info = info.cpu().numpy()
    r = min(k, p, q)
    assert p >= q, "both workloads have p >= q: G = B in the one-sided Jacobi SVD"
    _, Vt0, U0t = ops.gesvj(B.T.contiguous())
    U0t, Vt0 = U0t[:r].contiguous(), Vt0[:r].contiguous()
    V0 = ops.gemm(Sinv, Vt0, transb=True)
    parts = [U0t, V0, ops.gemm(U0t, ops.gemm(Sx, U0t, transb=True)), ops.gemm(V0, ops.gemm(Syy, V0), transa=True),
             ops.gemm(U0t, ops.gemm(Sxy, V0))]
    hp = [x.cpu().numpy() for x in parts]
    rrr_tail(hp[0].T, hp[1], hp[2], hp[3], hp[4], k, 1e-8)
    mark("svd_and_tail", t0)
    return out, info


def gpu(reps):
    import torch

    from cca_zoo_b200.linear import CCAR3

    device = torch.device("cuda", 0)
    print(json.dumps({"card": card()}), flush=True)
    for name, w in WORKLOADS.items():
        views = host_views(w["n"], w["dims"])
        p, q = w["dims"]
        runs = [stages(views, w["k"], device) for _ in range(reps + 1)][1:]
        info = runs[-1][1]
        med = {s: float(np.median([r[0][s] for r in runs])) for s in runs[0][0]}
        iters = int(info[0])
        per_it = med["admm"] / max(iters, 1)
        fits = []
        for _ in range(reps + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            CCAR3(latent_dimensions=w["k"], lambda_=LAMBDA).fit(views)
            torch.cuda.synchronize()
            fits.append(time.perf_counter() - t0)
        print(json.dumps({"workload": name, "n": w["n"], "dims": w["dims"], "k": w["k"],
                          "stages_ms": {s: round(1e3 * v, 3) for s, v in med.items()},
                          "admm_iters": iters, "admm_stopped": bool(info[3]), "admm_ms_per_iter": round(1e3 * per_it, 4),
                          "admm_tflops": round(2.0 * p * p * q / per_it / 1e12, 2),
                          "fit_ms": round(1e3 * float(np.median(fits[1:])), 2)}), flush=True)


def reference(ref_iters):
    from oracle import refshim

    refshim.install()
    from cca_zoo.linear import CCAR3 as Ref

    for name, w in WORKLOADS.items():
        views = host_views(w["n"], w["dims"])
        t0 = time.perf_counter()
        est = Ref(latent_dimensions=w["k"], lambda_=LAMBDA, max_iter=ref_iters).fit(views)
        dt = time.perf_counter() - t0
        assert est.weights_[0].shape == (w["dims"][0], w["k"])
        print(json.dumps({"workload": name, "reference_fit_s": round(dt, 2), "reference_max_iter": ref_iters,
                          "cpus": os.cpu_count()}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--ref-iters", type=int, default=3)
    a = ap.parse_args()
    if a.reference:
        reference(a.ref_iters)
    else:
        gpu(a.reps)


if __name__ == "__main__":
    main()
