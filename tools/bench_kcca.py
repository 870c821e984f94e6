"""Time the KCCA fit: KCCA(latent_dimensions=8, c=0.1, kernel="rbf") on standardised JointData, 2 views x 256
features, n = 4096.

    python tools/bench_kcca.py                    # the GPU fit, stage by stage
    python tools/bench_kcca.py --reference 1024   # the reference's CPU fit at n = 1024 (needs the reference tree)

Prints one JSON line per measurement.  Each stage (the kernel matrices, the two kernel eigensolves, T, the top-k
eigensolve) and the whole fit end in a device synchronise and are timed on the host clock, warm, median of ``--reps``
runs.  The kernel matrices' rate is 2 n^2 d flop per view (the X X^T product on the fp64 tensor pipe) over their
time; ``--peak`` (TFLOP/s, default the data-sheet 67 of the H100 SXM fp64 tensor pipe) gives its share.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CFG = dict(n=4096, dims=[256, 256], k=8, c=0.1, kernel="rbf")


def host_views(n, dims):
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=len(dims), n_samples=n, n_features=dims, latent_dimensions=4, signal_to_noise=1.0,
                       random_state=0)
    return [(v - v.mean(axis=0)) / v.std(axis=0, ddof=1) for v in views]


def reference(n):
    from oracle import refshim

    refshim.install()
    from cca_zoo.nonparametric import KCCA as RefKCCA

    views = host_views(n, CFG["dims"])
    t0 = time.perf_counter()
    RefKCCA(latent_dimensions=CFG["k"], c=CFG["c"], kernel=CFG["kernel"]).fit(views)
    print(json.dumps({"what": "reference_fit_s", "n": n, "dims": CFG["dims"], "cpu_count": os.cpu_count(),
                      "seconds": time.perf_counter() - t0}))


def _timed(fn, reps):
    import torch

    out, ts = None, []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts))


def stages(reps, peak):
    import torch

    from cca_zoo_b200.nonparametric import KCCA
    from cca_zoo_b200.nonparametric import _kcca

    n, dims, k = CFG["n"], CFG["dims"], CFG["k"]
    views = [torch.from_numpy(v).cuda() for v in host_views(n, dims)]
    est = KCCA(latent_dimensions=k, c=CFG["c"], kernel=CFG["kernel"])
    est.fit(views)                                          # warm-up of every shape
    _, fit_s = _timed(lambda: est.fit(views), reps)
    X, args = est.train_views_, est._kernel_args
    (K, knorm), t_k = _timed(lambda: _kcca.kernel_matrices(X, args), reps)
    (lams, U, sweeps), t_eig = _timed(lambda: _kcca.eigenbases(K, knorm), reps)
    lam_h = [lam.cpu().numpy() for lam in lams]
    beta, D, keep = _kcca.eigenbasis_scales(lam_h, [CFG["c"]] * len(dims), est.eps, n)
    idx = [torch.from_numpy(np.flatnonzero(kp)).cuda() for kp in keep]
    Uk = [u.index_select(0, ix) for u, ix in zip(U, idx)]
    dk = [torch.from_numpy(Di[kp].copy()).cuda() for Di, kp in zip(D, keep)]
    T, t_T = _timed(lambda: _kcca.whitened_matrix(Uk, dk), reps)
    (_, top_sweeps), t_top = _timed(lambda: _kcca.top_eigenvectors(T), reps)
    flop = 2.0 * n * n * sum(dims)
    print(json.dumps({"what": "kcca_fit", **CFG, "fit_s": fit_s, "kernels_s": t_k,
                      "kernels_tflops": flop / t_k / 1e12, "kernels_share_of_peak": flop / t_k / 1e12 / peak,
                      "peak_tflops_assumed": peak, "kernel_syevj_s": t_eig, "kernel_syevj_sweeps": sweeps,
                      "T_s": t_T, "T_order": int(T.shape[0]), "topk_syevj_s": t_top, "topk_sweeps": top_sweeps,
                      "fit_info": est._fit_info}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=int, default=0, help="time the reference's CPU fit at this n instead")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--peak", type=float, default=67.0)
    a = ap.parse_args()
    if a.reference:
        reference(a.reference)
        return
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"what": "gpu", "nvidia_smi": q.stdout.strip()}))
    stages(a.reps, a.peak)


if __name__ == "__main__":
    main()
