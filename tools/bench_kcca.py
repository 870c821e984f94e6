"""Time the KCCA fit: KCCA(latent_dimensions=8, c=0.1, kernel="rbf") on standardised JointData, 2 views x 256
features, n = 4096; with ``--model kgcca`` KGCCA(latent_dimensions=8, kernel="rbf") on 3 views x 256 features at
n = 4096; with ``--model ktcca`` KTCCA(latent_dimensions=4, kernel="rbf") on 3 views x 256 features at n = 320 and on
2 views x 256 features at n = 4096.

    python tools/bench_kcca.py                    # the GPU fit, stage by stage
    python tools/bench_kcca.py --reference 1024   # the reference's CPU fit at n = 1024 (needs the reference tree)
    python tools/bench_kcca.py --model kgcca      # KGCCA's stages; with --reference N the reference at n = N
    python tools/bench_kcca.py --model ktcca      # KTCCA's stages; with --reference N the reference at n = N, 3 views

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
KGCCA_CFG = dict(n=4096, dims=[256, 256, 256], k=8, c=0.1, kernel="rbf")
KTCCA_CFGS = [dict(n=320, dims=[256, 256, 256], k=4, c=0.1, kernel="rbf"),
              dict(n=4096, dims=[256, 256], k=4, c=0.1, kernel="rbf")]


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


def reference_other(model, n):
    """The reference's KGCCA or KTCCA CPU fit at n (KTCCA: tensorly's parafac restated by oracle/tcca.py)."""
    from oracle import refshim

    refshim.install()
    import cca_zoo.nonparametric._ktcca as ref_ktcca
    from cca_zoo.nonparametric import KGCCA as RefKGCCA

    from oracle import tcca as TC

    ref_ktcca.parafac = TC.parafac
    cfg = KGCCA_CFG if model == "kgcca" else KTCCA_CFGS[0]
    Est = RefKGCCA if model == "kgcca" else ref_ktcca.KTCCA
    views = host_views(n, cfg["dims"])
    t0 = time.perf_counter()
    Est(latent_dimensions=cfg["k"], c=cfg["c"], kernel=cfg["kernel"]).fit(views)
    print(json.dumps({"what": f"reference_{model}_fit_s", "n": n, "dims": cfg["dims"], "cpu_count": os.cpu_count(),
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


def _kernel_stages(est, views, reps):
    """Time the fit and the shared stages: the kernel matrices and their eigensolves."""
    from cca_zoo_b200.nonparametric import _kcca

    est.fit(views)                                          # warm-up of every shape
    _, fit_s = _timed(lambda: est.fit(views), reps)
    X, args = est.train_views_, est._kernel_args
    (K, knorm), t_k = _timed(lambda: _kcca.kernel_matrices(X, args), reps)
    (lams, V, sweeps), t_eig = _timed(lambda: _kcca.eigenbases(K, knorm), reps)
    del K
    lam_h = [lam.cpu().numpy() for lam in lams]
    return fit_s, t_k, t_eig, sweeps, lam_h, V


def stages_kgcca(reps):
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.nonparametric import KGCCA
    from cca_zoo_b200.nonparametric import _kcca, _kgcca

    cfg = KGCCA_CFG
    n, dims, k = cfg["n"], cfg["dims"], cfg["k"]
    views = [torch.from_numpy(v).cuda() for v in host_views(n, dims)]
    est = KGCCA(latent_dimensions=k, c=cfg["c"], kernel=cfg["kernel"])
    fit_s, t_k, t_eig, sweeps, lam_h, V = _kernel_stages(est, views, reps)
    g, _, _ = _kgcca.gcca_scales(lam_h, [cfg["c"]] * len(dims), [1.0] * len(dims), est.eps, n)
    gd = [torch.from_numpy(x).cuda() for x in g]

    def build_q():
        Q = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        for Vi, gi in zip(V, gd):
            ops.gemm(ops.scale(Vi, rows=gi), Vi, transa=True, beta=1.0, out=Q)
        return Q

    Q, t_q = _timed(build_q, reps)
    (_, _, q_sweeps), t_top = _timed(lambda: _kcca._syevj(Q, float(Q.abs().sum(dim=1).max().item()), "Q"), reps)
    print(json.dumps({"what": "kgcca_fit", **cfg, "fit_s": fit_s, "kernels_s": t_k, "kernel_syevj_s": t_eig,
                      "kernel_syevj_sweeps": sweeps, "Q_s": t_q, "Q_syevj_s": t_top, "Q_sweeps": q_sweeps}))


def stages_ktcca(reps):
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.linear._tcca import random_start_columns
    from cca_zoo_b200.nonparametric import KTCCA
    from cca_zoo_b200.nonparametric import _ktcca

    for cfg in KTCCA_CFGS:
        n, dims, k = cfg["n"], cfg["dims"], cfg["k"]
        views = [torch.from_numpy(v).cuda() for v in host_views(n, dims)]
        est = KTCCA(latent_dimensions=k, c=cfg["c"], kernel=cfg["kernel"], random_state=0)
        fit_s, t_k, t_eig, sweeps, lam_h, V = _kernel_stages(est, views, reps)
        d, _, _ = _ktcca.tensor_scales(lam_h, [cfg["c"]] * len(dims), est.eps)
        dd = [torch.from_numpy(x).cuda() for x in d]
        Z, t_z = _timed(lambda: [ops.gemm(ops.scale(Vi, rows=di), Vi, transa=True) for Vi, di in zip(V, dd)], reps)
        M, t_m = _timed(lambda: ops.tcca_moment(Z), reps)
        shape = [n] * len(dims)
        _, t_als = _timed(lambda: ops.tcca_fit(M, shape, k, ops.TCCA_MAX_ITER,
                                               rand=random_start_columns(shape, k, 0)), reps)
        print(json.dumps({"what": "ktcca_fit", **cfg, "fit_s": fit_s, "kernels_s": t_k, "kernel_syevj_s": t_eig,
                          "kernel_syevj_sweeps": sweeps, "Z_s": t_z, "moment_s": t_m, "cp_als_s": t_als,
                          "fit_info_iters": est._fit_info["iters"]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", type=int, default=0, help="time the reference's CPU fit at this n instead")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--peak", type=float, default=67.0)
    ap.add_argument("--model", choices=["kcca", "kgcca", "ktcca"], default="kcca")
    a = ap.parse_args()
    if a.reference:
        reference(a.reference) if a.model == "kcca" else reference_other(a.model, a.reference)
        return
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"what": "gpu", "nvidia_smi": q.stdout.strip()}))
    {"kcca": lambda: stages(a.reps, a.peak), "kgcca": lambda: stages_kgcca(a.reps),
     "ktcca": lambda: stages_ktcca(a.reps)}[a.model]()


if __name__ == "__main__":
    main()
