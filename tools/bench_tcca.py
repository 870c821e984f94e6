"""Time the TCCA fit: TCCA(latent_dimensions=4) on standardised float32 JointData, 3 views x 128 features, n = 1e5.

    python tools/bench_tcca.py                 # the GPU fit, stage by stage, and the small comparison size
    python tools/bench_tcca.py --reference     # the reference's CPU time at the comparison size (needs the reference
                                               # tree; tensorly's parafac restated by oracle/tcca.py)

Prints one JSON line per measurement.  Each stage (moment pass, whiteners, Z, the Khatri-Rao contraction, the ALS
loop) ends in a device synchronise and is timed on the host clock, warm, median of ``--reps`` runs.  The contraction's
rate is 2 n prod(p) flop over its time; ``--peak`` (TFLOP/s, default the data-sheet 67 of the H100 SXM fp64 tensor
pipe) gives its share.  The reference builds an n x prod(p) array, so its comparison size is n = 2000, 3 x 32 (0.5 GB).
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

BIG = dict(n=100_000, dims=[128, 128, 128], k=4)
SMALL = dict(n=2000, dims=[32, 32, 32], k=4)


def host_views(n, dims):
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=len(dims), n_samples=n, n_features=dims, latent_dimensions=4, signal_to_noise=1.0,
                       random_state=0, dtype=np.float32)
    return [((v - v.mean(axis=0)) / v.std(axis=0, ddof=1)).astype(np.float32) for v in views]


def reference():
    from oracle import refshim

    refshim.install()
    import cca_zoo.linear._tcca as ref_tcca

    from oracle import tcca as O

    ref_tcca.parafac = O.parafac
    views = host_views(SMALL["n"], SMALL["dims"])
    t0 = time.perf_counter()
    ref_tcca.TCCA(latent_dimensions=SMALL["k"]).fit(views)
    print(json.dumps({"what": "reference_fit_s", **SMALL, "seconds": time.perf_counter() - t0}))


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


def stages(cfg, reps, peak):
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.linear import TCCA
    from cca_zoo_b200.linear._tcca import random_start_columns

    n, dims, k = cfg["n"], cfg["dims"], cfg["k"]
    views = [torch.from_numpy(v).cuda() for v in host_views(n, dims)]
    est = TCCA(latent_dimensions=k)
    est.fit(views)                                          # warm-up of every shape
    _, fit_s = _timed(lambda: est.fit(views), reps)
    dev = views[0].device
    mom, t_mom = _timed(lambda: est._local_moments(views, dev), reps)
    C, _, _ = est._covariance_stage(mom[0], n, dims, torch.float32, True)
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    S, t_white = _timed(lambda: [est._whitener(C[off[i]:off[i + 1], off[i]:off[i + 1]], 0.0)
                                 for i in range(len(dims))], reps)
    Z, t_z = _timed(lambda: [est._whitened(v, s, i) for i, (v, s) in enumerate(zip(views, S))], reps)
    M, t_kr = _timed(lambda: ops.tcca_moment(Z), reps)
    rand = random_start_columns(dims, k, None)
    st, t_als = _timed(lambda: ops.tcca_fit(M, dims, k, ops.TCCA_MAX_ITER, rand=rand), reps)
    iters = int(st[0].item())
    flop = 2.0 * n * float(np.prod(dims))
    print(json.dumps({"what": "tcca_fit", **cfg, "fit_s": fit_s, "moments_s": t_mom, "whiten_s": t_white,
                      "z_s": t_z, "contraction_s": t_kr, "contraction_tflops": flop / t_kr / 1e12,
                      "contraction_share_of_peak": flop / t_kr / 1e12 / peak, "peak_tflops_assumed": peak,
                      "als_s": t_als, "als_iters": iters}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--peak", type=float, default=67.0)
    a = ap.parse_args()
    if a.reference:
        reference()
        return
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    print(json.dumps({"what": "gpu", "nvidia_smi": q.stdout.strip()}))
    stages(BIG, a.reps, a.peak)
    stages(SMALL, a.reps, a.peak)


if __name__ == "__main__":
    main()
