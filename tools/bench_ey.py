"""Time the Eckart-Young gradient fit: CCA_EY(latent_dimensions=16, c=0.1, learning_rate=1e-3) on standardised float32
JointData, n = 1e5, widths [1024, 1024].

    python tools/bench_ey.py                 # the GPU fit: full batch (1000 steps, tol=0) and batch sizes 512, 4096
    python tools/bench_ey.py --reference     # the reference's CPU time per step (needs the reference tree)

Prints one JSON line per measurement.  The full-batch line reports the whole fit (moment pass included) and the
steps alone (the ccab_ey_fit call, CUDA events); the mini-batch lines report the fit's wall time per step, the host's
index draws included.  ``--reference`` times 3 full-batch steps and 20 steps per batch size of the reference's loop
and extrapolates the full batch to 1000 steps.
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

N, DIMS, K = 100_000, [1024, 1024], 16
KW = dict(latent_dimensions=K, c=0.1, learning_rate=1e-3, tol=0.0, random_state=0)


def host_views():
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=2, n_samples=N, n_features=DIMS, latent_dimensions=4, signal_to_noise=0.5,
                       random_state=0, dtype=np.float32)
    return [((v - v.mean(axis=0)) / v.std(axis=0, ddof=1)).astype(np.float32) for v in views]


def reference():
    from oracle import refshim

    refshim.install()
    from cca_zoo.linear import CCA_EY

    views = host_views()
    for bs, steps in ((None, 3), (512, 20), (4096, 20)):
        est = CCA_EY(max_iter=steps, batch_size=bs, **KW)
        t0 = time.perf_counter()
        est.fit(views)
        dt = time.perf_counter() - t0
        line = {"impl": "reference-cpu", "batch_size": bs, "steps_timed": steps, "us_per_step": 1e6 * dt / steps}
        if bs is None:
            line["fit_1000_steps_s_extrapolated"] = dt / steps * 1000
        print(json.dumps(line), flush=True)


def gpu():
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.datasets import joint_data_device
    from cca_zoo_b200.linear import CCA_EY

    views = joint_data_device(n_views=2, n_samples=N, n_features=DIMS, latent_dimensions=4, signal_to_noise=0.5,
                              random_state=0, dtype=torch.float32)
    views = [(v - v.mean(dim=0)) / v.std(dim=0) for v in views]
    torch.cuda.synchronize()
    dev = torch.cuda.get_device_properties(0)
    info = {"gpu": dev.name}

    def timed_fit(**kw):
        est = CCA_EY(**KW, **kw)
        est.fit(views)                     # warm-up (library load, workspace allocation)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        est.fit(views)
        torch.cuda.synchronize()
        return est, time.perf_counter() - t0

    est, dt = timed_fit(max_iter=1000)
    # the steps alone: one ccab_ey_fit call of 1000 steps on the fit's covariance
    C, dims, n = est._fit_device(views)
    init = np.vstack(est.weights_)
    fit = ops.ey_fit(dims, init, 0.1, 1e-3, 0.9, 0.0, cov=C)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fit.run(1000)
    e1.record()
    e1.synchronize()
    steps_ms = e0.elapsed_time(e1)
    print(json.dumps({**info, "impl": "cuda", "batch_size": None, "steps": est._fit_info["iters"], "fit_s": dt,
                      "steps_ms": steps_ms, "us_per_step": 1e3 * steps_ms / 1000}), flush=True)
    for bs in (512, 4096):
        est, dt = timed_fit(max_iter=300, batch_size=bs)
        print(json.dumps({**info, "impl": "cuda", "batch_size": bs, "steps": est._fit_info["iters"],
                          "calls": est._fit_info["calls"], "fit_s": dt,
                          "us_per_step": 1e6 * dt / est._fit_info["iters"]}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true")
    args = ap.parse_args()
    reference() if args.reference else gpu()
