"""Time the GFA fit: GFA(latent_dimensions=16, tol=0, max_iter=10000) on standardised float32 JointData, n = 1e5,
widths [1024, 1024].

    python tools/bench_gfa.py                 # the GPU fit, phase by phase
    python tools/bench_gfa.py --reference     # the reference's CPU time per iteration (needs the reference tree)

Prints one JSON line per measurement: the moment pass, the X^T z0 product and the loop (the ccab_gfa_fit call) on
CUDA events, and the host's posterior sampling (wall time).  ``--samples`` sets num_posterior_samples (default 10:
the reference's default of 1000 makes a 1000 x n x k array of z draws, 12.8 GB at this size).  ``--reference`` times
a few iterations of the reference's loop and extrapolates to max_iter.
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


def host_views():
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=2, n_samples=N, n_features=DIMS, latent_dimensions=4, signal_to_noise=0.5,
                       random_state=0, dtype=np.float32)
    return [((v - v.mean(axis=0)) / v.std(axis=0, ddof=1)).astype(np.float32) for v in views]


def reference(max_iter, samples):
    from oracle import refshim

    refshim.install()
    from cca_zoo.probabilistic import GFA

    views = host_views()
    steps = 5
    t0 = time.perf_counter()
    GFA(latent_dimensions=K, tol=0.0, max_iter=steps, num_posterior_samples=samples).fit(views)
    dt = time.perf_counter() - t0
    print(json.dumps({"impl": "reference-cpu", "iters_timed": steps, "ms_per_iter": 1e3 * dt / steps,
                      "fit_s_extrapolated": dt / steps * max_iter, "host_cores": os.cpu_count()}), flush=True)


def gpu(max_iter, samples):
    import torch

    from cca_zoo_b200 import ops
    from cca_zoo_b200.probabilistic import GFA

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    views = [torch.from_numpy(v).to(dev) for v in host_views()]
    est = GFA(latent_dimensions=K, tol=0.0, max_iter=max_iter, num_posterior_samples=samples)
    est.fit(views)                                    # warm-up: loads the library, compiles nothing
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    ev[0].record()
    mom, n_local, dims, in_dtype = est._local_moments(views, dev)
    C, dims, n = est._covariance_stage(mom, n_local, dims, in_dtype, True)
    ev[3].record()
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    G = C.mul(n - 1)
    gdiag, cdiag = G.diagonal().cpu().numpy(), C.diagonal().cpu().numpy()
    y_const = np.array([gdiag[off[i]:off[i + 1]].sum() for i in range(2)])
    datavar = np.array([cdiag[off[i]:off[i + 1]].sum() for i in range(2)])
    rng = np.random.default_rng(0)
    z0 = rng.standard_normal((n, K))
    torch.cuda.synchronize()
    ev[1].record()
    XtZ0 = est._xt_z0(views, z0, off)
    ev[2].record()
    fit = ops.gfa_fit(dims, G, n, XtZ0, z0.T @ z0, datavar, y_const, 0.0, True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fit.run(max_iter)
    e1.record()
    st = fit.result()
    loop_ms = e0.elapsed_time(e1)
    z = est._latent_mean(views, st["B"], off)
    t1 = time.perf_counter()
    a_ard = 1e-14 + np.array(dims) / 2.0
    a_tau = 1e-14 + n * np.array(dims) / 2.0
    est._draw_posterior_samples(rng, z, st["cov_z"], [st["W"][off[i]:off[i + 1]] for i in range(2)],
                                list(st["cov_w"]), a_ard, list(st["b_ard"]), a_tau, st["b_tau"], dims)
    post_s = time.perf_counter() - t1
    print(json.dumps({"impl": "cca_zoo_b200", "gpu": torch.cuda.get_device_name(dev), "n": N, "dims": DIMS, "k": K,
                      "moment_pass_ms": ev[0].elapsed_time(ev[3]), "xtz0_ms": ev[1].elapsed_time(ev[2]),
                      "loop_ms": loop_ms, "iters": st["iters"], "us_per_iter": 1e3 * loop_ms / st["iters"],
                      "n_components": st["k"], "posterior_samples": samples, "posterior_host_s": post_s}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--max-iter", type=int, default=10000)
    ap.add_argument("--samples", type=int, default=10)
    a = ap.parse_args()
    (reference if a.reference else gpu)(a.max_iter, a.samples)


if __name__ == "__main__":
    main()
