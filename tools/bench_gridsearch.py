"""Time GridSearchCV's two routes on the same seeded data: rCCA, 2 views x 256 features (float32), n = 2e5, a grid of
10 ``c`` values, 5 folds.

    python tools/bench_gridsearch.py                # the moment route and the generic route on the GPU
    python tools/bench_gridsearch.py --reference    # the reference's GridSearchCV on the host CPUs as well (needs the
                                                    # reference tree)

The generic route is what the reference does, on this package's estimators: sklearn's GridSearchCV over a
view-splitting wrapper, one fit and one score per (candidate, fold).  The moment route reads the data once for all rows
and once per fold's test rows, fits every candidate from the moments and scores each fold's candidates in one call.
Each route is run once to warm up, then timed ``--reps`` times on the host clock with a device synchronise before
every clock read; the median is reported.  The split scores of the two routes are compared, and the card's name and
power limit are read in the same run.  Prints one JSON line.
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

N, DIMS, FOLDS = 200_000, (256, 256), 5
GRID = {"c": [float(c) for c in np.linspace(0.0, 0.9, 10)]}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def data():
    from cca_zoo_b200.datasets import joint_data

    return joint_data(n_views=2, n_samples=N, n_features=list(DIMS), latent_dimensions=4, signal_to_noise=1.0,
                      random_state=0, dtype=np.float32)


def split_scores(gs):
    return np.array([gs.cv_results_[f"split{s}_test_score"] for s in range(FOLDS)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reference", action="store_true")
    args = ap.parse_args()
    views = data()
    out = {"workload": f"rCCA, widths {list(DIMS)} float32, n = {N}, {len(GRID['c'])} c values, {FOLDS} folds"}
    if args.reference:
        from oracle import refshim

        refshim.install()
        from cca_zoo.linear import rCCA as RefRCCA
        from cca_zoo.model_selection import GridSearchCV as RefGridSearchCV

        t0 = time.perf_counter()
        ref = RefGridSearchCV(RefRCCA(), GRID, cv=FOLDS).fit(views)
        out["reference_cpu_s"] = time.perf_counter() - t0
        out["reference_best_params"] = ref.best_params_
    import torch

    from cca_zoo_b200.linear import rCCA
    from cca_zoo_b200.model_selection import GridSearchCV

    def run(generic):
        gs = GridSearchCV(rCCA(), GRID, cv=FOLDS)
        if generic:
            gs._moment_route = lambda *a: (None, False)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gs.fit(views)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, gs

    times = {"moment": [], "generic": []}
    result = {}
    for rep in range(args.reps + 1):
        for route in ("moment", "generic"):          # alternated, so drift on a shared host hits both
            dt, gs = run(route == "generic")
            if rep:
                times[route].append(dt)
            result[route] = gs
    diff = float(np.abs(split_scores(result["moment"]) - split_scores(result["generic"])).max())
    out.update({
        "card": card(),
        "moment_route_s": float(np.median(times["moment"])),
        "generic_route_s": float(np.median(times["generic"])),
        "speedup": float(np.median(times["generic"]) / np.median(times["moment"])),
        "max_split_score_diff": diff,
        "best_params": result["moment"].best_params_,
        "same_best": result["moment"].best_params_ == result["generic"].best_params_,
        "reps": args.reps,
    })
    print(json.dumps(out))


if __name__ == "__main__":
    main()
