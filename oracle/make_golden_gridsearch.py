"""Generate tests/golden/reference_outputs_gridsearch.{npz,json} from the UNMODIFIED reference: GridSearchCV
(cca_zoo/model_selection/_search.py) on CPU.

    python oracle/make_golden_gridsearch.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  Every case records the reference's split scores, their mean, std and
rank, best_params_, best_score_ and the best estimator's score on a held-out set; the npz holds the seeded views the
cases run on.  A case is kept only when its best mean score beats the runner-up by at least 1e-6 relative, so that
best_params_ is decided by the data and not by rounding.  The npz is written with fixed zip timestamps and the json
with sorted keys, so a rerun reproduces both files byte for byte.
"""
from __future__ import annotations

import io
import json
import os
import sys
import warnings
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

from sklearn.model_selection import KFold, RepeatedKFold, ShuffleSplit  # noqa: E402

from cca_zoo import linear as ref  # noqa: E402
from cca_zoo.model_selection import GridSearchCV as RefGridSearchCV  # noqa: E402

N_TRAIN, N_TEST, DIMS = 150, 60, (10, 8, 6)
#: splitters by name (the GPU test rebuilds them from the same names)
SPLITTERS = {
    "int4": lambda: 4,
    "kfold_shuffle": lambda: KFold(4, shuffle=True, random_state=0),
    "shuffle_split": lambda: ShuffleSplit(3, test_size=0.3, random_state=0),
    "repeated_kfold": lambda: RepeatedKFold(n_splits=3, n_repeats=2, random_state=0),
}
# name, estimator class name, constructor kwargs, param grid, number of views, splitter name
CASES = [
    ("rcca_c", "rCCA", dict(latent_dimensions=2), {"c": [0.0, 0.1, 0.5, 0.9]}, 2, "int4"),
    ("rcca_perview_c", "rCCA", {}, {"c": [[0.1, 0.5], [0.5, 0.1], [0.9, 0.9]]}, 2, "kfold_shuffle"),
    ("cca_k", "CCA", {}, {"latent_dimensions": [1, 2, 3]}, 2, "shuffle_split"),
    ("pls_k", "PLS", {}, {"latent_dimensions": [1, 2]}, 2, "repeated_kfold"),
    ("mcca_3", "MCCA", dict(latent_dimensions=2), {"c": [0.1, 0.5, 0.9]}, 3, "int4"),
    ("gcca_3", "GCCA", {}, {"latent_dimensions": [1, 2], "c": [0.2, 0.6]}, 3, "kfold_shuffle"),
    # SCCA_PMD's tau leaves every split score of these views unchanged (a tie the filter drops): its grid is over k
    ("pmd_k", "SCCA_PMD", dict(random_state=0, tau=0.5), {"latent_dimensions": [1, 2]}, 2, "int4"),
    # ElasticCCA stops when the weights move less than tol; at its default 1e-6 the reference's own split scores sit
    # up to 1.4e-4 from the converged ones on these views, so the case runs both sides to tol = 1e-11 (5e-6 apart
    # from tol = 1e-9)
    ("elastic_alpha", "ElasticCCA", dict(random_state=0, tol=1e-11, max_iter=5000), {"alpha": [0.01, 0.1, 1.0]}, 2,
     "shuffle_split"),
    ("grid_list", "rCCA", {}, [{"c": [0.1]}, {"c": [0.5], "latent_dimensions": [2]}], 2, "repeated_kfold"),
    ("invalid_c", "rCCA", {}, {"c": [0.1, 2.0, 0.5]}, 2, "kfold_shuffle"),
]


def make_views():
    """Train and held-out views with two shared latent directions (float64)."""
    rng = np.random.default_rng(2024)
    n = N_TRAIN + N_TEST
    z = rng.standard_normal((n, 2))
    views = [z @ rng.standard_normal((2, p)) + rng.standard_normal((n, p)) for p in DIMS]
    return [v[:N_TRAIN] for v in views], [v[N_TRAIN:] for v in views]


def _plain(v):
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, np.generic):
        return v.item()
    return v


def run_case(est_name, kwargs, grid, m, splitter, train, test):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gs = RefGridSearchCV(getattr(ref, est_name)(**kwargs), grid, cv=SPLITTERS[splitter]()).fit(train[:m])
    r = gs.cv_results_
    n_splits = len([k for k in r if k.startswith("split") and k.endswith("_test_score")])
    return {
        "split_scores": np.array([r[f"split{s}_test_score"] for s in range(n_splits)]).T,   # candidates x splits
        "mean": np.asarray(r["mean_test_score"]), "std": np.asarray(r["std_test_score"]),
        "rank": np.asarray(r["rank_test_score"]),
        "best_params": {k: _plain(v) for k, v in gs.best_params_.items()},
        "best_score": float(gs.best_score_), "held_out_score": float(gs.score(test[:m])),
        "warnings": sorted({w.category.__name__ for w in rec
                            if w.category.__name__ in ("FitFailedWarning", "UserWarning")}),
    }


def write_npz(path, arrays):
    """np.savez without the wall-clock timestamps of the zip entries."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


def main():
    train, test = make_views()
    arrays = {}
    for i in range(len(DIMS)):
        arrays[f"train_{i}"], arrays[f"test_{i}"] = train[i], test[i]
    meta = {"n_train": N_TRAIN, "n_test": N_TEST, "dims": list(DIMS), "cases": {}, "dropped": []}
    for name, est_name, kwargs, grid, m, splitter in CASES:
        out = run_case(est_name, kwargs, grid, m, splitter, train, test)
        means = np.sort(out["mean"][np.isfinite(out["mean"])])[::-1]
        if len(means) > 1 and (means[0] - means[1]) < 1e-6 * abs(means[0]):
            meta["dropped"].append(name)
            continue
        for key in ("split_scores", "mean", "std", "rank"):
            arrays[f"{name}__{key}"] = out[key]
        meta["cases"][name] = {"estimator": est_name, "kwargs": kwargs, "grid": grid, "n_views": m,
                               "splitter": splitter, "best_params": out["best_params"],
                               "best_score": out["best_score"], "held_out_score": out["held_out_score"],
                               "warnings": out["warnings"]}
    gdir = os.path.join(ROOT, "tests", "golden")
    write_npz(os.path.join(gdir, "reference_outputs_gridsearch.npz"), arrays)
    with open(os.path.join(gdir, "reference_outputs_gridsearch.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"kept {sorted(meta['cases'])}, dropped {meta['dropped']}")


if __name__ == "__main__":
    main()
