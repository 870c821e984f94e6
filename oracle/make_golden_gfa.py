"""Generate tests/golden/reference_outputs_gfa.{npz,json} from the UNMODIFIED reference: GFA
(cca_zoo/probabilistic/_gfa.py).

    python oracle/make_golden_gfa.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  The reference records no statistics, so they come from the data-space
restatement (oracle/gfa.py:ref_gfa_fit) after checking that its weights agree with the reference's, and from the Gram
form (oracle/gfa.py:cov_gfa_fit).  A case is kept only when every relative change of z lies at least 1e-3 tol away
from tol and every pruning statistic at least 1e-3 * 1e-7 away from 1e-7, in both forms: then a last-bit difference
in the arithmetic cannot move n_iter_ or n_components_.
"""
from __future__ import annotations

import json
import os
import sys
import warnings

import numpy as np

warnings.filterwarnings("ignore", category=RuntimeWarning)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

from cca_zoo.probabilistic import GFA  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import gfa as O  # noqa: E402

N_TEST = 60          # held-out rows appended to the generated data sets (the conftest ones get noisy copies) (transform / score / log_likelihood)
DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "three_correlated_views": ("conftest", {"name": "three_correlated_views"}),
    "joint2": ("joint", dict(n_views=2, n_samples=400, n_features=[10, 8], latent_dimensions=2,
                             signal_to_noise=2.0, random_state=3)),
    "private": ("private", {"seed": 1, "n": 150}),
    "ragged4": ("joint", dict(n_views=4, n_samples=500, n_features=[7, 13, 5, 9], latent_dimensions=2,
                              signal_to_noise=1.0, random_state=5)),
}
CASES = [
    ("two_views", "two_views", dict(latent_dimensions=2)),
    ("three_views", "three_correlated_views", dict(latent_dimensions=2, tol=1e-3)),
    ("prune", "joint2", dict(latent_dimensions=4)),
    ("no_drop", "joint2", dict(latent_dimensions=3, drop_k=False, max_iter=1500)),
    ("uncentred", "joint2", dict(latent_dimensions=3, center=False)),
    ("private", "private", dict(latent_dimensions=4)),
    ("ragged4", "ragged4", dict(latent_dimensions=3, random_state=2)),
]
SAMPLES = 3


def _private(seed, n):
    """The data of the reference's test_gfa_identifies_private_factor, plus N_TEST more rows of the same model."""
    rng = np.random.default_rng(seed)
    n = n + N_TEST
    zs, zp = rng.standard_normal((n, 1)), rng.standard_normal((n, 1))
    y1 = zs @ rng.standard_normal((1, 5)) + zp @ rng.standard_normal((1, 5)) + 0.1 * rng.standard_normal((n, 5))
    y2 = zs @ rng.standard_normal((1, 4)) + 0.1 * rng.standard_normal((n, 4))
    return [y1, y2]


def build_dataset(name):
    """(train views, held-out views)."""
    kind, args = DATASETS[name]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        test = [v + 0.1 * rng.standard_normal(v.shape) for v in views]
        return views, test
    if kind == "private":
        views = _private(**args)
    else:
        views = joint_data(**dict(args, n_samples=args["n_samples"] + N_TEST))
    return [v[:-N_TEST] for v in views], [v[-N_TEST:] for v in views]


def fit_case(name, kw, views):
    """(reference estimator, whether the case is a usable parity target)."""
    est = GFA(**dict(kw, num_posterior_samples=SAMPLES)).fit(views)
    rkw = {k: v for k, v in kw.items() if k != "latent_dimensions"}
    r = O.ref_gfa_fit(views, kw["latent_dimensions"], **rkw)
    st, (rels, drops) = O.cov_gfa_fit(views, kw["latent_dimensions"], **rkw)
    ref = np.vstack(est.weights_)
    scale = max(float(np.abs(ref).max()), 1e-300)
    err = max(float(np.abs(np.vstack(r["W"]) - ref).max()), float(np.abs(st["W"] - ref).max())) / scale
    assert r["n_iter"] == est.n_iter_ and r["k"] == est.n_components_, name
    tol = kw.get("tol", 1e-4)
    margin_rel = min([np.inf] + [abs(x - tol) / tol for x in np.concatenate([r["rel"], rels])])
    margin_drop = min([np.inf] + [abs(x - 1e-7) / 1e-7 for x in np.concatenate([r["drop"], drops])])
    ok = (err < 1e-12 and st["iters"] == est.n_iter_ and st["k"] == est.n_components_ and margin_rel >= 1e-3
          and margin_drop >= 1e-3)
    print(name, kw["random_state"], est.n_iter_, est.n_components_, f"err {err:.1e} rel margin {margin_rel:.1e} "
          f"drop margin {margin_drop:.1e}", "" if ok else "dropped")
    return est, ok


def main():
    out, meta = {}, {"datasets": DATASETS, "n_test": N_TEST, "samples": SAMPLES, "cases": [], "dropped": []}
    for name, ds, base in CASES:
        views, test = build_dataset(ds)
        for seed in range(base.get("random_state", 0), base.get("random_state", 0) + 4):
            kw = dict(base, random_state=seed)
            est, ok = fit_case(name, kw, views)
            if ok:
                break
            meta["dropped"].append(f"{name}@{seed}")
        if not ok:
            continue
        kwargs = dict(kw, num_posterior_samples=SAMPLES)
        for i, (w, mu) in enumerate(zip(est.weights_, est.means_)):
            out[f"{name}/w{i}"], out[f"{name}/mean{i}"] = np.asarray(w), np.asarray(mu)
        out[f"{name}/view_relevance"] = np.asarray(est.view_relevance_)
        out[f"{name}/n_iter"] = np.asarray([est.n_iter_])
        out[f"{name}/n_components"] = np.asarray([est.n_components_])
        for key, val in est.posterior_samples_.items():
            out[f"{name}/post/{key}"] = np.asarray(val)
        out[f"{name}/transform"] = est.transform(test)[0]
        out[f"{name}/score"] = np.asarray(est.score(test))
        out[f"{name}/log_likelihood"] = np.asarray([est.log_likelihood(test)])
        out[f"{name}/loadings0"] = est.get_factor_loadings(test)[0]
        meta["cases"].append(dict(name=name, dataset=ds, kwargs=kwargs))
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_gfa.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_gfa.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
