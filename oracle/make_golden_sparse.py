"""Generate tests/golden/reference_outputs_sparse.{npz,json} from the UNMODIFIED reference: the sparse / ALS estimators
(PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span, SCCA_ADMM of cca_zoo/linear/_iterative.py).

    python oracle/make_golden_sparse.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  The reference records no iteration counts, so the sweeps per
dimension come from the Gram-space restatement (oracle/sparse.py:cov_als_fit) after checking that its weights
agree with the reference's.  A case is kept only when every convergence delta of every sweep lies at least
1e-3 * tol away from tol: then a last-bit difference in the arithmetic cannot move the sweep at which a dimension stops.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

from cca_zoo.linear import PLS_ALS, SCCA_ADMM, SCCA_PMD, ParkhomenkoCCA, SCCA_Span  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import sparse as S  # noqa: E402

DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "three_views": ("conftest", {"name": "three_views"}),
    "joint3_sparse": ("joint", dict(n_views=3, n_samples=2000, n_features=[96, 64, 48], latent_dimensions=3,
                                    signal_to_noise=0.5, random_state=4)),
}
MODELS = {"pls": PLS_ALS, "pmd": SCCA_PMD, "parkhomenko": ParkhomenkoCCA, "span": SCCA_Span, "admm": SCCA_ADMM}
KWARGS = {"pls": {}, "pmd": {"tau": 0.4}, "parkhomenko": {"tau": 0.5}, "span": {"span": 4}, "admm": {"tau": 0.1}}
COMMON = dict(latent_dimensions=3, max_iter=300, random_state=1)


def build_dataset(name, dtype="f64"):
    kind, args = DATASETS[name]
    views = conftest_views(args["name"]) if kind == "conftest" else joint_data(**args)
    return [v.astype(np.float32) for v in views] if dtype == "f32" else views


def cases():
    out = []
    for ds in DATASETS:
        for center in (True, False):
            for kind in MODELS:
                out.append((f"{kind}_{ds}_{'c' if center else 'nc'}", kind,
                            dict(COMMON, center=center, **KWARGS[kind]), ds, "f64"))
    out.append(("pmd_two_views_pv", "pmd", dict(COMMON, tau=[0.3, 0.6]), "two_views", "f64"))
    out.append(("span_two_views_pv", "span", dict(COMMON, span=[3, 5]), "two_views", "f64"))
    out.append(("parkhomenko_three_views_pv", "parkhomenko", dict(COMMON, tau=[0.2, 0.5, 0.4]), "three_views", "f64"))
    out.append(("pmd_joint3_sparse_f32", "pmd", dict(COMMON, tau=0.4), "joint3_sparse", "f32"))
    return out


def main():
    out, meta = {}, {"datasets": DATASETS, "cases": [], "dropped": []}
    for name, kind, kwargs, ds, dt in cases():
        views = build_dataset(ds, dt)
        est = MODELS[kind](**kwargs).fit(views)
        dims = [v.shape[1] for v in views]
        params = S.als_params(kind, dims, tau=kwargs.get("tau"), span=kwargs.get("span"))
        vs, _ = S.setup_fit([v.astype(np.float64) for v in views], kwargs["center"] if "center" in kwargs else True)
        X = np.hstack(vs)
        W, iters, deltas = S.cov_als_fit(X.T @ X, dims, X.shape[0], kind, kwargs["latent_dimensions"], params=params,
                                         max_iter=kwargs["max_iter"], random_state=kwargs["random_state"],
                                         return_info=True)
        tol = 1e-6
        margin = min(abs(x - tol) for dl in deltas for x in dl)
        if dt == "f64":
            err = max(float(np.abs(a - b).max()) for a, b in zip(W, est.weights_))
            assert err < 1e-10, f"{name}: restatement differs from the reference by {err:.2e}"
        if margin < 1e-3 * tol:
            meta["dropped"].append(name)
            print(name, "dropped: a convergence delta lies within 1e-3 tol of tol")
            continue
        for i, (w, mu) in enumerate(zip(est.weights_, est.means_)):
            out[f"{name}/w{i}"], out[f"{name}/mean{i}"] = np.asarray(w), np.asarray(mu)
        out[f"{name}/iters"] = np.asarray(iters)
        out[f"{name}/restated_w"] = np.vstack(W)
        meta["cases"].append(dict(name=name, model=kind, kwargs=kwargs, dataset=ds, dtype=dt, params=params))
        print(name, iters)
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_sparse.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_sparse.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
