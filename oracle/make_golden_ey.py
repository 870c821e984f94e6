"""Generate tests/golden/reference_outputs_ey.{npz,json} from the UNMODIFIED reference: the Eckart-Young gradient
estimators (CCA_EY, PLS_EY, MCCA_EY of cca_zoo/linear/gradient/).

    python oracle/make_golden_ey.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  The reference records no step counts, so they come from the
data-space restatement (oracle/ey.py:ref_ey_fit) after checking that its weights agree with the reference's.  A case
with tol > 0 is kept only when every |prev_obj - obj| lies at least 1e-3 * tol away from tol: then a last-bit
difference in the arithmetic cannot move the step at which the fit stops.
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

from cca_zoo.linear import CCA_EY, MCCA_EY, PLS_EY  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import ey as E  # noqa: E402

DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "correlated_views": ("conftest", {"name": "correlated_views"}),
    "three_correlated_views": ("conftest", {"name": "three_correlated_views"}),
    "joint3_std": ("joint_std", dict(n_views=3, n_samples=2000, n_features=[12, 10, 8], latent_dimensions=3,
                                     signal_to_noise=0.5, random_state=4)),
}
MODELS = {"cca": CCA_EY, "pls": PLS_EY, "mcca": MCCA_EY}
ON = {"two_views": ("cca", "pls"), "correlated_views": ("cca", "pls"), "three_correlated_views": ("mcca", "cca"),
      "joint3_std": ("cca", "pls", "mcca")}
COMMON = dict(latent_dimensions=2, max_iter=150, random_state=1)


def build_dataset(name, dtype="f64"):
    kind, args = DATASETS[name]
    if kind == "conftest":
        views = conftest_views(args["name"])
    else:
        views = [(v - v.mean(axis=0)) / v.std(axis=0, ddof=1) for v in joint_data(**args)]
    return [v.astype(np.float32) for v in views] if dtype == "f32" else views


def cases():
    out = []
    for ds, kinds in ON.items():
        for kind in kinds:
            for bs in (None, 16, 64):
                for center in (True, False):
                    kw = dict(COMMON, center=center, batch_size=bs)
                    out.append((f"{kind}_{ds}_{bs or 'full'}_{'c' if center else 'nc'}", kind, kw, ds, "f64"))
    for bs in (None, 16, 64):
        out.append((f"cca_c03_two_views_{bs or 'full'}", "cca", dict(COMMON, c=0.3, batch_size=bs), "two_views", "f64"))
        out.append((f"cca_c03_joint3_std_{bs or 'full'}", "cca", dict(COMMON, c=0.3, batch_size=bs), "joint3_std",
                    "f64"))
    out.append(("cca_joint3_std_full_f32", "cca", dict(COMMON, c=0.1), "joint3_std", "f32"))
    out.append(("pls_joint3_std_64_f32", "pls", dict(COMMON, batch_size=64), "joint3_std", "f32"))
    out.append(("cca_correlated_views_full_tol", "cca", dict(COMMON, max_iter=1000, tol=1e-5), "correlated_views",
                "f64"))
    out.append(("pls_correlated_views_full_tol", "pls", dict(COMMON, max_iter=1000, tol=1e-5), "correlated_views",
                "f64"))
    out.append(("cca_two_views_diverge", "cca", dict(latent_dimensions=2, max_iter=300, random_state=0, batch_size=12,
                                                     learning_rate=0.5), "two_views", "f64"))
    return out


def main():
    out, meta = {}, {"datasets": DATASETS, "cases": [], "dropped": []}
    for name, kind, kwargs, ds, dt in cases():
        views = build_dataset(ds, dt)
        est = MODELS[kind](**kwargs).fit(views)
        rkw = {k: v for k, v in kwargs.items() if k != "latent_dimensions"}
        W, iters, deltas = E.ref_ey_fit([v for v in views], kind, kwargs["latent_dimensions"], **rkw)
        if dt == "f64":
            ref = np.vstack(est.weights_)
            if np.isnan(ref).all():
                assert np.isnan(np.vstack(W)).all(), name
            else:
                scale = float(np.abs(ref).max())
                err = max(float(np.abs(a - b).max()) for a, b in zip(W, est.weights_)) / scale
                bs = kwargs.get("batch_size")
                if bs is None or bs >= views[0].shape[0]:
                    K, _, _ = E.cov_ey_fit(views, kind, kwargs["latent_dimensions"], **{k: v for k, v in rkw.items()
                                                                                       if k != "batch_size"})
                else:
                    K, _, _ = E.mb_ey_fit(views, kind, kwargs["latent_dimensions"], **rkw)
                err = max(err, float(np.abs(np.vstack(K) - ref).max()) / scale)
                if err > 1e-12:
                    # the steps amplify rounding differences: not a usable parity target at 1e-9
                    meta["dropped"].append(name)
                    print(name, f"dropped: restatement and reference differ by {err:.1e} (relative)")
                    continue
        tol = kwargs.get("tol", 1e-6)
        finite = [d for d in deltas if np.isfinite(d)]
        margin = min(abs(x - tol) for x in finite) if finite else np.inf
        if margin < 1e-3 * tol:
            meta["dropped"].append(name)
            print(name, "dropped: a |change of the objective| lies within 1e-3 tol of tol")
            continue
        for i, (w, mu) in enumerate(zip(est.weights_, est.means_)):
            out[f"{name}/w{i}"], out[f"{name}/mean{i}"] = np.asarray(w), np.asarray(mu)
        out[f"{name}/iters"] = np.asarray([iters])
        out[f"{name}/restated_w"] = np.vstack(W)
        meta["cases"].append(dict(name=name, model=kind, kwargs=kwargs, dataset=ds, dtype=dt))
        print(name, iters, "nan" if np.isnan(np.vstack(est.weights_)).any() else "")
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_ey.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_ey.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
