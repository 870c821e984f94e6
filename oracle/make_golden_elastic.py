"""Generate tests/golden/reference_outputs_elastic.{npz,json} from the UNMODIFIED reference: ElasticCCA and SCCA_IPLS
(cca_zoo/linear/_iterative.py:522-623, 730-831).

    python oracle/make_golden_elastic.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  Every case is fitted twice: at its ``tol`` and at ``tol / 100`` (the
tolerance of both the ALS loop and sklearn's coordinate descent), with sklearn's ConvergenceWarning an error in the
tight run.  The per-view, per-dimension spread between the two runs records how sensitive the reference is to its own
tolerance; the tests compare against it.  A tight run that does not converge is recorded as such (spread None).
"""
from __future__ import annotations

import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

refshim.install()

from sklearn.exceptions import ConvergenceWarning  # noqa: E402

from cca_zoo.linear import SCCA_IPLS, ElasticCCA  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import elastic as E  # noqa: E402

DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "three_views": ("conftest", {"name": "three_views"}),
    "two_views_test": ("conftest", {"name": "two_views_test"}),
    "two_views_short": ("conftest", {"name": "two_views", "rows": 9}),     # n = 9 <= d_i: G_ii singular throughout
    "joint3": ("joint", dict(n_views=3, n_samples=500, n_features=[24, 16, 12], latent_dimensions=3,
                             signal_to_noise=0.5, random_state=4)),
}
MODELS = {"elastic": ElasticCCA, "ipls": SCCA_IPLS}
SETTINGS = {
    "lasso": dict(alpha=0.02, l1_ratio=1.0),
    "enet": dict(alpha=0.05, l1_ratio=0.5),
    "ridge": dict(alpha=0.5, l1_ratio=0.0),
    "pv": dict(alpha=[0.01, 0.05], l1_ratio=0.5),
    "default": dict(),
    "big": dict(alpha=10.0, l1_ratio=1.0),
    "ref": dict(alpha=0.1, l1_ratio=1.0),
}
TOL = 1e-6


def build_dataset(name):
    kind, args = DATASETS[name]
    if kind == "joint":
        return joint_data(**args)
    return [v[:args.get("rows")] for v in conftest_views(args["name"])]


def cases():
    out = []
    for kind in MODELS:
        for ds in ("two_views", "three_views"):
            for st in ("lasso", "enet", "ridge", "default"):
                for center in (True, False):
                    out.append((kind, ds, st, center))
        out.append((kind, "two_views", "pv", True))
        out.append((kind, "two_views", "big", True))
        out.append((kind, "two_views", "ref", True))
        out.append((kind, "two_views_test", "default", True))    # n = 20 > d, then singular from dimension 2
        out.append((kind, "two_views_short", "default", True))
        out.append((kind, "two_views_short", "ridge", True))
        out.append((kind, "joint3", "enet", True))
        out.append((kind, "joint3", "default", True))
    return out


def _fit(cls, kwargs, views, tight):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if tight:
            warnings.simplefilter("error", ConvergenceWarning)
        return cls(**kwargs).fit(views)


def main():
    out, meta = {}, {"datasets": DATASETS, "tol": TOL, "cases": []}
    for kind, ds, st, center in cases():
        name = f"{kind}_{ds}_{st}_{'c' if center else 'nc'}"
        views = build_dataset(ds)
        kwargs = dict(latent_dimensions=3, max_iter=300, random_state=1, center=center, tol=TOL, **SETTINGS[st])
        est = _fit(MODELS[kind], kwargs, views, False)
        try:
            tight = _fit(MODELS[kind], dict(kwargs, tol=TOL / 100), views, True)
            spread = [np.abs(a - b).max(axis=0).tolist() for a, b in zip(est.weights_, tight.weights_)]
            for i, w in enumerate(tight.weights_):
                out[f"{name}/tight_w{i}"] = np.asarray(w)
        except ConvergenceWarning:
            spread = None
        for i, w in enumerate(est.weights_):
            out[f"{name}/w{i}"] = np.asarray(w)
        params = E.elastic_params(kind, len(views), SETTINGS[st].get("alpha"), SETTINGS[st].get("l1_ratio"))
        W, iters = E.ref_elastic_fit(views, kind, 3, params, max_iter=300, tol=TOL, random_state=1, center=center)
        out[f"{name}/restated_w"] = np.vstack(W)
        out[f"{name}/iters"] = np.asarray(iters)
        err = [np.abs(a - b).max(axis=0).tolist() for a, b in zip(W, est.weights_)]
        meta["cases"].append(dict(name=name, model=kind, kwargs=kwargs, dataset=ds, setting=st, params=params,
                                  spread=spread, restated_err=err))
        print(name, iters, "spread", None if spread is None else f"{max(map(max, spread)):.1e}",
              "err", f"{max(map(max, err)):.1e}")
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_elastic.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_elastic.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
