"""Generate tests/golden/reference_outputs_tcca.{npz,json} from the UNMODIFIED reference: TCCA
(cca_zoo/linear/_tcca.py).

    python oracle/make_golden_tcca.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  tensorly is not installed, so the reference's ``parafac`` is bound to
the restatement oracle/tcca.py:parafac, which also records the iteration count, the reconstruction errors and the
start's singular-value gaps.  A case is kept only when every |rec_prev - rec| lies at least 1e-3 (relative) away from
the 1e-8 tolerance and every start gap (sigma_k - sigma_{k+1}) / sigma_1 is at least 1e-3: then a last-bit difference
in the arithmetic cannot change the iteration count or the start.
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

import cca_zoo.linear._tcca as ref_tcca  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402
from oracle import tcca as O  # noqa: E402

N_TEST = 40
DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "three_views": ("conftest", {"name": "three_views"}),
    "ragged4": ("joint", dict(n_views=4, n_samples=300, n_features=[5, 7, 4, 6], latent_dimensions=2,
                              signal_to_noise=1.0, random_state=1)),
    "ragged5": ("joint", dict(n_views=5, n_samples=200, n_features=[3, 4, 5, 3, 4], latent_dimensions=2,
                              signal_to_noise=1.0, random_state=2)),
    "rankdef": ("rankdef", {"seed": 3, "n": 120}),
    "joint3": ("joint", dict(n_views=3, n_samples=400, n_features=[6, 5, 4], latent_dimensions=2,
                             signal_to_noise=2.0, random_state=4)),
}
CASES = [
    ("two_views", "two_views", dict(latent_dimensions=2)),
    ("three_views", "three_views", dict(latent_dimensions=2)),
    ("ragged4_c", "ragged4", dict(latent_dimensions=3, c=[0.1, 0.0, 0.3, 0.5])),
    ("ragged5", "ragged5", dict(latent_dimensions=2)),
    ("k_gt_p_rs0", "three_views", dict(latent_dimensions=8, random_state=0)),
    ("k_gt_p_rs42", "three_views", dict(latent_dimensions=8, random_state=42)),
    ("scalar_c", "three_views", dict(latent_dimensions=3, c=0.3)),
    ("eps_floor", "rankdef", dict(latent_dimensions=2, eps=1e-2)),
    ("uncentred", "joint3", dict(latent_dimensions=2, center=False)),
    ("joint3", "joint3", dict(latent_dimensions=2)),
    ("joint3_k4", "joint3", dict(latent_dimensions=4, random_state=0)),
]


def _rankdef(seed, n):
    """Three views, the last one rank-deficient (its third column is the sum of the first two)."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, 1))
    a = z @ rng.standard_normal((1, 4)) + rng.standard_normal((n, 4))
    b = z @ rng.standard_normal((1, 3)) + rng.standard_normal((n, 3))
    c = z @ rng.standard_normal((1, 2)) + rng.standard_normal((n, 2))
    return [a, b, np.hstack([c, c[:, :1] + c[:, 1:]])]


def build_dataset(name):
    """(train views, held-out views)."""
    kind, args = DATASETS[name]
    if kind == "conftest":
        views = conftest_views(args["name"])
        rng = np.random.default_rng(99)
        return views, [v[:N_TEST] + 0.1 * rng.standard_normal(v[:N_TEST].shape) for v in views]
    if kind == "rankdef":
        views = _rankdef(args["seed"], args["n"] + N_TEST)
    else:
        views = joint_data(**dict(args, n_samples=args["n_samples"] + N_TEST))
    return [v[:-N_TEST] for v in views], [v[-N_TEST:] for v in views]


def fit_case(name, kw, views):
    """(reference estimator, info of its parafac, whether the case is a usable parity target)."""
    info = {}

    def parafac(tensor, rank, **kwargs):
        return O.parafac(tensor, rank, info=info, **kwargs)

    ref_tcca.parafac = parafac
    est = ref_tcca.TCCA(**kw).fit(views)
    rkw = {k: v for k, v in kw.items() if k != "latent_dimensions"}
    w_cov, _, st = O.cov_tcca_fit(views, kw["latent_dimensions"], **rkw)
    err = max(float(np.abs(a - b).max() / np.abs(a).max()) for a, b in zip(est.weights_, w_cov))
    rec = np.asarray(info["rec"])
    margin = min([np.inf] + [abs(abs(d) - O.TOL) / O.TOL for d in np.diff(rec)])
    gap = min([np.inf] + list(info["gaps"]))
    ok = margin >= 1e-3 and gap >= 1e-3 and err < 1e-11 and st["iters"] == info["iters"]
    print(f"{name}: iters {info['iters']} stop {info['stop']} err {err:.1e} rec margin {margin:.1e} gap {gap:.1e}",
          "" if ok else "dropped")
    return est, info, ok


def main():
    out, meta = {}, {"datasets": DATASETS, "n_test": N_TEST, "cases": [], "dropped": []}
    for name, ds, kw in CASES:
        views, test = build_dataset(ds)
        est, info, ok = fit_case(name, kw, views)
        if not ok:
            meta["dropped"].append(name)
            continue
        for i, (w, mu) in enumerate(zip(est.weights_, est.means_)):
            out[f"{name}/w{i}"], out[f"{name}/mean{i}"] = np.asarray(w), np.asarray(mu)
        out[f"{name}/rec"] = np.asarray(info["rec"])
        out[f"{name}/transform"] = np.stack(est.transform(test))
        out[f"{name}/score"] = np.asarray(est.score(test))
        meta["cases"].append(dict(name=name, dataset=ds, kwargs=kw, iters=int(info["iters"]), stop=bool(info["stop"])))
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_tcca.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_tcca.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays;", "dropped:", meta["dropped"] or "none")


if __name__ == "__main__":
    main()
