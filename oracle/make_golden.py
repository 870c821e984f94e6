"""Generate tests/golden/*.npz from the UNMODIFIED reference (run in the authoring container).

    python oracle/make_golden.py

TEST INFRASTRUCTURE ONLY.  Imports /root/reference through oracle/refshim.py, fits the
reference estimators / evaluates the reference objective on seeded inputs and stores
inputs' recipe + outputs.  The fixtures travel to the GPU box; the reference does not.
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

import torch  # noqa: E402
from cca_zoo.datasets import JointData  # noqa: E402
from cca_zoo.deep.objectives import CCALoss, MCCALoss  # noqa: E402
from cca_zoo.linear import CCA, GCCA, MCCA, PLS, rCCA  # noqa: E402

from cca_zoo_b200.datasets import conftest_views, joint_data  # noqa: E402

MODELS = {"CCA": CCA, "rCCA": rCCA, "PLS": PLS, "MCCA": MCCA, "GCCA": GCCA}

# name -> (kind, args): inputs are rebuilt from this recipe by tests/golden_io.py
DATASETS = {
    "two_views": ("conftest", {"name": "two_views"}),
    "three_views": ("conftest", {"name": "three_views"}),
    "correlated_views": ("conftest", {"name": "correlated_views"}),
    "quickstart": ("joint", dict(n_views=2, n_samples=200, n_features=[50, 50],
                                 latent_dimensions=2, signal_to_noise=2.0, random_state=0)),
    "joint2_med": ("joint", dict(n_views=2, n_samples=3000, n_features=[96, 80],
                                 latent_dimensions=6, signal_to_noise=2.0 / 96, random_state=1)),
    "joint3_med": ("joint", dict(n_views=3, n_samples=2500, n_features=[64, 48, 40],
                                 latent_dimensions=5, signal_to_noise=2.0 / 64, random_state=2)),
    "joint4_gcca": ("joint", dict(n_views=4, n_samples=600, n_features=[24, 20, 28, 16],
                                  latent_dimensions=4, signal_to_noise=0.1, random_state=3)),
}

CASES = [
    # (case name, model, kwargs, dataset, dtype)
    ("cca_two", "CCA", dict(latent_dimensions=2), "two_views", "f64"),
    ("cca_corr", "CCA", dict(latent_dimensions=2), "correlated_views", "f64"),
    ("rcca01_corr", "rCCA", dict(latent_dimensions=2, c=0.1), "correlated_views", "f64"),
    ("rcca_pv_two", "rCCA", dict(latent_dimensions=3, c=[0.2, 0.7]), "two_views", "f64"),
    ("pls_corr", "PLS", dict(latent_dimensions=2), "correlated_views", "f64"),
    ("rcca_nocenter", "rCCA", dict(latent_dimensions=2, c=0.05, center=False), "two_views", "f64"),
    ("cca_quick", "CCA", dict(latent_dimensions=2), "quickstart", "f64"),
    ("cca_quick32", "CCA", dict(latent_dimensions=2), "quickstart", "f32"),
    ("rcca_med", "rCCA", dict(latent_dimensions=6, c=0.1), "joint2_med", "f64"),
    ("rcca_med32", "rCCA", dict(latent_dimensions=6, c=0.1), "joint2_med", "f32"),
    ("mcca_two", "MCCA", dict(latent_dimensions=2), "two_views", "f64"),
    ("mcca_three", "MCCA", dict(latent_dimensions=2), "three_views", "f64"),
    ("mcca_three_c", "MCCA", dict(latent_dimensions=2, c=0.3, pca=False), "three_views", "f64"),
    ("mcca_three_pv", "MCCA", dict(latent_dimensions=3, c=[0.1, 0.2, 0.3]), "three_views", "f64"),
    ("mcca_med", "MCCA", dict(latent_dimensions=5, c=0.05), "joint3_med", "f64"),
    ("mcca_med32", "MCCA", dict(latent_dimensions=5, c=0.05), "joint3_med", "f32"),
    ("gcca_three", "GCCA", dict(latent_dimensions=2), "three_views", "f64"),
    ("gcca_three_cw", "GCCA", dict(latent_dimensions=2, c=0.2, view_weights=[1.0, 1.0, 2.0]),
     "three_views", "f64"),
    ("gcca_med", "GCCA", dict(latent_dimensions=4, c=0.1), "joint4_gcca", "f64"),
]

LOSS_CASES = [
    # (name, kind, batch, widths, eps, seed)
    ("loss_16x4", "cca", 16, [4, 4], 1e-4, 0),
    ("loss_256x16", "cca", 256, [16, 12], 1e-5, 1),
    ("loss_1024x64", "cca", 1024, [64, 64], 1e-5, 2),
    ("mloss_512x8x3", "mcca", 512, [8, 8, 6], 1e-5, 3),
]


def build_dataset(name):
    kind, args = DATASETS[name]
    if kind == "conftest":
        return conftest_views(args["name"])
    views = joint_data(**args)
    ref = JointData(**args).sample()
    for a, b in zip(views, ref):  # the generator must reproduce the reference's draws
        assert np.array_equal(a, b), "joint_data diverged from reference JointData"
    return views


def loss_inputs(batch, widths, seed):
    """Correlated representations: shared latent + noise (torch CPU generator, seeded)."""
    g = torch.Generator().manual_seed(seed)
    zl = torch.randn(batch, 4, generator=g, dtype=torch.float64)
    out = []
    for w in widths:
        a = torch.randn(4, w, generator=g, dtype=torch.float64)
        out.append(zl @ a + 0.5 * torch.randn(batch, w, generator=g, dtype=torch.float64))
    return out


def main():
    out = {}
    meta = {"datasets": DATASETS, "cases": [], "loss_cases": []}
    for name, model, kwargs, ds, dt in CASES:
        views = build_dataset(ds)
        if dt == "f32":
            views = [v.astype(np.float32) for v in views]
        est = MODELS[model](**kwargs).fit(views)
        for i, w in enumerate(est.weights_):
            out[f"{name}/w{i}"] = np.asarray(w)
        for i, mu in enumerate(est.means_):
            out[f"{name}/mean{i}"] = np.asarray(mu)
        out[f"{name}/score"] = np.asarray(est.score(views))
        meta["cases"].append(dict(name=name, model=model, kwargs=kwargs, dataset=ds, dtype=dt))
        print(name, out[f"{name}/score"])
    # held-out score of the README quickstart (README.md:52-72)
    args = DATASETS["quickstart"][1]
    gen = JointData(**args)
    train = gen.sample()
    test = gen.sample()
    est = CCA(latent_dimensions=2).fit(train)
    out["quickstart_test/v0"], out["quickstart_test/v1"] = test
    out["quickstart_test/score"] = est.score(test)
    print("quickstart test", out["quickstart_test/score"])

    for name, kind, batch, widths, eps, seed in LOSS_CASES:
        zs = [z.clone().requires_grad_(True) for z in loss_inputs(batch, widths, seed)]
        fn = CCALoss(eps=eps) if kind == "cca" else MCCALoss(eps=eps)
        loss = fn(zs)
        loss.backward()
        out[f"{name}/loss"] = np.array(loss.item())
        for i, z in enumerate(zs):
            out[f"{name}/grad{i}"] = z.grad.numpy()
        meta["loss_cases"].append(dict(name=name, kind=kind, batch=batch, widths=widths,
                                       eps=eps, seed=seed))
        print(name, loss.item())

    gdir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(gdir, exist_ok=True)
    # the large float64 arrays keep 30 of their 52 mantissa bits (relative rounding <= 1e-9, far below every tolerance
    # they are checked with), which keeps the compressed file under 1 MB
    out = {k: (v.view(np.uint64) & ~np.uint64((1 << 22) - 1)).view(np.float64)
           if v.dtype == np.float64 and v.nbytes >= 16384 else v for k, v in out.items()}
    np.savez_compressed(os.path.join(gdir, "reference_outputs.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
