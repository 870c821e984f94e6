"""Record what the unmodified reference computes for the checks that once ran against it live: the oracle's
estimator cases (tests/test_oracle_vs_reference.py), the data generators, the fixed-seed differential fuzz of the
host logic (tools/fuzz_vs_reference.py, tools/fuzz_loss_vs_reference.py) and the model-selection scores of
tests/test_dropin_vs_reference.py.  Needs the reference tree (oracle/refshim.py); writes tests/golden/
reference_live.npz, reference_fuzz.npz and reference_fuzz_loss.npz.

    python oracle/make_golden_live.py
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from tests import fake_ops  # noqa: E402,F401  (before refshim: the reference has its own `tests` package)
import fuzz_loss_vs_reference  # noqa: E402
import fuzz_vs_reference  # noqa: E402
from oracle import refshim  # noqa: E402

FUZZ_SEED, FUZZ_TRIALS = 20240924, 200

RCCA_CASES = [(ds, c) for ds in ["two_views", "correlated_views"] for c in [0.0, 0.1, [0.2, 0.7], 1.0]]
MCCA_CASES = [(0.0, True), (0.0, False), (0.3, False), ([0.1, 0.2, 0.3], True)]
GCCA_CASES = [(0.0, None), (0.2, [1.0, 1.0, 2.0])]
PARTIAL_CASES = [(0.0, True, 2), (0.2, True, 3), ([0.1, 0.3], False, 2)]
GRCCA_CASES = [(0.0, 0.0, 2), (0.5, 0.0, 2), ([0.3, 0.6, 0.0], [0.5, 2.0, 1.0], 3)]
CENTER_MODELS = ["MCCA", "MCCA_pca", "GCCA", "GCCA_w"]
JOINT_ARGS = dict(n_views=3, n_samples=77, latent_dimensions=3, n_features=[5, 9, 4],
                  signal_to_noise=[0.5, 1.0, 2.0], random_state=11)
FIXTURES = ["two_views", "three_views", "correlated_views", "two_views_test"]
DROPIN_GRIDS = {"rCCA": (2, {"c": [0.0, 0.1, 0.5, 0.9]}), "MCCA": (3, {"c": [0.0, 0.3], "eps": [1e-6, 1e-3]}),
                "GCCA": (3, {"c": [0.1, 0.6]})}


def key(*parts):
    return "/".join(str(p) for p in parts)


def dropin_views():
    rng = np.random.default_rng(0)
    lat = rng.standard_normal((150, 2))
    return [lat @ rng.standard_normal((2, 8)) + rng.standard_normal((150, 8)),
            lat @ rng.standard_normal((2, 6)) + rng.standard_normal((150, 6)),
            lat @ rng.standard_normal((2, 5)) + rng.standard_normal((150, 5))]


def grcca_groups(v):
    rng = np.random.default_rng(5)
    return [rng.integers(0, 3, size=x.shape[1]) for x in v]


def partial_confounds(v):
    return np.random.default_rng(7).standard_normal((v[0].shape[0], 3)) + 0.7


def put_weights(out, k, est):
    for i, w in enumerate(est.weights_):
        out[key(k, f"w{i}")] = np.asarray(w)
    for i, m in enumerate(est.means_):
        out[key(k, f"mean{i}")] = np.asarray(m)


def live_outputs():
    import importlib.util

    from cca_zoo.datasets import JointData
    from cca_zoo.linear import GCCA, GRCCA, MCCA, PartialCCA, rCCA
    from cca_zoo.model_selection import GridSearchCV

    from cca_zoo_b200.datasets import conftest_views

    out = {}
    for ds, c in RCCA_CASES:
        v = conftest_views(ds)
        est = rCCA(latent_dimensions=3, c=c).fit(v)
        put_weights(out, key("rcca", ds, c), est)
        out[key("rcca", ds, c, "score")] = np.asarray(est.score(v))
    v3 = conftest_views("three_views")
    for c, pca in MCCA_CASES:
        put_weights(out, key("mcca", c, pca), MCCA(latent_dimensions=3, c=c, pca=pca).fit(v3))
    for c, mu in GCCA_CASES:
        put_weights(out, key("gcca", c, mu), GCCA(latent_dimensions=3, c=c, view_weights=mu).fit(v3))
    for c, center, nv in PARTIAL_CASES:
        v = v3[:nv]
        est = PartialCCA(latent_dimensions=2, c=c, center=center).fit(v, partials=partial_confounds(v))
        put_weights(out, key("partial", c, center, nv), est)
        for i, b in enumerate(est.confound_betas_):
            out[key("partial", c, center, nv, f"beta{i}")] = np.asarray(b)
    for c, mu, nv in GRCCA_CASES:
        v = v3[:nv]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            put_weights(out, key("grcca", c, mu, nv), GRCCA(latent_dimensions=2, c=c, mu=mu).fit(
                v, feature_groups=grcca_groups(v)))
    vs = [x + 1.3 for x in v3]
    for model in CENTER_MODELS:
        if model.startswith("MCCA"):
            est = MCCA(latent_dimensions=3, c=0.1, center=False, pca=model.endswith("pca")).fit(vs)
        else:
            vw = [1.0, 2.0, 0.5] if model.endswith("w") else None
            est = GCCA(latent_dimensions=3, c=0.1, center=False, view_weights=vw).fit(vs)
        put_weights(out, key("center", model), est)
    v = conftest_views("two_views")
    v = [v[0], np.hstack([v[1], v[1][:, :1]])]
    put_weights(out, key("ridge_rank_deficient"), rCCA(latent_dimensions=9, c=0.2).fit(v))
    for i, x in enumerate(JointData(**JOINT_ARGS).sample()):
        out[key("joint_data", i)] = np.asarray(x)
    spec = importlib.util.spec_from_file_location("ref_conftest", os.path.join(refshim.REFERENCE_ROOT, "tests",
                                                                                "conftest.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    for name in FIXTURES:
        for i, x in enumerate(getattr(mod, name).__wrapped__()):
            out[key("fixture", name, i)] = np.asarray(x)
    views = dropin_views()
    for name, (nv, grid) in DROPIN_GRIDS.items():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gs = GridSearchCV(getattr(__import__("cca_zoo.linear", fromlist=[name]), name)(latent_dimensions=2),
                              param_grid=grid, cv=3).fit(views[:nv])
        out[key("dropin", name, "mean_test_score")] = np.asarray(gs.cv_results_["mean_test_score"], dtype=np.float64)
    return out


def main():
    refshim.install()
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_live.npz"), **live_outputs())
    np.savez_compressed(os.path.join(gdir, "reference_fuzz.npz"), **fuzz_vs_reference.record(FUZZ_SEED, FUZZ_TRIALS))
    np.savez_compressed(os.path.join(gdir, "reference_fuzz_loss.npz"),
                        **fuzz_loss_vs_reference.record(FUZZ_SEED, FUZZ_TRIALS))


if __name__ == "__main__":
    main()
