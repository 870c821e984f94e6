"""Generate tests/golden/reference_outputs_kgcca.{npz,json} from the UNMODIFIED reference: KGCCA
(cca_zoo/nonparametric/_kgcca.py).

    python oracle/make_golden_kgcca.py

TEST INFRASTRUCTURE ONLY (see make_golden.py).  Every case records the reference's weights_, its training scores
K_i weights_i, the held-out transform and score, and its spreads: the largest change of the weights, of the training
scores, of the held-out transform and of the held-out score over three refits with the inputs perturbed by 1e-15
(relative, seeded), as oracle/make_golden_kcca.py measures the first two.
The reference's weights are pinv(K_i) T with numpy's cutoff 1e-15 sigma_max, so for a rank-deficient kernel matrix
they carry rounding noise in its null space, and the spread measures that noise.  A case is kept only when the
eigenvalue gap (theta_k - theta_{k+1}) / theta_1 of Q is at least 1e-3 and no view's min f_i lies within 1e-3 eps of
eps (the switch of its floor).
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

from cca_zoo.nonparametric import KGCCA as RefKGCCA  # noqa: E402

from cca_zoo_b200.datasets import joint_data  # noqa: E402
from oracle import kcca as O  # noqa: E402
from oracle import kgcca as G  # noqa: E402

N_TEST = 30
DATASETS = {
    "two": dict(n_views=2, n_samples=60, n_features=[8, 6], latent_dimensions=2, signal_to_noise=1.0, random_state=0),
    "three": dict(n_views=3, n_samples=100, n_features=[5, 7, 4], latent_dimensions=2, signal_to_noise=1.0,
                  random_state=1),
    "four": dict(n_views=4, n_samples=90, n_features=[5, 7, 4, 6], latent_dimensions=2, signal_to_noise=2.0,
                 random_state=2),
    "five": dict(n_views=5, n_samples=80, n_features=[3, 4, 5, 3, 4], latent_dimensions=2, signal_to_noise=1.0,
                 random_state=3),
    "three200": dict(n_views=3, n_samples=200, n_features=[6, 5, 8], latent_dimensions=2, signal_to_noise=1.0,
                     random_state=6),
    "large": dict(n_views=2, n_samples=400, n_features=[10, 12], latent_dimensions=3, signal_to_noise=2.0,
                  random_state=5),
}
# name, dataset, transform of the data ("abs": non-negative, "f32": rounded to float32), estimator kwargs
CASES = [
    ("linear_three", "three", None, dict(latent_dimensions=3)),
    ("linear_two", "two", None, dict(latent_dimensions=2)),
    ("linear_c05_weights", "three", None, dict(latent_dimensions=2, c=0.5, view_weights=[1.0, 2.0, 0.5])),
    ("poly_three", "three", None, dict(latent_dimensions=2, kernel="poly", degree=2.0)),
    ("polynomial_explicit", "three", None, dict(latent_dimensions=2, kernel="polynomial", gamma=0.1, degree=3.0,
                                                coef0=0.5)),
    ("rbf_three", "three", None, dict(latent_dimensions=3, kernel="rbf")),
    ("rbf_large", "large", None, dict(latent_dimensions=2, kernel="rbf")),
    ("rbf_uncentred", "two", None, dict(latent_dimensions=2, kernel="rbf", center=False, gamma=0.05)),
    ("rbf_f32", "three", "f32", dict(latent_dimensions=2, kernel="rbf", gamma=0.05)),
    ("rbf_scalar_weight", "two", None, dict(latent_dimensions=2, kernel="rbf", view_weights=2.0, c=0.3)),
    ("sigmoid", "two", None, dict(latent_dimensions=2, kernel="sigmoid", gamma=0.05, c=0.5)),
    ("cosine", "three", None, dict(latent_dimensions=2, kernel="cosine")),
    ("laplacian_three", "three200", None, dict(latent_dimensions=3, kernel="laplacian")),
    ("chi2_uncentred", "two", "abs", dict(latent_dimensions=2, kernel="chi2", gamma=0.5, center=False)),
    ("additive_chi2_uncentred", "two", "abs", dict(latent_dimensions=2, kernel="additive_chi2", c=0.5,
                                                   center=False)),
    ("perview_four", "four", None, dict(latent_dimensions=2, kernel=["rbf", "poly", "linear", "laplacian"],
                                        gamma=[0.1, None, None, 0.2], c=[0.1, 0.5, 0.2, 0.05], degree=2.0,
                                        view_weights=[1.0, 0.5, 2.0, 1.5])),
    ("ragged_five", "five", None, dict(latent_dimensions=3, kernel="rbf", c=[0.1, 0.2, 0.3, 0.4, 0.5])),
    ("kernel_params_dropped", "two", None, dict(latent_dimensions=2, kernel="rbf", kernel_params={"foo": 1.0})),
]


def build_dataset(name, how):
    """(train views, held-out views)."""
    views = joint_data(**dict(DATASETS[name], n_samples=DATASETS[name]["n_samples"] + N_TEST))
    if how == "abs":
        views = [np.abs(v) for v in views]
    elif how == "f32":
        views = [v.astype(np.float32).astype(np.float64) for v in views]
    return [v[:-N_TEST] for v in views], [v[-N_TEST:] for v in views]


def _settings(est):
    return [dict(metric=est._kernel[i], gamma=est._gamma[i], degree=est._degree[i], coef0=est._coef0[i],
                 filter_params=True, **(est._kp[i] or {})) for i in range(est.n_views_)]


def _scores(est, X):
    return [K @ w for K, w in zip(O.kernels(X, _settings(est)), est.weights_)]


def fit_case(name, kw, views, test, seed):
    est = RefKGCCA(**kw).fit(views)
    sc = _scores(est, est.train_views_)
    rng = np.random.default_rng(seed)
    tr, score = est.transform(test), est.score(test)
    spread_w = spread_s = spread_t = spread_c = 0.0
    for _ in range(3):
        pv = [v * (1.0 + 1e-15 * rng.standard_normal(v.shape)) for v in views]
        p = RefKGCCA(**kw).fit(pv)
        spread_w = max(spread_w, O.rel_err(p.weights_, est.weights_))
        spread_s = max(spread_s, O.rel_err(O.align(_scores(p, p.train_views_), sc), sc))
        spread_t = max(spread_t, O.rel_err(O.align(p.transform(test), tr), tr))
        spread_c = max(spread_c, float(np.abs(p.score(test) - score).max()))
    info = {}
    rkw = {a: b for a, b in kw.items() if a != "latent_dimensions"}
    w_eig, X, st = G.eig_kgcca_fit(views, kw["latent_dimensions"], info=info, **rkw)
    ev = info["evals"]
    k = min(kw["latent_dimensions"], len(ev) - 1)
    gap = (ev[k - 1] - ev[k]) / ev[0]
    eps = kw.get("eps", 1e-6)
    floor = min(abs(f - eps) / eps for f in info["fmin"])
    err_w = O.rel_err(w_eig, est.weights_)
    err_s = O.rel_err(O.align([K @ w for K, w in zip(O.kernels(X, st), w_eig)], sc), sc)
    ok = gap >= 1e-3 and floor >= 1e-3
    print(f"{name}: gap {gap:.1e} floor margin {floor:.1e} spread w {spread_w:.1e} s {spread_s:.1e} t {spread_t:.1e} "
          f"score {spread_c:.1e} eig vs ref w {err_w:.1e} s {err_s:.1e}", "" if ok else "dropped")
    return est, sc, spread_w, spread_s, spread_t, spread_c, ok


def main():
    out, meta = {}, {"datasets": DATASETS, "n_test": N_TEST, "cases": [], "dropped": []}
    for seed, (name, ds, how, kw) in enumerate(CASES):
        views, test = build_dataset(ds, how)
        est, sc, sw, ss, st_, sc_, ok = fit_case(name, kw, views, test, seed)
        if not ok:
            meta["dropped"].append(name)
            continue
        for i, (w, s) in enumerate(zip(est.weights_, sc)):
            out[f"{name}/w{i}"], out[f"{name}/s{i}"] = np.asarray(w), np.asarray(s)
        out[f"{name}/transform"] = np.stack(est.transform(test))
        out[f"{name}/score"] = np.asarray(est.score(test))
        meta["cases"].append(dict(name=name, dataset=ds, how=how, kwargs=kw, spread_w=sw, spread_s=ss, spread_t=st_,
                                  spread_score=sc_))
    gdir = os.path.join(ROOT, "tests", "golden")
    np.savez_compressed(os.path.join(gdir, "reference_outputs_kgcca.npz"), **out)
    with open(os.path.join(gdir, "reference_outputs_kgcca.json"), "w") as f:
        json.dump(meta, f, indent=1)
    print("wrote", len(out), "arrays;", "dropped:", meta["dropped"] or "none")


if __name__ == "__main__":
    main()
