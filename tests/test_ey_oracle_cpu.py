"""The kernel-form restatements of the Eckart-Young gradient estimators (oracle/ey.py: the covariance route for full
batches, the raw-view mini-batch route) against the reference's golden vectors (tests/golden/reference_outputs_ey.npz),
step counts included; the stacked-QR initialisation identity; the float32 drift the GPU tests allow; and the
estimators' host logic (route selection, parameter validation, clone / get_params, pickling) on the torch-CPU
stand-in."""
import json
import os
import pickle

import numpy as np
import pytest
from sklearn.base import clone
from sklearn.utils._param_validation import InvalidParameterError

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import ey as E

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_ey.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_ey.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def _inputs(case):
    kind, args = META["datasets"][case["dataset"]]
    if kind == "conftest":
        views = conftest_views(args["name"])
    else:
        views = [(v - v.mean(axis=0)) / v.std(axis=0, ddof=1) for v in joint_data(**args)]
    return [v.astype(np.float32) for v in views] if case["dtype"] == "f32" else views


def _restate(case, views):
    kw = dict(case["kwargs"])
    k = kw.pop("latent_dimensions")
    bs = kw.pop("batch_size", None)
    if bs is None or bs >= views[0].shape[0]:
        return E.cov_ey_fit(views, case["model"], k, **kw)
    return E.mb_ey_fit(views, case["model"], k, bs, **kw)


def test_ey_golden_covers_models_routes_and_datasets():
    assert {c["model"] for c in CASES.values()} == {"cca", "pls", "mcca"}
    assert {c["dataset"] for c in CASES.values()} == set(META["datasets"])
    assert {c["kwargs"].get("batch_size") for c in CASES.values()} >= {None, 16, 64}
    assert any(c["dtype"] == "f32" for c in CASES.values())
    assert any(c["kwargs"].get("c") == 0.3 for c in CASES.values())
    assert any(int(NPZ[f"{n}/iters"][0]) < c["kwargs"]["max_iter"] for n, c in CASES.items())   # a tol stop
    assert any(np.isnan(NPZ[f"{n}/w0"]).all() for n in CASES)                                      # a divergent fit


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["dtype"] == "f64"))
def test_ey_restatements_match_golden(name):
    case = CASES[name]
    views = _inputs(case)
    W, iters, _ = _restate(case, views)
    assert iters == int(NPZ[f"{name}/iters"][0])
    W = np.vstack(W)
    R = np.vstack([NPZ[f"{name}/w{i}"] for i in range(len(views))])
    if np.isnan(R).all():
        assert np.isnan(W).all()
        return
    err = float(np.abs(W - R).max()) / float(np.abs(R).max())
    assert err < 1e-12, f"{name}: {err:.2e}"


@pytest.mark.parametrize("shape", [(50, 2), (300, 4), (2000, 8), (17, 8), (100, 32)])
def test_stacked_qr_gives_the_householder_r(shape):
    rng = np.random.default_rng(shape[0] * 100 + shape[1])
    z0 = rng.standard_normal(shape) @ rng.standard_normal((shape[1], shape[1])) + 3.0
    r_full = np.linalg.qr(z0, mode="r")
    r_stack = E.stacked_r(z0)
    assert np.array_equal(np.sign(np.diag(r_full)), np.sign(np.diag(r_stack)))
    assert float(np.abs(r_full - r_stack).max()) / float(np.abs(r_full).max()) < 1e-12


def test_float32_grade_covariance_drift_is_within_the_gpu_tolerance():
    """The GPU tests allow 1e-3 (relative to max |w|) for float32 views: a covariance perturbed at float32 grade
    (relative 2^-22 per element, symmetric) moves the full-batch weights by much less."""
    from tests.test_ey_gpu import F32_TOL

    for name in (n for n, c in CASES.items() if c["dtype"] == "f32"):
        case = CASES[name]
        views = [v.astype(np.float64) for v in _inputs(case)]
        kw = dict(case["kwargs"])
        k = kw.pop("latent_dimensions")
        kw.pop("batch_size", None)
        X = np.hstack(views)
        X = X - X.mean(axis=0)
        C = X.T @ X / (X.shape[0] - 1)
        noise = np.random.default_rng(0).uniform(-1, 1, C.shape) * 2.0 ** -22
        Cp = C * (1.0 + 0.5 * (noise + noise.T))
        W0, _, _ = E.cov_ey_fit(views, case["model"], k, C=C, **kw)
        W1, _, _ = E.cov_ey_fit(views, case["model"], k, C=Cp, **kw)
        W0, W1 = np.vstack(W0), np.vstack(W1)
        drift = float(np.abs(W0 - W1).max()) / float(np.abs(W0).max())
        assert drift < 1e-2 * F32_TOL, f"{name}: drift {drift:.2e}"


# ---------------------------------------------------------------------------------------------------- host logic
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_ey

    fake_ops.install(monkeypatch)
    fake_ops_ey.install(monkeypatch)
    return fake_ops_ey


def _cls(kind):
    from cca_zoo_b200 import linear

    return {"cca": linear.CCA_EY, "pls": linear.PLS_EY, "mcca": linear.MCCA_EY}[kind]


@pytest.mark.parametrize("bs,route", [(None, "covariance"), (50, "covariance"), (500, "covariance"),
                                      (49, "minibatch"), (16, "minibatch")])
def test_ey_route_selection(standin, bs, route):
    views = conftest_views("two_views")
    est = _cls("cca")(latent_dimensions=2, batch_size=bs, max_iter=20, random_state=0).fit(views)
    assert est._fit_info["route"] == route and est._fit_info["iters"] == 20


@pytest.mark.parametrize("name", ["cca_two_views_full_c", "pls_correlated_views_64_nc", "mcca_joint3_std_16_c",
                                  "cca_correlated_views_full_tol"])
def test_ey_estimators_on_the_standin_match_golden(standin, name):
    case = CASES[name]
    est = _cls(case["model"])(**case["kwargs"]).fit(_inputs(case))
    R = np.vstack([NPZ[f"{name}/w{i}"] for i in range(len(est.weights_))])
    assert est._fit_info["iters"] == int(NPZ[f"{name}/iters"][0])
    assert float(np.abs(np.vstack(est.weights_) - R).max()) / float(np.abs(R).max()) < 1e-9


def test_ey_parameter_validation():
    views = conftest_views("two_views")
    with pytest.raises(InvalidParameterError):
        _cls("cca")(c=1.5).fit(views)
    with pytest.raises(InvalidParameterError):
        _cls("mcca")(c=-0.1).fit(views)
    with pytest.raises(InvalidParameterError):
        _cls("pls")(latent_dimensions=0).fit(views)


def test_ey_get_params_clone_and_pickle():
    from cca_zoo_b200.linear import gradient

    assert gradient.CCA_EY is _cls("cca") and gradient.PLS_EY is _cls("pls") and gradient.MCCA_EY is _cls("mcca")
    assert _cls("cca")().get_params()["c"] == 0.0
    assert "c" not in _cls("pls")().get_params()
    assert _cls("pls")().c == 1.0
    names = ["latent_dimensions", "center", "c", "learning_rate", "max_iter", "batch_size", "tol", "momentum",
             "random_state", "precision", "device"]
    import inspect

    assert list(inspect.signature(_cls("cca").__init__).parameters)[1:] == names
    est = _cls("mcca")(latent_dimensions=3, c=0.2, batch_size=32, random_state=5)
    cl = clone(est)
    assert cl.get_params() == est.get_params()
    assert pickle.loads(pickle.dumps(est)).get_params() == est.get_params()


def test_ey_fitted_model_pickles(standin):
    views = conftest_views("two_views")
    est = _cls("cca")(latent_dimensions=2, batch_size=16, max_iter=10, random_state=0).fit(views)
    back = pickle.loads(pickle.dumps(est))
    for a, b in zip(est.weights_, back.weights_):
        assert np.array_equal(a, b)
