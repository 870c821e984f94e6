"""KGCCA and KTCCA without a GPU: the reference's data-space fits (oracle/kgcca.py, oracle/ktcca.py) and the eigenbasis
routes the device takes against the reference's golden outputs, within tolerances set from each case's own spread; the
linear KGCCA matrix Q against its closed form; and the estimators' host logic on the torch-CPU stand-in (golden
parity, parameter broadcasting, limits and errors before any kernel, the unsupported paths)."""
import inspect

import numpy as np
import pytest

from oracle import kcca as O
from oracle import kgcca as OG
from oracle import ktcca as OT
from tests.kgcca_ktcca_golden import GOLDEN, KGCCA, KTCCA

ROUTES = {"KGCCA": (OG.ref_kgcca_fit, OG.eig_kgcca_fit), "KTCCA": (OT.ref_ktcca_fit, OT.eig_ktcca_fit)}
ALL_CASES = [(model, name) for model, g in GOLDEN.items() for name in sorted(g.cases)]


def _split(g, name):
    kw = g.kwargs(name)
    return kw.pop("latent_dimensions"), kw


def _scores(X, st, w):
    return [K @ a for K, a in zip(O.kernels(X, st), w)]


@pytest.mark.parametrize("model", sorted(GOLDEN))
def test_golden_covers_the_cases(model):
    g = GOLDEN[model]
    kinds = set()
    for c in g.cases.values():
        ker = c["kwargs"].get("kernel", "linear")
        kinds |= set(ker) if isinstance(ker, list) else {ker}
    assert kinds >= {"linear", "poly", "polynomial", "rbf", "sigmoid", "cosine", "laplacian", "chi2", "additive_chi2"}
    assert {len(g.inputs(n)[0]) for n in g.cases} >= {2, 3, 4, 5}
    assert any(not c["kwargs"].get("center", True) for c in g.cases.values())
    assert any(c["how"] == "f32" for c in g.cases.values())
    assert any(isinstance(c["kwargs"].get("c"), list) for c in g.cases.values())
    assert not g.meta["dropped"]
    if model == "KGCCA":
        assert any(isinstance(c["kwargs"].get("view_weights"), list) for c in g.cases.values())
        assert any(isinstance(c["kwargs"].get("view_weights"), float) for c in g.cases.values())
        assert max(g.meta["datasets"][c["dataset"]]["n_samples"] for c in g.cases.values()
                   if c["kwargs"].get("kernel") == "rbf") >= 400
    else:
        assert any(c["kwargs"]["latent_dimensions"] > g.meta["datasets"][c["dataset"]]["n_samples"]
                   for c in g.cases.values())


@pytest.mark.parametrize("model,name", ALL_CASES)
@pytest.mark.parametrize("route", ["ref", "eig"])
def test_restatements_match_golden(model, name, route):
    g = GOLDEN[model]
    k, kw = _split(g, name)
    views, test = g.inputs(name)
    ref = g.outputs(name)
    tol_w, tol_t, tol_c = g.tolerances(name)
    w, X, st = ROUTES[model][route == "eig"](views, k, **kw)
    assert O.rel_err(w, ref["w"]) < tol_w
    assert O.rel_err(O.align(_scores(X, st, w), ref["s"]), ref["s"]) < tol_t
    tr = np.stack(O.transform(X, st, O.align(w, ref["w"]), test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_t
    np.testing.assert_allclose(O.score(X, st, w, test), ref["score"], rtol=0, atol=tol_c)


@pytest.mark.parametrize("c", [0.1, 0.7])
def test_linear_kgcca_q_is_the_gcca_matrix_of_the_gram(c):
    """With a linear kernel, K_i B_i^-1 K_i = X_i ((1 - c_i) X_i^T X_i + c_i I)^-1 X_i^T on the range of K_i: Q is
    GCCA's matrix built on the unscaled Gram (not the covariance scaling of linear/_gcca.py), up to the eps floor."""
    views, _ = KGCCA.inputs("linear_three")
    mu = [1.0, 2.0, 0.5]
    info = {}
    OG.eig_kgcca_fit(views, 2, c=c, eps=1e-12, view_weights=mu, info=info)
    X = [v - v.mean(axis=0) for v in views]
    Q = sum(m * x @ np.linalg.solve((1.0 - c) * x.T @ x + c * np.eye(x.shape[1]), x.T) for m, x in zip(mu, X))
    np.testing.assert_allclose(info["Q"], Q, rtol=0, atol=1e-9 * np.abs(Q).max())


# ----------------------------------------------------------------------------------------------------------------------
# host logic on the torch-CPU stand-in
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def standin(monkeypatch):
    from cca_zoo_b200.nonparametric import _kgcca, _ktcca
    from tests import fake_ops, fake_ops_kcca, fake_ops_tcca

    fake_ops.install(monkeypatch)
    fake_ops_kcca.install(monkeypatch)
    fake_ops_tcca.install(monkeypatch)
    monkeypatch.setattr(_kgcca, "ops", fake_ops)
    monkeypatch.setattr(_ktcca, "ops", fake_ops)
    return fake_ops_kcca, fake_ops_tcca


def _estimator(model):
    import cca_zoo_b200.nonparametric as nonparametric

    return getattr(nonparametric, model)


@pytest.mark.parametrize("model,name", ALL_CASES)
def test_estimator_on_the_standin_matches_golden(standin, model, name):
    g = GOLDEN[model]
    k, kw = _split(g, name)
    views, test = g.inputs(name)
    ref = g.outputs(name)
    tol_w, tol_t, tol_c = g.tolerances(name)
    est = _estimator(model)(latent_dimensions=k, **kw).fit(views)
    n = views[0].shape[0]
    assert est.n_views_ == len(views) and est.n_features_in_ == [v.shape[1] for v in views] and est.n_samples_ == n
    for mu, v in zip(est.means_, views):
        np.testing.assert_allclose(mu, v.mean(axis=0) if kw.get("center", True) else 0.0, rtol=0, atol=1e-14)
    kk = min(k, n) if model == "KGCCA" else k
    assert all(w.dtype == np.float64 and w.shape == (n, kk) for w in est.weights_)
    assert O.rel_err(est.weights_, ref["w"]) < tol_w
    est.weights_ = O.align(est.weights_, ref["w"])
    tr = np.stack(est.transform(test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_t
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=tol_c)
    if model == "KTCCA":
        assert est._fit_info["iters"] == g.cases[name]["iters"]
        assert est._fit_info["stop"] == g.cases[name]["stop"]


def test_ktcca_draws_tensorlys_random_start_columns(standin):
    from cca_zoo_b200.linear._tcca import random_start_columns
    from cca_zoo_b200.nonparametric import KTCCA as Est

    views = KTCCA.inputs("k_gt_n_rs0")[0]
    Est(**KTCCA.kwargs("k_gt_n_rs0")).fit(views)
    n = views[0].shape[0]
    drawn = standin[1].CALLS["rand"]
    for a, b in zip(drawn, random_start_columns([n] * 3, 16, 0)):
        np.testing.assert_array_equal(a, b)
    assert drawn[0].shape == (n, 16 - n)


@pytest.mark.parametrize("model,name", [("KGCCA", "rbf_f32"), ("KTCCA", "rbf_f32")])
def test_float32_views_are_computed_in_float64(standin, model, name):
    g = GOLDEN[model]
    views = g.inputs(name)[0]
    a = _estimator(model)(**g.kwargs(name)).fit(views)
    b = _estimator(model)(**g.kwargs(name)).fit([v.astype(np.float32) for v in views])
    for x, y in zip(a.weights_, b.weights_):
        assert y.dtype == np.float64
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("model", ["KGCCA", "KTCCA"])
def test_parameter_errors_before_any_kernel(standin, model):
    from sklearn.utils._param_validation import InvalidParameterError

    Est = _estimator(model)
    views = GOLDEN[model].inputs("cosine")[0]
    with pytest.raises(InvalidParameterError):
        Est(latent_dimensions=0).fit(views)
    with pytest.raises(ValueError, match="length 3"):
        Est(c=[0.1, 0.2]).fit(views)
    with pytest.raises(ValueError, match="not supported"):
        Est(kernel="precomputed").fit(views)
    with pytest.raises(ValueError, match="not supported"):
        Est(kernel=lambda x, y: x @ y).fit(views)
    with pytest.raises(ValueError, match="not supported"):
        Est(kernel="nope").fit(views)
    for key in ("gamma", "degree", "coef0"):
        with pytest.raises(TypeError, match=f"multiple values for keyword argument '{key}'"):
            Est(kernel="poly", kernel_params={key: 1.0}).fit(views)
    with pytest.raises(TypeError, match="gamma"):
        Est(kernel="chi2", center=False).fit([np.abs(v) for v in views])
    if model == "KGCCA":
        with pytest.raises(ValueError, match="'view_weights' must be a scalar or a list of length 3"):
            Est(view_weights=[1.0, 2.0]).fit(views)
    else:
        with pytest.raises(InvalidParameterError):
            Est(random_state=-1).fit(views)
    assert standin[0].CALLS["kernel"] == 0 and standin[0].CALLS["syevj"] == 0


def test_limits_before_any_kernel(standin):
    from cca_zoo_b200.nonparametric import KGCCA as G
    from cca_zoo_b200.nonparametric import KTCCA as T

    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match="at most 8 views"):
        G().fit([rng.standard_normal((10, 2)) for _ in range(9)])
    with pytest.raises(ValueError, match="n = 8192"):
        G().fit([np.zeros((8193, 1)), np.zeros((8193, 1))])
    with pytest.raises(ValueError, match="at most 8 views"):
        T().fit([rng.standard_normal((2, 2)) for _ in range(9)])
    with pytest.raises(ValueError, match="at most 64 latent"):
        T(latent_dimensions=65).fit([rng.standard_normal((10, 2)) for _ in range(2)])
    with pytest.raises(ValueError, match="2\\^25"):
        T().fit([np.zeros((323, 1))] * 3)
    with pytest.raises(ValueError, match="2\\^25"):
        T().fit([np.zeros((5793, 1))] * 2)
    assert standin[0].CALLS["kernel"] == 0 and standin[0].CALLS["syevj"] == 0
    assert standin[1].CALLS["moment"] == 0 and standin[1].CALLS["fit"] == 0


@pytest.mark.parametrize("model", ["KGCCA", "KTCCA"])
@pytest.mark.filterwarnings("ignore:invalid value encountered")
def test_data_errors_before_the_eigensolve(standin, model):
    Est = _estimator(model)
    views = GOLDEN[model].inputs("rbf_three")[0]
    with pytest.raises(ValueError, match="negative"):
        Est(kernel="chi2", gamma=0.5).fit(views)           # centred views have negative entries
    with pytest.raises(np.linalg.LinAlgError, match="did not converge"):
        Est(kernel="poly", degree=0.5).fit(views)          # (x.y / d + 1)^0.5 of negative bases: NaN
    assert standin[0].CALLS["syevj"] == 0


@pytest.mark.parametrize("model", ["KGCCA", "KTCCA"])
def test_unsupported_paths(standin, monkeypatch, model):
    from cca_zoo_b200 import parallel

    Est = _estimator(model)
    views = GOLDEN[model].inputs("rbf_three")[0]
    with pytest.raises(NotImplementedError, match=f"{model} has no partial_fit"):
        Est().partial_fit(views)
    with pytest.raises(NotImplementedError, match="block covariance"):
        Est()._solve(None, None, None)
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(NotImplementedError, match=f"{model} has no sharded fit"):
        Est().fit(views)


def test_exports_and_reference_signatures():
    from cca_zoo_b200.nonparametric import KCCA, KGCCA, KTCCA  # noqa: F401

    common = dict(latent_dimensions=1, center=True, c=0.1, kernel="linear", gamma=None, degree=1.0, coef0=1.0,
                  kernel_params=None)
    want = {KGCCA: dict(common, view_weights=None, eps=1e-6, device=None),
            KTCCA: dict(common, eps=1e-3, random_state=None, device=None)}
    for Est, defaults in want.items():
        params = inspect.signature(Est.__init__).parameters
        assert list(params)[1:] == list(defaults)
        assert {k: p.default for k, p in params.items() if k != "self"} == defaults
