"""KCCA without a GPU: the reference's data-space fit (oracle/kcca.py:ref_kcca_fit) and the eigenbasis route the
device takes (eig_kcca_fit) against the reference's golden outputs (tests/golden/reference_outputs_kcca.npz), within
tolerances set from each case's own spread; the reference's two statements about KCCA; and KCCA's host logic on the
torch-CPU stand-in (parameter broadcasting, limits and errors before any kernel, kernel_params handling, transform)."""
import numpy as np
import pytest

from oracle import kcca as O
from tests.kcca_golden import CASES, inputs, kwargs, outputs, tolerances


def _split(name):
    kw = kwargs(name)
    return kw.pop("latent_dimensions"), kw


def _scores(X, st, w):
    return [K @ a for K, a in zip(O.kernels(X, st), w)]


def test_kcca_golden_covers_the_cases():
    kinds = set()
    for c in CASES.values():
        ker = c["kwargs"].get("kernel", "linear")
        kinds |= set(ker) if isinstance(ker, list) else {ker}
    assert kinds >= {"linear", "poly", "polynomial", "rbf", "sigmoid", "cosine", "laplacian", "chi2", "additive_chi2"}
    assert {"linear_c1e-4", "linear_c10", "perview_four", "ragged_five", "rbf_f32", "chi2_uncentred",
            "kernel_params_dropped", "polynomial_explicit"} <= set(CASES)
    assert any(not c["kwargs"].get("center", True) for c in CASES.values())


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("route", ["ref", "eig"])
def test_restatements_match_golden(name, route):
    k, kw = _split(name)
    views, test = inputs(name)
    ref = outputs(name)
    tol_w, tol_s = tolerances(name)
    fit = O.ref_kcca_fit if route == "ref" else O.eig_kcca_fit
    w, X, st = fit(views, k, **kw)
    assert O.rel_err(w, ref["w"]) < tol_w
    assert O.rel_err(O.align(_scores(X, st, w), ref["s"]), ref["s"]) < tol_s
    tr = np.stack(O.transform(X, st, O.align(w, ref["w"]), test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_s
    np.testing.assert_allclose(O.score(X, st, w, test), ref["score"], rtol=0, atol=tol_s)


def test_linear_kcca_with_small_c_matches_cca():
    """tests/nonparametric/test_kcca.py: a linear KCCA with c = 1e-4 scores like CCA."""
    views, test = inputs("linear_c1e-4")
    w, X, st = O.eig_kcca_fit(views, 2, c=1e-4)
    kc = O.score(X, st, w, test)
    Xc = [v - v.mean(axis=0) for v in views]
    n = Xc[0].shape[0]
    C11, C22, C12 = (Xc[0].T @ Xc[0] / (n - 1), Xc[1].T @ Xc[1] / (n - 1), Xc[0].T @ Xc[1] / (n - 1))
    L1, L2 = np.linalg.cholesky(np.linalg.inv(C11)), np.linalg.cholesky(np.linalg.inv(C22))
    U, _, Vt = np.linalg.svd(L1.T @ C12 @ L2)
    a, b = L1 @ U[:, :2], L2 @ Vt[:2].T
    t = [(test[0] - views[0].mean(axis=0)) @ a, (test[1] - views[1].mean(axis=0)) @ b]
    cca = np.array([np.corrcoef(t[0][:, j], t[1][:, j])[0, 1] for j in range(2)])
    np.testing.assert_allclose(kc, cca, rtol=0, atol=1e-3)


def test_correlation_does_not_increase_with_c():
    """tests/nonparametric/test_kcca.py: more regularisation, no higher training correlation (c = 10 included)."""
    views = inputs("rbf")[0]
    corr = []
    for c in (0.01, 0.1, 0.5, 0.9, 10.0):
        w, X, st = O.eig_kcca_fit(views, 1, c=c, kernel="rbf")
        corr.append(O.score(X, st, w, X)[0])
    assert all(a >= b - 1e-12 for a, b in zip(corr, corr[1:]))


# ----------------------------------------------------------------------------------------------------------------------
# host logic on the torch-CPU stand-in
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_kcca

    fake_ops.install(monkeypatch)
    fake_ops_kcca.install(monkeypatch)
    return fake_ops_kcca


@pytest.mark.parametrize("name", sorted(CASES))
def test_kcca_on_the_standin_matches_golden(standin, name):
    from cca_zoo_b200.nonparametric import KCCA

    k, kw = _split(name)
    views, test = inputs(name)
    ref = outputs(name)
    tol_w, tol_s = tolerances(name)
    est = KCCA(latent_dimensions=k, **kw).fit(views)
    assert est.n_views_ == len(views) and est.n_features_in_ == [v.shape[1] for v in views]
    assert est.n_samples_ == views[0].shape[0]
    for mu, v in zip(est.means_, views):
        np.testing.assert_allclose(mu, v.mean(axis=0) if kw.get("center", True) else 0.0, rtol=0, atol=1e-14)
    assert all(w.dtype == np.float64 and w.shape == (views[0].shape[0], k) for w in est.weights_)
    assert O.rel_err(est.weights_, ref["w"]) < tol_w
    w = O.align(est.weights_, ref["w"])
    est.weights_ = w
    tr = np.stack(est.transform(test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_s
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=tol_s)


def test_kcca_float32_views_are_computed_in_float64(standin):
    from cca_zoo_b200.nonparametric import KCCA

    views = inputs("rbf_f32")[0]
    a = KCCA(**kwargs("rbf_f32")).fit(views)
    b = KCCA(**kwargs("rbf_f32")).fit([v.astype(np.float32) for v in views])
    for x, y in zip(a.weights_, b.weights_):
        assert y.dtype == np.float64
        np.testing.assert_array_equal(x, y)


def test_kcca_parameter_errors_before_any_kernel(standin):
    from sklearn.utils._param_validation import InvalidParameterError

    from cca_zoo_b200.nonparametric import KCCA

    views = inputs("cosine")[0]
    with pytest.raises(InvalidParameterError):
        KCCA(latent_dimensions=0).fit(views)
    with pytest.raises(ValueError, match="length 3"):
        KCCA(c=[0.1, 0.2]).fit(views)
    with pytest.raises(ValueError, match="not supported"):
        KCCA(kernel="precomputed").fit(views)
    with pytest.raises(ValueError, match="not supported"):
        KCCA(kernel=lambda x, y: x @ y).fit(views)
    with pytest.raises(ValueError, match="not supported"):
        KCCA(kernel="nope").fit(views)
    for key in ("gamma", "degree", "coef0"):
        with pytest.raises(TypeError, match=f"multiple values for keyword argument '{key}'"):
            KCCA(kernel="poly", kernel_params={key: 1.0}).fit(views)
    with pytest.raises(TypeError, match="gamma"):
        KCCA(kernel="chi2", center=False).fit([np.abs(v) for v in views])
    assert standin.CALLS["kernel"] == 0 and standin.CALLS["syevj"] == 0


def test_kcca_limits_before_any_kernel(standin):
    from cca_zoo_b200.nonparametric import KCCA

    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match="at most 8 views"):
        KCCA().fit([rng.standard_normal((10, 2)) for _ in range(9)])
    with pytest.raises(ValueError, match="n = 8192"):
        KCCA().fit([np.zeros((8193, 1)), np.zeros((8193, 1))])
    with pytest.raises(ValueError, match="16384"):
        KCCA().fit([np.zeros((4097, 1))] * 4)
    assert standin.CALLS["kernel"] == 0 and standin.CALLS["syevj"] == 0


@pytest.mark.filterwarnings("ignore:invalid value encountered")
def test_kcca_data_errors_before_the_eigensolve(standin):
    from cca_zoo_b200.nonparametric import KCCA

    views = inputs("rbf")[0]
    with pytest.raises(ValueError, match="negative"):
        KCCA(kernel="chi2", gamma=0.5).fit(views)           # centred views have negative entries
    with pytest.raises(np.linalg.LinAlgError, match="did not converge"):
        KCCA(kernel="poly", degree=0.5).fit(views)          # (x.y / d + 1)^0.5 of negative bases: NaN
    assert standin.CALLS["syevj"] == 0


def test_kcca_kernel_params_broadcast_and_drop(standin):
    from cca_zoo_b200.nonparametric import KCCA
    from cca_zoo_b200.nonparametric._kcca import kernel_arguments

    assert kernel_arguments("rbf", None, 3.0, 2.0, {"foo": 1}, 4) == ("rbf", 0.25, 1.0, 1.0)
    assert kernel_arguments("sigmoid", 0.5, 3.0, 2.0, None, 4) == ("sigmoid", 0.5, 1.0, 2.0)
    assert kernel_arguments("poly", None, 3.0, 2.0, {}, 8) == ("poly", 0.125, 3.0, 2.0)
    assert kernel_arguments("additive_chi2", None, 3.0, 2.0, {}, 8)[0] == "additive_chi2"
    views = inputs("perview_four")[0]
    est = KCCA(**kwargs("perview_four")).fit(views)
    assert [a[0] for a in est._kernel_args] == ["rbf", "poly", "linear", "laplacian"]
    assert est._kernel_args[1][1] == 1.0 / views[1].shape[1]


def test_kcca_unsupported_paths(standin, monkeypatch):
    from cca_zoo_b200 import parallel
    from cca_zoo_b200.nonparametric import KCCA

    views = inputs("rbf")[0]
    with pytest.raises(NotImplementedError, match="partial_fit"):
        KCCA().partial_fit(views)
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(NotImplementedError, match="sharded"):
        KCCA().fit(views)


def test_kcca_is_exported():
    import cca_zoo_b200.nonparametric as nonparametric

    assert nonparametric.__all__ == ["KCCA"]
