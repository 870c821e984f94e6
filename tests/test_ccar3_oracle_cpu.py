"""CCAR3 without a GPU: the moment-form restatement (oracle/ccar3.py:moment_ccar3_fit) against the reference's golden
outputs (tests/golden/reference_outputs_ccar3.npz), the Ledoit-Wolf scalar against sklearn, ports of the reference's
CCAR3 tests, and CCAR3's host logic on the torch-CPU stand-in (parameter errors and their order, the view count,
padding, the zero-B path, the unsupported paths)."""
import numpy as np
import pytest
from sklearn.covariance import LedoitWolf
from sklearn.utils._param_validation import InvalidParameterError

from cca_zoo_b200.datasets import conftest_views
from cca_zoo_b200.linear._ccar3 import ledoit_wolf_shrinkage
from oracle import ccar3 as O
from tests.ccar3_golden import CASES, align, inputs, kwargs, outputs, rel_err, tolerance


def _split(name):
    kw = kwargs(name)
    return kw.pop("latent_dimensions"), kw


def test_ccar3_golden_covers_the_cases():
    names = set(CASES)
    assert {"uncentred", "tight_tol", "capped", "padded", "zero_b", "p_gt_n", "ragged"} <= names
    assert any(n.endswith("_lw0") for n in names) and any(n.endswith("_lw1") for n in names)
    assert any("lowdim" in n for n in names) and any("lam0.3" in n for n in names)
    assert CASES["capped"]["iters"] == 5


@pytest.mark.parametrize("name", sorted(CASES))
def test_moment_restatement_matches_golden(name):
    k, kw = _split(name)
    views, _ = inputs(name)
    ref = outputs(name)
    info = {}
    w, means = O.moment_ccar3_fit(views, k, info=info, **kw)
    if kw.get("highdim", True):
        assert info["iters"] == ref["iters"]
    if not np.any(ref["w"][0]):
        assert not np.any(w[0]) and not np.any(w[1])
        return
    assert rel_err(align(w, ref["w"]), ref["w"]) < max(tolerance(name), 1e-9)
    for mu, g in zip(means, ref["means"]):
        np.testing.assert_allclose(mu if kw.get("center", True) else 0 * mu, g, rtol=0, atol=1e-13)


@pytest.mark.parametrize("shift", [0.0, 3.0])
@pytest.mark.parametrize("q", [1, 2, 8])
def test_ledoit_wolf_scalar_matches_sklearn(shift, q):
    rng = np.random.default_rng(q)
    Y = rng.standard_normal((57, q)) @ rng.standard_normal((q, q)) + shift
    lw = LedoitWolf().fit(Y)
    Yc = Y - Y.mean(axis=0)
    Sc = Yc.T @ Yc / Y.shape[0]
    s, mu = ledoit_wolf_shrinkage(float(np.sum(Sc ** 2)), float(np.trace(Sc)), float(np.sum(np.sum(Yc ** 2, 1) ** 2)),
                                  Y.shape[0], q)
    assert abs(s - lw.shrinkage_) < 1e-13
    np.testing.assert_allclose((1 - s) * Sc + s * mu * np.eye(q), lw.covariance_, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(O.ledoit_wolf_data(Y)[0], lw.covariance_, rtol=1e-13, atol=1e-15)


def test_inverse_admm_matches_data_space_admm():
    """The inverse form B = B0 + rho M (Z - U) is the reference's two triangular solves, iterate for iterate."""
    X, Y = conftest_views("correlated_views")
    X, Y = X - X.mean(0), Y - Y.mean(0)
    n, p = X.shape
    Si = O.sqrt_inv_psd(Y.T @ Y / n)
    M = np.linalg.inv(X.T @ X / n + (1.0 + 1e-8) * np.eye(p))
    B0 = M @ (X.T @ (Y @ Si) / n)
    for max_iter in (1, 2, 7, 10_000):
        ta, tb = [], []
        Za, _ = O.admm_ref(X, Y @ Si, 0.05, 1.0, max_iter, 1e-4, 1e-8, ta)
        Zb, _, it, _, _, _ = O.admm_inverse(M, B0, 0.05, 1.0, 1e-4, max_iter, tb)
        assert it == len(ta) == len(tb)
        np.testing.assert_allclose(Zb, Za, rtol=0, atol=1e-12)
        assert np.array_equal(np.linalg.norm(Za, axis=1) == 0, np.linalg.norm(Zb, axis=1) == 0)


# ----------------------------------------------------------------------------------------------------------------------
# ports of the reference's tests (tests/linear/test_eigendecomposition.py, test_parameter_constraints.py), restated
# ----------------------------------------------------------------------------------------------------------------------
def test_ref_lambda0_highdim_matches_lowdim():
    views = conftest_views("correlated_views")
    kw = dict(k=2, ledoit_wolf=False)
    lo, _ = O.moment_ccar3_fit(views, highdim=False, **kw)
    hi, _ = O.moment_ccar3_fit(views, highdim=True, lambda_=0.0, tol=1e-8, **kw)
    X = [v - v.mean(0) for v in views]
    s_lo = [np.corrcoef(X[0] @ lo[0][:, j], X[1] @ lo[1][:, j])[0, 1] for j in range(2)]
    s_hi = [np.corrcoef(X[0] @ hi[0][:, j], X[1] @ hi[1][:, j])[0, 1] for j in range(2)]
    np.testing.assert_allclose(s_hi, s_lo, atol=1e-4)


def test_ref_sparsity():
    views = conftest_views("two_views")
    w, _ = O.moment_ccar3_fit(views, 2, lambda_=0.3, ledoit_wolf=False, tol=1e-8)
    rn = np.linalg.norm(w[0], axis=1)
    assert np.any(rn < 1e-3) and np.any(rn > 1e-2)
    corr = conftest_views("correlated_views")
    dense, _ = O.moment_ccar3_fit(corr, 2, lambda_=0.0, ledoit_wolf=False)
    sparse, _ = O.moment_ccar3_fit(corr, 2, lambda_=0.05, ledoit_wolf=False)
    assert np.all(np.linalg.norm(dense[0], axis=1) > 1e-8)
    rs = np.linalg.norm(sparse[0], axis=1)
    assert np.any(rs == 0.0) and np.any(rs > 1e-8)


# ----------------------------------------------------------------------------------------------------------------------
# host logic on the torch-CPU stand-in
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_ccar3

    fake_ops.install(monkeypatch)
    fake_ops_ccar3.install(monkeypatch)
    return fake_ops_ccar3


@pytest.mark.parametrize("name", sorted(CASES))
def test_ccar3_on_the_standin_matches_golden(standin, name):
    from cca_zoo_b200.linear import CCAR3

    k, kw = _split(name)
    views, test = inputs(name)
    est = CCAR3(latent_dimensions=k, **kw).fit(views)
    ref = outputs(name)
    info = est._fit_info
    assert info["route"] == ("admm" if kw.get("highdim", True) else "closed_form")
    if kw.get("highdim", True):
        assert info["iters"] == ref["iters"]
    assert info["r_eff"] == min(k, *[v.shape[1] for v in views])
    assert (info["shrinkage"] is None) == (not kw.get("ledoit_wolf", True))
    assert est.n_views_ == 2 and est.n_features_in_ == [v.shape[1] for v in views]
    assert est.n_samples_ == views[0].shape[0]
    for w, g in zip(est.weights_, ref["w"]):
        assert w.dtype == np.float64 and w.shape == g.shape
    if not np.any(ref["w"][0]):
        assert not np.any(est.weights_[0]) and not np.any(est.weights_[1])
        return
    assert rel_err(align(est.weights_, ref["w"]), ref["w"]) < max(tolerance(name), 1e-9)
    tr = est.transform(test)
    assert rel_err(align(tr, ref["transform"]), ref["transform"]) < max(tolerance(name, "spread_t"), 1e-9)
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=max(tolerance(name, "spread_score"), 1e-9))


def test_padding_and_zero_b_on_the_standin(standin):
    from cca_zoo_b200.linear import CCAR3

    views = conftest_views("two_views")
    est = CCAR3(latent_dimensions=9).fit(views)
    assert est.weights_[0].shape == (10, 9) and est.weights_[1].shape == (8, 9)
    assert not np.any(est.weights_[0][:, 8:]) and not np.any(est.weights_[1][:, 8:])
    assert np.all(np.linalg.norm(est.weights_[0][:, :8], axis=0) > 0)
    zero = CCAR3(latent_dimensions=3, lambda_=1e3).fit(views)
    assert zero.weights_[0].shape == (10, 3) and not np.any(zero.weights_[0]) and not np.any(zero.weights_[1])


@pytest.mark.parametrize("kw", [{"lambda_": -0.1}, {"highdim": "nope"}, {"ledoit_wolf": "nope"}, {"rho": 0.0},
                                {"max_iter": 0}, {"tol": 0.0}, {"eps": 0.0}, {"latent_dimensions": 0}])
def test_invalid_params_raise_before_any_call(standin, kw):
    from cca_zoo_b200.linear import CCAR3

    with pytest.raises(InvalidParameterError):
        CCAR3(**kw).fit(conftest_views("two_views"))
    assert standin.CALLS == {"norm4": 0, "admm": 0}


def test_errors_and_their_order(standin, monkeypatch):
    from cca_zoo_b200 import ops
    from cca_zoo_b200.linear import CCAR3

    three = conftest_views("three_views")
    with pytest.raises(InvalidParameterError):               # parameters first
        CCAR3(rho=-1.0).fit(three)
    with pytest.raises(ValueError, match="CCAR3 requires exactly 2 views, got 3. Use MCCA for more than 2 views."):
        CCAR3().fit(three)
    with pytest.raises(ValueError, match="same number of samples|inconsistent"):   # views before the view count
        CCAR3().fit([three[0], three[1][:10], three[2]])
    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match="at most 512"):
        CCAR3().fit([rng.standard_normal((20, 3)), rng.standard_normal((20, ops.CCAR3_MAX_Q + 1))])
    CCAR3(highdim=False).fit([rng.standard_normal((20, 3)), rng.standard_normal((20, ops.CCAR3_MAX_Q + 1))])
    monkeypatch.setattr(ops, "CCAR3_MAX_P", 4)
    from tests import fake_ops

    monkeypatch.setattr(fake_ops, "CCAR3_MAX_P", 4)
    standin.CALLS.update(norm4=0, admm=0)
    with pytest.raises(ValueError, match="at most 4"):
        CCAR3().fit([rng.standard_normal((20, 5)), rng.standard_normal((20, 2))])
    assert standin.CALLS == {"norm4": 0, "admm": 0}


def test_unsupported_paths(standin):
    from cca_zoo_b200.linear import CCAR3

    with pytest.raises(NotImplementedError):
        CCAR3().partial_fit(conftest_views("two_views"))


def test_reference_fit_transform_and_score_shapes(standin):
    from cca_zoo_b200.linear import CCAR3

    views = conftest_views("two_views")
    for highdim in (False, True):
        model = CCAR3(latent_dimensions=2, highdim=highdim).fit(views)
        for arr, v in zip(model.transform(views), views):
            assert arr.shape == (v.shape[0], 2)
        assert model.score(views).shape == (2,)
    CCAR3(lambda_=0.1, highdim=False, rho=2.0, max_iter=100, tol=1e-3).fit(views)
