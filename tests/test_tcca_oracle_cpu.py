"""TCCA without a GPU: the reference's data-space path (oracle/tcca.py:ref_tcca_fit) against the device algorithm
restated in float64 (cov_tcca_fit) and both against the reference's golden outputs
(tests/golden/reference_outputs_tcca.npz); ports of the reference's TCCA tests; and TCCA's host logic on the
torch-CPU stand-in (validation and limits before any kernel, the unsupported paths, the order of the random draws)."""
import numpy as np
import pytest
from sklearn.utils._param_validation import InvalidParameterError

from oracle import tcca as O
from tests.tcca_golden import CASES, inputs, kwargs, outputs


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max()) / max(float(np.abs(np.asarray(b)).max()), 1e-300)


def _split(name):
    kw = kwargs(name)
    return kw.pop("latent_dimensions"), kw


def test_tcca_golden_covers_the_cases():
    assert {"two_views", "three_views", "ragged4_c", "ragged5", "k_gt_p_rs0", "k_gt_p_rs42", "scalar_c", "eps_floor",
            "uncentred", "joint3"} <= set(CASES)
    assert any(c["stop"] for c in CASES.values()) and any(not c["stop"] and c["iters"] == 100 for c in CASES.values())


@pytest.mark.parametrize("name", sorted(CASES))
def test_ref_and_cov_restatements_match_golden(name):
    k, kw = _split(name)
    views = inputs(name)[0]
    ref = outputs(name)
    info = {}
    w_ref, _ = O.ref_tcca_fit(views, k, info=info, **kw)
    w_cov, means, st = O.cov_tcca_fit(views, k, **kw)
    assert info["iters"] == st["iters"] == ref["iters"]
    assert st["stop"] == ref["stop"]
    for a, b, g in zip(w_ref, w_cov, ref["w"]):
        assert _rel(b, a) < 1e-11
        assert _rel(a, g) < 1e-12
        assert _rel(b, g) < 1e-11
    np.testing.assert_allclose(st["rec"], ref["rec"], rtol=1e-10, atol=0)
    for mu, g in zip(means, ref["means"]):
        np.testing.assert_allclose(mu if kw.get("center", True) else 0 * mu, g, rtol=0, atol=1e-14)


def test_two_views_reduce_to_cca():
    """With two views the tensor is the whitened cross-covariance and CP-ALS finds its singular vectors: TCCA's
    weights are CCA's directions."""
    views = inputs("two_views")[0]
    w, _, _ = O.cov_tcca_fit(views, 2)
    X = [v - v.mean(axis=0) for v in views]
    n = X[0].shape[0]
    C11, C22, C12 = X[0].T @ X[0] / (n - 1), X[1].T @ X[1] / (n - 1), X[0].T @ X[1] / (n - 1)
    S = [O.whiteners(views)[i] for i in range(2)]
    U, _, Vt = np.linalg.svd(S[0] @ C12 @ S[1])
    cca = [S[0] @ U[:, :2], S[1] @ Vt[:2].T]
    for wt, wc, Cii in zip(w, cca, (C11, C22)):
        for r in range(2):
            cos = abs(wt[:, r] @ Cii @ wc[:, r]) / np.sqrt((wt[:, r] @ Cii @ wt[:, r]) * (wc[:, r] @ Cii @ wc[:, r]))
            assert abs(cos - 1.0) < 1e-10


def test_parafac_reproducible_and_seeded():
    """tests/linear/test_tcca.py: the same random_state gives the same fit; the random start columns come from one
    RandomState in mode order."""
    views = inputs("k_gt_p_rs0")[0]
    a, _ = O.ref_tcca_fit(views, 8, random_state=0)
    b, _ = O.ref_tcca_fit(views, 8, random_state=0)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    c, _ = O.ref_tcca_fit(views, 8, random_state=42)
    assert max(_rel(x, y) for x, y in zip(a, c)) > 1e-6


# ----------------------------------------------------------------------------------------------------------------------
# host logic on the torch-CPU stand-in
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_tcca

    fake_ops.install(monkeypatch)
    fake_ops_tcca.install(monkeypatch)
    return fake_ops_tcca


@pytest.mark.parametrize("name", sorted(CASES))
def test_tcca_on_the_standin_matches_golden(standin, name):
    from cca_zoo_b200.linear import TCCA

    k, kw = _split(name)
    views, test = inputs(name)
    est = TCCA(latent_dimensions=k, **kw).fit(views)
    ref = outputs(name)
    assert est._fit_info["iters"] == ref["iters"]
    assert est.n_views_ == len(views) and est.n_features_in_ == [v.shape[1] for v in views]
    assert est.n_samples_ == views[0].shape[0]
    for w, g in zip(est.weights_, ref["w"]):
        assert w.dtype == np.float64
        assert _rel(w, g) < 1e-11
    assert _rel(np.stack(est.transform(test)), ref["transform"]) < 1e-10
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=1e-10)


def test_tcca_random_draws_follow_tensorly_order(standin):
    from cca_zoo_b200.linear import TCCA
    from cca_zoo_b200.linear._tcca import random_start_columns

    views = inputs("k_gt_p_rs42")[0]
    TCCA(latent_dimensions=9, random_state=42).fit(views)
    rand = standin.CALLS["rand"]
    rng = np.random.RandomState(42)
    expect = [None, rng.random_sample((8, 1)), rng.random_sample((6, 3))]     # widths (10, 8, 6): modes 1 and 2
    assert rand[0] is None
    for got, want in zip(rand[1:], expect[1:]):
        np.testing.assert_array_equal(got, want)
    np.random.seed(7)
    first = random_start_columns([2, 3], 4, None)
    np.random.seed(7)
    assert all(np.array_equal(a, b) for a, b in zip(first, O.random_columns([2, 3], 4, np.random.mtrand._rand)))


def test_tcca_parameter_validation(standin):
    from cca_zoo_b200.linear import TCCA

    views = inputs("three_views")[0]
    for bad in (dict(random_state=-1), dict(eps=0.0), dict(eps=-1.0), dict(c=1.5), dict(c=-0.1),
                dict(latent_dimensions=0)):
        with pytest.raises(InvalidParameterError):
            TCCA(**bad).fit(views)
    with pytest.raises(ValueError, match="length 3"):
        TCCA(c=[0.1, 0.2]).fit(views)
    assert standin.CALLS["moment"] == 0 and standin.CALLS["fit"] == 0


def test_tcca_limits_raise_before_any_kernel(standin):
    from cca_zoo_b200.linear import TCCA

    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match="at most 64 latent"):
        TCCA(latent_dimensions=65).fit([rng.standard_normal((10, 3))] * 3)
    with pytest.raises(ValueError, match="at most 8 views"):
        TCCA().fit([rng.standard_normal((10, 2)) for _ in range(9)])
    with pytest.raises(ValueError, match="2\\^25"):
        TCCA().fit([np.zeros((4, 256)), np.zeros((4, 256)), np.zeros((4, 513))])
    with pytest.raises(ValueError, match="singular vectors"):
        TCCA(latent_dimensions=3).fit([rng.standard_normal((10, 10)), rng.standard_normal((10, 2))])
    assert standin.CALLS["moment"] == 0 and standin.CALLS["fit"] == 0


def test_tcca_unsupported_paths(standin, monkeypatch):
    from cca_zoo_b200 import parallel
    from cca_zoo_b200.linear import TCCA

    views = inputs("three_views")[0]
    with pytest.raises(NotImplementedError, match="partial_fit"):
        TCCA().partial_fit(views)
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(NotImplementedError, match="sharded"):
        TCCA().fit(views)


def test_tcca_is_exported():
    import cca_zoo_b200.linear as lin

    assert "TCCA" in lin.__all__
    from cca_zoo_b200.linear import TCCA  # noqa: F401
