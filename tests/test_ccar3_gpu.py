"""CCAR3 on the GPU: golden parity with the reference (tests/golden/reference_outputs_ccar3.npz) for float64 views
(weights up to a joint sign per component pair within the recorded spread, exact ADMM iteration counts and zero-row
patterns, held-out transform and score) and float32 views, the reference's behavioural tests, bit-identical refits,
no launch before a validation error, and one large p > n fit against the float64 moment-form restatement."""
import numpy as np
import pytest
import torch
from sklearn.utils._param_validation import InvalidParameterError

from cca_zoo_b200 import _lib
from cca_zoo_b200.datasets import conftest_views, joint_data
from cca_zoo_b200.linear import CCAR3
from oracle import ccar3 as O
from tests.ccar3_golden import CASES, align, inputs, kwargs, outputs, rel_err, tolerance

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_parity_float64(name):
    kw = kwargs(name)
    views, test = inputs(name)
    ref = outputs(name)
    est = CCAR3(**kw).fit(views)
    if kw.get("highdim", True):
        assert est._fit_info["iters"] == ref["iters"]
    for w, g in zip(est.weights_, ref["w"]):
        assert w.dtype == np.float64 and w.shape == g.shape
        # the reference's LAPACK SVD leaves rounding-level entries (~1e-17) in the rows the ADMM zeroed; the one-sided
        # Jacobi left vectors B v / sigma keep them exactly zero
        gn = np.linalg.norm(g, axis=1)
        assert np.array_equal(np.linalg.norm(w, axis=1) == 0, gn <= 1e-12 * max(float(gn.max()), 1e-300))
    if not np.any(ref["w"][0]):
        assert not np.any(est.weights_[0]) and not np.any(est.weights_[1])
        return
    assert rel_err(align(est.weights_, ref["w"]), ref["w"]) < tolerance(name)
    tr = est.transform(test)
    assert rel_err(align(tr, ref["transform"]), ref["transform"]) < tolerance(name, "spread_t")
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=tolerance(name, "spread_score"))


@pytest.mark.parametrize("name", ["two_views_lam0.05_lw1", "correlated_views_lam0.3_lw0", "uncentred", "ragged"])
def test_golden_parity_float32(name):
    kw = kwargs(name)
    views, _ = inputs(name)
    ref = outputs(name)
    est = CCAR3(**kw).fit([v.astype(np.float32) for v in views])
    assert all(w.dtype == np.float64 for w in est.weights_)
    assert rel_err(align(est.weights_, ref["w"]), ref["w"]) < 1e-3


def test_reference_behaviour():
    corr = conftest_views("correlated_views")
    lo = CCAR3(latent_dimensions=2, highdim=False, ledoit_wolf=False).fit(corr).score(corr)
    hi = CCAR3(latent_dimensions=2, highdim=True, ledoit_wolf=False, lambda_=0.0, tol=1e-8).fit(corr).score(corr)
    np.testing.assert_allclose(hi, lo, atol=1e-4)
    dense = CCAR3(latent_dimensions=2, lambda_=0.0, ledoit_wolf=False).fit(corr)
    sparse = CCAR3(latent_dimensions=2, lambda_=0.05, ledoit_wolf=False).fit(corr)
    assert np.all(np.linalg.norm(dense.weights_[0], axis=1) > 1e-8)
    rs = np.linalg.norm(sparse.weights_[0], axis=1)
    assert np.any(rs == 0.0) and np.any(rs > 1e-8)
    two = conftest_views("two_views")
    assert CCAR3(latent_dimensions=2).fit(two).score(two).shape == (2,)
    with pytest.raises(ValueError, match="exactly 2 views"):
        CCAR3().fit(conftest_views("three_views"))


def test_refits_are_bit_identical():
    views, _ = inputs("ragged")
    a = CCAR3(latent_dimensions=3, lambda_=0.02).fit(views)
    b = CCAR3(latent_dimensions=3, lambda_=0.02).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        assert np.array_equal(x, y)
    assert a._fit_info == b._fit_info


def test_no_launch_before_validation_errors():
    lib = _lib.load()
    two = conftest_views("two_views")
    rng = np.random.default_rng(0)
    before = lib.ccab_launch_count()
    for bad in (lambda: CCAR3(rho=0.0).fit(two), lambda: CCAR3().fit(conftest_views("three_views")),
                lambda: CCAR3().fit([rng.standard_normal((20, 3)), rng.standard_normal((20, 600))]),
                lambda: CCAR3().fit([rng.standard_normal((20, 16385)), rng.standard_normal((20, 3))])):
        with pytest.raises((ValueError, InvalidParameterError)):
            bad()
    assert lib.ccab_launch_count() == before


def test_large_p_gt_n_fit_matches_moment_form():
    views = joint_data(n_views=2, n_samples=1000, n_features=[4096, 512], latent_dimensions=4, signal_to_noise=1.0,
                       random_state=11)
    kw = dict(lambda_=0.05, max_iter=30)
    est = CCAR3(latent_dimensions=4, **kw).fit(views)
    info = {}
    w, _ = O.moment_ccar3_fit(views, 4, info=info, **kw)
    assert est._fit_info["iters"] == info["iters"]
    sig = info["sigma"]
    assert np.all(-np.diff(sig[:5]) > 1e-3 * sig[0])
    assert rel_err(align(est.weights_, w), w) < 1e-6
    assert np.array_equal(np.linalg.norm(est.weights_[0], axis=1) == 0, np.linalg.norm(w[0], axis=1) == 0)
    assert torch.cuda.is_available()
