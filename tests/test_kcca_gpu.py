"""KCCA on the GPU against the reference's golden outputs (tests/golden/reference_outputs_kcca.npz), within the
tolerances set from each case's spread, for float64 and float32 views: weights_, held-out transform (the test views not
centred) and score.  Refits are bit-identical; every limit and parameter error is raised before any kernel launches;
the data-dependent errors before the first eigensolve; syevj converges on a seeded n = 8192 rbf kernel matrix."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import _lib, ops
from cca_zoo_b200.nonparametric import KCCA
from oracle import kcca as O
from tests.kcca_golden import CASES, inputs, kwargs, outputs, tolerances

pytestmark = pytest.mark.gpu


def _launches():
    return int(_lib.load().ccab_launch_count())


def _check(est, name, test):
    ref = outputs(name)
    tol_w, tol_s = tolerances(name)
    for w in est.weights_:
        assert w.dtype == np.float64
    assert O.rel_err(est.weights_, ref["w"]) < tol_w
    est.weights_ = O.align(est.weights_, ref["w"])
    tr = np.stack(est.transform(test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_s
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=tol_s)


@pytest.mark.parametrize("name", sorted(CASES))
def test_kcca_matches_golden_float64(name):
    views, test = inputs(name)
    _check(KCCA(**kwargs(name)).fit(views), name, test)


def test_kcca_matches_golden_float32():
    """The reference ran on the float64 copy of float32-rounded views: float32 views are computed in float64."""
    views, test = inputs("rbf_f32")
    _check(KCCA(**kwargs("rbf_f32")).fit([v.astype(np.float32) for v in views]), "rbf_f32", test)


def test_kcca_refits_bit_identical_and_inputs_unmodified():
    views = inputs("perview_four")[0]
    dev = [torch.from_numpy(v).cuda() for v in views]
    before = [v.clone() for v in dev]
    a = KCCA(**kwargs("perview_four")).fit(dev)
    b = KCCA(**kwargs("perview_four")).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        np.testing.assert_array_equal(x, y)
    assert all(torch.equal(x, y) for x, y in zip(dev, before))
    assert all(t.is_cuda and t.dtype == torch.float64 for t in a.train_views_)


def test_kcca_errors_before_any_kernel():
    rng = np.random.default_rng(0)
    views = [rng.standard_normal((20, 3)), rng.standard_normal((20, 4))]
    torch.cuda.synchronize()
    start = _launches()
    cases = [(ValueError, dict(), [rng.standard_normal((10, 2)) for _ in range(9)]),
             (ValueError, dict(), [np.zeros((8193, 1))] * 2),
             (ValueError, dict(), [np.zeros((4097, 1))] * 4),
             (ValueError, dict(kernel="precomputed"), views),
             (ValueError, dict(kernel="nope"), views),
             (ValueError, dict(kernel=lambda x, y: x @ y.T), views),
             (TypeError, dict(kernel="rbf", kernel_params={"gamma": 1.0}), views),
             (TypeError, dict(kernel="poly", kernel_params=[{}, {"coef0": 1.0}]), views)]
    for exc, kw, v in cases:
        with pytest.raises(exc):
            KCCA(**kw).fit(v)
    assert _launches() == start


def test_kcca_data_errors_before_the_eigensolve(monkeypatch):
    views = inputs("rbf")[0]
    calls = []
    real = ops.syevj
    monkeypatch.setattr(ops, "syevj", lambda *a, **k: calls.append(1) or real(*a, **k))
    with pytest.raises(ValueError, match="negative"):
        KCCA(kernel="chi2", gamma=0.5).fit(views)
    with pytest.raises(np.linalg.LinAlgError, match="did not converge"):
        KCCA(kernel="poly", degree=0.5).fit(views)
    assert not calls


def test_syevj_converges_on_an_n8192_rbf_kernel_matrix():
    from cca_zoo_b200.datasets import joint_data

    x = joint_data(n_views=1, n_samples=8192, n_features=64, latent_dimensions=4, random_state=0)[0]
    x = (x - x.mean(axis=0)) / x.std(axis=0)
    X = torch.from_numpy(x).cuda()
    K = ops.pairwise_kernel(X, None, "rbf", gamma=1.0 / 64)
    shift = float(K.abs().sum(dim=1).max())
    lam, evt, info = ops.syevj(K, shift=shift, return_info=True)
    print(f"n = 8192 rbf kernel matrix: syevj converged={info['converged']} in {info['sweeps']} sweeps")
    assert info["converged"] and info["sweeps"] < 64
    U = evt[:8]
    resid = ops.gemm(U, K) - lam[:8, None] * U
    assert float(resid.abs().max()) < 1e-9 * float(lam[0])
