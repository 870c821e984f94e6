"""KGCCA and KTCCA on the GPU against the reference's golden outputs (tests/golden/reference_outputs_{kgcca,ktcca}.npz),
within the tolerances set from each case's spreads, for float64 and float32 views: weights_, held-out transform (the
test views not centred) and score.  Refits are bit-identical and leave device inputs unmodified; every limit and
parameter error is raised before any kernel launches; the data-dependent errors before the first eigensolve; and each
estimator matches its numpy eigenbasis restatement once at a large supported shape."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import _lib, ops
from cca_zoo_b200.nonparametric import KGCCA, KTCCA
from oracle import kcca as O
from oracle import kgcca as OG
from oracle import ktcca as OT
from tests.kgcca_ktcca_golden import GOLDEN

pytestmark = pytest.mark.gpu

ESTIMATORS = {"KGCCA": KGCCA, "KTCCA": KTCCA}
ALL_CASES = [(model, name) for model, g in GOLDEN.items() for name in sorted(g.cases)]


def _launches():
    return int(_lib.load().ccab_launch_count())


def _check(est, model, name, test):
    g = GOLDEN[model]
    ref = g.outputs(name)
    tol_w, tol_t, tol_c = g.tolerances(name)
    for w in est.weights_:
        assert w.dtype == np.float64
    assert O.rel_err(est.weights_, ref["w"]) < tol_w
    est.weights_ = O.align(est.weights_, ref["w"])
    tr = np.stack(est.transform(test))
    assert np.abs(tr - ref["transform"]).max() / np.abs(ref["transform"]).max() < tol_t
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=tol_c)
    if model == "KTCCA":
        assert est._fit_info["iters"] == g.cases[name]["iters"]


@pytest.mark.parametrize("model,name", ALL_CASES)
def test_matches_golden_float64(model, name):
    views, test = GOLDEN[model].inputs(name)
    _check(ESTIMATORS[model](**GOLDEN[model].kwargs(name)).fit(views), model, name, test)


@pytest.mark.parametrize("model", sorted(ESTIMATORS))
def test_matches_golden_float32(model):
    """The reference ran on the float64 copy of float32-rounded views: float32 views are computed in float64."""
    views, test = GOLDEN[model].inputs("rbf_f32")
    est = ESTIMATORS[model](**GOLDEN[model].kwargs("rbf_f32")).fit([v.astype(np.float32) for v in views])
    _check(est, model, "rbf_f32", test)


@pytest.mark.parametrize("model", sorted(ESTIMATORS))
def test_refits_bit_identical_and_inputs_unmodified(model):
    g = GOLDEN[model]
    views = g.inputs("perview_four")[0]
    dev = [torch.from_numpy(v).cuda() for v in views]
    before = [v.clone() for v in dev]
    a = ESTIMATORS[model](**g.kwargs("perview_four")).fit(dev)
    b = ESTIMATORS[model](**g.kwargs("perview_four")).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        np.testing.assert_array_equal(x, y)
    assert all(torch.equal(x, y) for x, y in zip(dev, before))
    assert all(t.is_cuda and t.dtype == torch.float64 for t in a.train_views_)


def test_errors_before_any_kernel():
    rng = np.random.default_rng(0)
    views = [rng.standard_normal((20, 3)), rng.standard_normal((20, 4))]
    torch.cuda.synchronize()
    start = _launches()
    common = [(ValueError, dict(kernel="precomputed"), views),
              (ValueError, dict(kernel="nope"), views),
              (ValueError, dict(kernel=lambda x, y: x @ y.T), views),
              (ValueError, dict(c=[0.1, 0.2, 0.3]), views),
              (TypeError, dict(kernel="rbf", kernel_params={"gamma": 1.0}), views),
              (TypeError, dict(kernel="poly", kernel_params=[{}, {"coef0": 1.0}]), views)]
    cases = [(KGCCA, *c) for c in common] + [(KTCCA, *c) for c in common]
    cases += [(KGCCA, ValueError, dict(), [rng.standard_normal((10, 2)) for _ in range(9)]),
              (KGCCA, ValueError, dict(), [np.zeros((8193, 1))] * 2),
              (KGCCA, ValueError, dict(view_weights=[1.0]), views),
              (KTCCA, ValueError, dict(), [rng.standard_normal((2, 2)) for _ in range(9)]),
              (KTCCA, ValueError, dict(latent_dimensions=65), views),
              (KTCCA, ValueError, dict(), [np.zeros((323, 1))] * 3),
              (KTCCA, ValueError, dict(), [np.zeros((5793, 1))] * 2)]
    for Est, exc, kw, v in cases:
        with pytest.raises(exc):
            Est(**kw).fit(v)
    assert _launches() == start


@pytest.mark.parametrize("model", sorted(ESTIMATORS))
def test_data_errors_before_the_eigensolve(monkeypatch, model):
    views = GOLDEN[model].inputs("rbf_three")[0]
    calls = []
    real = ops.syevj
    monkeypatch.setattr(ops, "syevj", lambda *a, **k: calls.append(1) or real(*a, **k))
    with pytest.raises(ValueError, match="negative"):
        ESTIMATORS[model](kernel="chi2", gamma=0.5).fit(views)
    with pytest.raises(np.linalg.LinAlgError, match="did not converge"):
        ESTIMATORS[model](kernel="poly", degree=0.5).fit(views)
    assert not calls


def _large_views(m, n, dims, seed):
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=m, n_samples=n, n_features=dims, latent_dimensions=2, signal_to_noise=2.0,
                       random_state=seed)
    return [(v - v.mean(axis=0)) / v.std(axis=0) for v in views]


def test_kgcca_at_n2048_matches_its_restatement():
    views = _large_views(3, 2048, [32, 24, 16], 0)
    kw = dict(c=0.1, kernel="rbf")
    est = KGCCA(latent_dimensions=3, **kw).fit(views)
    info = {}
    w, X, st = OG.eig_kgcca_fit(views, 3, info=info, **kw)
    ev = info["evals"]
    err = O.rel_err(est.weights_, w)
    s_err = O.rel_err(O.align(O.transform(X, st, est.weights_, X), O.transform(X, st, w, X)),
                      O.transform(X, st, w, X))
    print(f"KGCCA n = 2048 rbf: sweeps {est._fit_info}, gap {(ev[2] - ev[3]) / ev[0]:.1e}, weights err {err:.1e}, "
          f"scores err {s_err:.1e}")
    assert err < 1e-6 and s_err < 1e-8


def test_ktcca_at_n322_three_views_matches_its_restatement():
    views = _large_views(3, 322, [8, 6, 5], 1)
    kw = dict(c=0.1, kernel="rbf", random_state=0)
    est = KTCCA(latent_dimensions=2, **kw).fit(views)
    info = {}
    w, X, st = OT.eig_ktcca_fit(views, 2, info=info, **kw)
    err = O.rel_err(est.weights_, w)
    s_err = O.rel_err(O.align(O.transform(X, st, est.weights_, X), O.transform(X, st, w, X)),
                      O.transform(X, st, w, X))
    print(f"KTCCA n = 322, 3 views: iters {est._fit_info['iters']} (numpy {info['state']['iters']}), weights err "
          f"{err:.1e}, scores err {s_err:.1e}")
    assert est._fit_info["iters"] == info["state"]["iters"]
    assert err < 1e-6 and s_err < 1e-8
