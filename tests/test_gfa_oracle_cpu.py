"""The Gram-form restatement of GFA (oracle/gfa.py:cov_gfa_fit, the step-for-step reference of the kernel) against
the reference's golden outputs (tests/golden/reference_outputs_gfa.npz), and GFA's host logic on the torch-CPU
stand-in: the whole fit flow, parameter validation, the k bound, clone / get_params, pickling and the unsupported
paths."""
import inspect
import pickle

import numpy as np
import pytest
from sklearn.base import clone
from sklearn.utils._param_validation import InvalidParameterError

from oracle import gfa as O
from tests.gfa_golden import CASES, inputs, outputs


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max()) / max(float(np.abs(np.asarray(b)).max()), 1e-300)


def test_gfa_golden_covers_the_cases():
    assert {"two_views", "three_views", "prune", "no_drop", "uncentred", "private", "ragged4"} <= set(CASES)
    assert any(outputs(n)["n_components"] < CASES[n]["kwargs"]["latent_dimensions"] for n in CASES)   # a prune
    assert any(not CASES[n]["kwargs"].get("center", True) for n in CASES)
    assert any(len(outputs(n)["w"]) == 4 for n in CASES)


@pytest.mark.parametrize("name", sorted(CASES))
def test_cov_gfa_fit_matches_golden(name):
    kw = dict(CASES[name]["kwargs"])
    kw.pop("num_posterior_samples")
    k = kw.pop("latent_dimensions")
    ref = outputs(name)
    st, _ = O.cov_gfa_fit(inputs(name)[0], k, **kw)
    assert st["iters"] == ref["n_iter"] and st["k"] == ref["n_components"]
    assert _rel(st["W"], np.vstack(ref["w"])) < 1e-12
    assert _rel(st["alpha"], ref["view_relevance"]) < 1e-12


def test_data_space_restatement_matches_golden():
    name = "uncentred"
    kw = dict(CASES[name]["kwargs"])
    kw.pop("num_posterior_samples")
    r = O.ref_gfa_fit(inputs(name)[0], kw.pop("latent_dimensions"), **kw)
    ref = outputs(name)
    assert r["n_iter"] == ref["n_iter"] and r["k"] == ref["n_components"]
    assert _rel(np.vstack(r["W"]), np.vstack(ref["w"])) < 1e-12


# ---------------------------------------------------------------------------------------------------- host logic
@pytest.fixture
def standin(monkeypatch):
    from tests import fake_ops, fake_ops_gfa

    fake_ops.install(monkeypatch)
    fake_ops_gfa.install(monkeypatch)
    return fake_ops_gfa


def _gfa(**kw):
    from cca_zoo_b200.probabilistic import GFA

    return GFA(**kw)


@pytest.mark.parametrize("name", ["prune", "uncentred"])
def test_gfa_on_the_standin_matches_golden(standin, name):
    ref = outputs(name)
    views, test = inputs(name)
    est = _gfa(**CASES[name]["kwargs"]).fit(views)
    assert est.n_iter_ == ref["n_iter"] and est.n_components_ == ref["n_components"]
    assert _rel(np.vstack(est.weights_), np.vstack(ref["w"])) < 1e-9
    for key, val in ref["post"].items():
        assert _rel(est.posterior_samples_[key], val) < 1e-9, key
    assert _rel(est.transform(test)[0], ref["transform"]) < 1e-9
    assert np.abs(est.score(test) - ref["score"]).max() < 1e-9
    assert _rel(est.get_factor_loadings(test)[0], ref["loadings0"]) < 1e-9
    assert abs(est.log_likelihood(test) - ref["log_likelihood"]) < 1e-9 * abs(ref["log_likelihood"])
    assert standin.CALLS["run"] >= 1


def test_gfa_k_bound_raises_before_any_kernel(standin):
    views, _ = inputs("prune")
    before = standin.CALLS["run"]
    with pytest.raises(ValueError, match="at most 64"):
        _gfa(latent_dimensions=65).fit(views)
    assert standin.CALLS["run"] == before


def test_gfa_parameter_validation():
    views, _ = inputs("prune")
    for kw in (dict(latent_dimensions=0), dict(max_iter=-1), dict(drop_k="yes"), dict(num_posterior_samples=-2),
               dict(precision="fp8")):
        with pytest.raises(InvalidParameterError):
            _gfa(**kw).fit(views)


def test_gfa_unsupported_paths(standin, monkeypatch):
    views, _ = inputs("prune")
    with pytest.raises(NotImplementedError):
        _gfa().partial_fit(views)
    from cca_zoo_b200 import parallel

    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(NotImplementedError, match="sharded"):
        _gfa().fit(views)


def test_gfa_get_params_clone_and_pickle(standin):
    names = ["latent_dimensions", "center", "max_iter", "tol", "drop_k", "num_posterior_samples", "random_state",
             "precision", "device"]
    from cca_zoo_b200.probabilistic import GFA

    assert list(inspect.signature(GFA.__init__).parameters)[1:] == names
    est = _gfa(latent_dimensions=3, tol=1e-3, drop_k=False, num_posterior_samples=5)
    assert clone(est).get_params() == est.get_params()
    assert pickle.loads(pickle.dumps(est)).get_params() == est.get_params()
    views, _ = inputs("prune")
    est = _gfa(latent_dimensions=3, max_iter=30, num_posterior_samples=2).fit(views)
    back = pickle.loads(pickle.dumps(est))
    for a, b in zip(est.weights_, back.weights_):
        assert np.array_equal(a, b)
    assert back.n_iter_ == 30 and back.posterior_samples_["z"].shape == (2, views[0].shape[0], est.n_components_)
