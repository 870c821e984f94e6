"""GPU parity of GFA against the reference's golden outputs (tests/golden/reference_outputs_gfa.npz,
oracle/make_golden_gfa.py): weights, view relevance, iteration count, pruning, posterior samples, transform, score,
factor loadings and the held-out log-likelihood.  float64 views: 1e-9 (relative to the largest entry); float32 views
(3xTF32 moments): 1e-3, with the iteration count not pinned."""
import numpy as np
import pytest
import torch

from tests.gfa_golden import CASES, inputs, outputs

pytestmark = pytest.mark.gpu

F32_TOL = 1e-3


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    return float(np.abs(a - b).max()) / max(float(np.abs(b).max()), 1e-300)


def _fit(name, dtype=np.float64):
    from cca_zoo_b200.probabilistic import GFA

    views, test = inputs(name)
    views = [v.astype(dtype) for v in views]
    return GFA(**CASES[name]["kwargs"]).fit(views), [t.astype(dtype) for t in test]


@pytest.mark.parametrize("name", sorted(CASES))
def test_gfa_matches_reference_golden(name):
    ref = outputs(name)
    est, test = _fit(name)
    assert est.n_iter_ == ref["n_iter"]
    assert est.n_components_ == ref["n_components"]
    assert _rel(np.vstack(est.weights_), np.vstack(ref["w"])) < 1e-9
    assert _rel(est.view_relevance_, ref["view_relevance"]) < 1e-9
    for mu, r in zip(est.means_, ref["means"]):
        assert np.allclose(mu, r, rtol=0, atol=1e-12)
    assert set(est.posterior_samples_) == set(ref["post"])
    for key, val in ref["post"].items():
        assert _rel(est.posterior_samples_[key], val) < 1e-9, key
    t = est.transform(test)
    assert isinstance(t, list) and len(t) == 1
    assert _rel(t[0], ref["transform"]) < 1e-9
    assert np.abs(est.score(test) - ref["score"]).max() < 1e-9
    assert abs(est.log_likelihood(test) - ref["log_likelihood"]) < 1e-9 * max(1.0, abs(ref["log_likelihood"]))
    assert _rel(est.get_factor_loadings(test)[0], ref["loadings0"]) < 1e-9
    assert est.n_views_ == len(est.weights_) and est.n_samples_ == inputs(name)[0][0].shape[0]


@pytest.mark.parametrize("name", sorted(CASES))
def test_gfa_float32_views(name):
    ref = outputs(name)
    est, test = _fit(name, np.float32)
    assert est.n_components_ == ref["n_components"]
    assert _rel(np.vstack(est.weights_), np.vstack(ref["w"])) < F32_TOL
    assert np.abs(est.score(test) - ref["score"]).max() < F32_TOL


def test_gfa_cuda_tensor_inputs_match_host_inputs():
    from cca_zoo_b200.probabilistic import GFA

    name = "prune"
    views, test = inputs(name)
    a = GFA(**CASES[name]["kwargs"]).fit(views)
    b = GFA(**CASES[name]["kwargs"]).fit([torch.from_numpy(v).cuda() for v in views])
    for x, y in zip(a.weights_, b.weights_):
        assert np.array_equal(x, y)
    dev_test = [torch.from_numpy(v).cuda() for v in test]
    assert _rel(b.transform(dev_test)[0], a.transform(test)[0]) < 1e-12
    assert np.abs(b.score(dev_test) - a.score(test)).max() < 1e-9


def test_gfa_reruns_are_bit_identical():
    a, _ = _fit("ragged4")
    b, _ = _fit("ragged4")
    for x, y in zip(a.weights_, b.weights_):
        assert np.array_equal(x, y)


def test_gfa_identifies_private_factor():
    """The reference's test_gfa_identifies_private_factor on the device (its data and random_state=0)."""
    from cca_zoo_b200.probabilistic import GFA

    views, _ = inputs("private")
    est = GFA(latent_dimensions=4, random_state=0).fit(views)
    assert np.max(est.view_relevance_[1] / est.view_relevance_[0]) > 1e4
