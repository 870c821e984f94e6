"""TCCA on the GPU against the reference's golden outputs (tests/golden/reference_outputs_tcca.npz): weights_,
transform and score to 1e-9 for float64 views and 1e-3 for float32 views, the iteration counts, bit-identical refits,
unmodified inputs and the tensor-size limit."""
import numpy as np
import pytest
import torch

from cca_zoo_b200.linear import TCCA
from tests.tcca_golden import CASES, inputs, kwargs, outputs

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max()) / max(float(np.abs(np.asarray(b)).max()), 1e-300)


@pytest.mark.parametrize("name", sorted(CASES))
def test_tcca_matches_golden_float64(name):
    views, test = inputs(name)
    ref = outputs(name)
    est = TCCA(**kwargs(name)).fit(views)
    assert est._fit_info["iters"] == ref["iters"] and est._fit_info["stop"] == ref["stop"]
    for w, g in zip(est.weights_, ref["w"]):
        assert w.dtype == np.float64
        assert _rel(w, g) < 1e-9
    assert _rel(np.stack(est.transform(test)), ref["transform"]) < 1e-9
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=1e-9)
    tdev = est.transform([torch.from_numpy(v).cuda() for v in test])
    assert _rel(np.stack(tdev), ref["transform"]) < 1e-9


@pytest.mark.parametrize("name", ["two_views", "three_views", "joint3", "uncentred"])
def test_tcca_matches_golden_float32(name):
    views, test = inputs(name)
    ref = outputs(name)
    est = TCCA(**kwargs(name)).fit([v.astype(np.float32) for v in views])
    for w, g in zip(est.weights_, ref["w"]):
        assert w.dtype == np.float64
        assert _rel(w, g) < 1e-3
    np.testing.assert_allclose(est.score(test), ref["score"], rtol=0, atol=1e-3)


def test_tcca_refits_bit_identical_and_inputs_unmodified():
    views = inputs("ragged4_c")[0]
    dev = [torch.from_numpy(v).cuda() for v in views]
    before = [v.clone() for v in dev]
    host_before = [v.copy() for v in views]
    a = TCCA(**kwargs("ragged4_c")).fit(dev)
    b = TCCA(**kwargs("ragged4_c")).fit(dev)
    for x, y in zip(a.weights_, b.weights_):
        np.testing.assert_array_equal(x, y)
    c = TCCA(**kwargs("ragged4_c")).fit(views)
    for x, y in zip(a.weights_, c.weights_):
        np.testing.assert_array_equal(x, y)
    assert all(torch.equal(x, y) for x, y in zip(dev, before))
    assert all(np.array_equal(x, y) for x, y in zip(views, host_before))


def test_tcca_tensor_limit():
    views = [np.zeros((4, 256)), np.zeros((4, 256)), np.zeros((4, 513))]
    with pytest.raises(ValueError, match="2\\^25"):
        TCCA().fit(views)
