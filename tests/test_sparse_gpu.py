"""GPU parity of the sparse / ALS estimators (PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span, SCCA_ADMM) against the
reference's golden vectors (tests/golden/reference_outputs_sparse.npz, oracle/make_golden_sparse.py) and the Gram-space
restatement (oracle/sparse.py:cov_als_fit).  Tolerances: 1e-9 for float64 inputs, 1e-3 for float32 inputs (they
iterate in float64 on a covariance of float32-grade accuracy)."""
import json
import os

import numpy as np
import pytest
import torch

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import sparse as S

pytestmark = pytest.mark.gpu

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_sparse.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_sparse.npz"))
CASES = {c["name"]: c for c in META["cases"]}
KINDS = ("pls", "pmd", "parkhomenko", "span", "admm")


def _cls(kind):
    from cca_zoo_b200 import linear

    return {"pls": linear.PLS_ALS, "pmd": linear.SCCA_PMD, "parkhomenko": linear.ParkhomenkoCCA,
            "span": linear.SCCA_Span, "admm": linear.SCCA_ADMM}[kind]


def _inputs(case):
    kind, args = META["datasets"][case["dataset"]]
    views = conftest_views(args["name"]) if kind == "conftest" else joint_data(**args)
    return [v.astype(np.float32) for v in views] if case["dtype"] == "f32" else views


def _golden(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return ws, [int(x) for x in NPZ[f"{name}/iters"]], NPZ[f"{name}/restated_w"]


def _restate(est, views, kind, **kw):
    """cov_als_fit on the Gram matrix of the covariance the estimator computed on the device."""
    C, dims, n = est._fit_device(views)
    G = C.to(torch.float64).cpu().numpy() * (n - 1)
    return S.cov_als_fit(G, dims, n, kind, est.latent_dimensions, params=est._view_params(dims), mu=float(est._mu),
                         max_iter=est.max_iter, tol=est.tol, random_state=est.random_state, **kw)


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["dtype"] == "f64"))
def test_sparse_matches_reference_golden(name):
    case = CASES[name]
    ref_w, ref_iters, _ = _golden(name)
    est = _cls(case["model"])(**case["kwargs"]).fit(_inputs(case))
    for w, r in zip(est.weights_, ref_w):
        assert w.dtype == np.float64 and w.shape == r.shape
        err = float(np.abs(w - r).max())
        assert err < 1e-9, f"weights differ from the reference by {err:.2e}"
    assert est._fit_info["iters"] == ref_iters


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["dtype"] == "f32"))
def test_sparse_float32_inputs(name):
    case = CASES[name]
    _, _, restated = _golden(name)
    est = _cls(case["model"])(**case["kwargs"]).fit(_inputs(case))
    W = np.vstack(est.weights_)
    assert W.dtype == np.float64
    assert float(np.abs(W - restated).max()) < 1e-3
    if case["model"] in ("pmd", "span"):
        # the support is the same wherever the threshold margin is large
        big = np.abs(restated) > 1e-2
        assert np.all(np.abs(W[big]) > 0.0)
        assert np.all(W[restated == 0.0] == 0.0)


@pytest.mark.parametrize("kind", KINDS)
def test_sparse_larger_problem_matches_restatement(kind):
    views = joint_data(n_views=3, n_samples=20000, n_features=[512, 384, 256], latent_dimensions=4,
                       signal_to_noise=0.3, random_state=7)
    kw = {"pmd": {"tau": 0.3}, "parkhomenko": {"tau": 2.0}, "span": {"span": 40}, "admm": {"tau": 0.1}}.get(kind, {})
    est = _cls(kind)(latent_dimensions=4, random_state=3, max_iter=200, **kw)
    W_ref, iters_ref, deltas = _restate(est, views, kind, return_info=True)
    est.fit(views)
    margin = min(abs(x - est.tol) for dl in deltas for x in dl)
    if margin > 1e-3 * est.tol:
        assert est._fit_info["iters"] == iters_ref
    for w, r in zip(est.weights_, W_ref):
        err = float(np.abs(w - r).max())
        assert err < 1e-9, f"{kind}: weights differ from the restatement by {err:.2e}"


def test_sparse_beyond_l2():
    """D = 4096: the Gram matrix (128 MB) does not fit in L2; fixed 50 sweeps."""
    views = joint_data(n_views=2, n_samples=6000, n_features=[2048, 2048], latent_dimensions=2,
                       signal_to_noise=0.2, random_state=11)
    est = _cls("pmd")(latent_dimensions=2, tau=0.3, tol=0.0, max_iter=50, random_state=0)
    W_ref, iters_ref = _restate(est, views, "pmd")
    est.fit(views)
    assert est._fit_info["iters"] == iters_ref == [50, 50]
    for w, r in zip(est.weights_, W_ref):
        assert float(np.abs(w - r).max()) < 1e-9


@pytest.mark.parametrize("kind", KINDS)
def test_sparse_reruns_bit_identical_and_partial_fit(kind):
    views = conftest_views("three_views")
    kw = dict(latent_dimensions=3, max_iter=300, random_state=1)
    a = _cls(kind)(**kw).fit(views)
    b = _cls(kind)(**kw).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        assert np.array_equal(x, y)
    p = _cls(kind)(**kw)
    for rows in (slice(0, 17), slice(17, 35), slice(35, 50)):
        p.partial_fit([v[rows] for v in views], solve=rows.stop == 50)
    for x, y in zip(a.weights_, p.weights_):
        assert float(np.abs(x - y).max()) < 1e-10


def test_sparse_one_library_call_per_fit(monkeypatch):
    from cca_zoo_b200 import _lib, ops

    lib = _lib.load()
    real = lib.ccab_als_fit
    calls = {"lib": 0, "ops": 0}

    def counted(*args):
        calls["lib"] += 1
        return real(*args)

    real_ops = ops.als_fit

    def counted_ops(*args, **kw):
        calls["ops"] += 1
        return real_ops(*args, **kw)

    monkeypatch.setattr(lib, "ccab_als_fit", counted)
    monkeypatch.setattr(ops, "als_fit", counted_ops)
    views = conftest_views("three_views")
    real_cpu, copies = torch.Tensor.cpu, []

    def counted_cpu(self, *a, **k):
        copies.append(tuple(self.shape))
        return real_cpu(self, *a, **k)

    C, dims, n = _cls("pmd")(latent_dimensions=3)._fit_device(views)
    init = np.zeros((3, sum(dims)))
    init[:, 0] = init[:, 10] = init[:, 18] = 1.0
    monkeypatch.setattr(torch.Tensor, "cpu", counted_cpu)
    W, iters = real_ops(C, dims, n, "pmd", [0.5, 0.5, 0.5], init, 100, 1e-6)
    monkeypatch.setattr(torch.Tensor, "cpu", real_cpu)
    assert calls["lib"] == 1 and len(copies) == 1 and W.shape == (24, 3)
    calls["lib"] = 0
    _cls("span")(latent_dimensions=3, span=3, random_state=0).fit(views)
    assert calls == {"lib": 1, "ops": 1}


def test_sparse_reference_sparsity_assertions():
    """cca_zoo tests/linear/test_iterative.py:179-219 on the same fixtures."""
    two = conftest_views("two_views")
    m = _cls("pmd")(latent_dimensions=1, tau=0.3, max_iter=200, random_state=0).fit(two)
    for w in m.weights:
        assert np.sum(np.abs(w) < 1e-10) > 0
    m = _cls("parkhomenko")(latent_dimensions=1, tau=0.5, max_iter=200, random_state=0).fit(two)
    for w in m.weights:
        assert np.sum(np.abs(w) < 1e-10) > 0
    span = two[0].shape[1] // 2
    m = _cls("span")(latent_dimensions=1, span=span, max_iter=200, random_state=0).fit(two)
    assert np.sum(np.abs(m.weights[0][:, 0]) > 1e-10) <= span
    m = _cls("admm")(latent_dimensions=1, tau=0.5, max_iter=200, random_state=0).fit(two)
    for w in m.weights:
        assert w.shape[0] > 0
    s = m.score(two)
    assert s.shape == (1,) and np.all(np.abs(s) <= 1.0 + 1e-9)


def test_sparse_argument_errors():
    from cca_zoo_b200 import ops

    views = conftest_views("two_views")
    C, dims, n = _cls("span")(latent_dimensions=1)._fit_device(views)
    init = np.ones((1, sum(dims))) / 3.0
    with pytest.raises(ValueError, match="span"):
        ops.als_fit(C, dims, n, "span", [0, 3], init, 10, 1e-6)
    with pytest.raises(ValueError, match="negative"):
        ops.als_fit(C, dims, n, "pmd", [-0.5, 0.5], init, 10, 1e-6)
