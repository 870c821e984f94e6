"""GPU parity of the Eckart-Young gradient estimators (CCA_EY, PLS_EY, MCCA_EY) against the reference's golden vectors
(tests/golden/reference_outputs_ey.npz, oracle/make_golden_ey.py) and the kernel-form restatements of oracle/ey.py.
Tolerances are relative to max |w|: 1e-9 for float64 inputs; F32_TOL for float32 inputs, whose moments (full batch)
carry float32-grade rounding (tests/test_ey_oracle_cpu.py measures that drift on the CPU)."""
import json
import os

import numpy as np
import pytest
import torch

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import ey as E

pytestmark = pytest.mark.gpu

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_ey.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_ey.npz"))
CASES = {c["name"]: c for c in META["cases"]}
F32_TOL = 1e-3


def _cls(kind):
    from cca_zoo_b200 import linear

    return {"cca": linear.CCA_EY, "pls": linear.PLS_EY, "mcca": linear.MCCA_EY}[kind]


def _inputs(case):
    kind, args = META["datasets"][case["dataset"]]
    if kind == "conftest":
        views = conftest_views(args["name"])
    else:
        views = [(v - v.mean(axis=0)) / v.std(axis=0, ddof=1) for v in joint_data(**args)]
    return [v.astype(np.float32) for v in views] if case["dtype"] == "f32" else views


def _golden(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return ws, int(NPZ[f"{name}/iters"][0]), NPZ[f"{name}/restated_w"]


def _route(kw, n):
    bs = kw.get("batch_size")
    return "covariance" if bs is None or bs >= n else "minibatch"


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["dtype"] == "f64"))
def test_ey_matches_reference_golden(name):
    case = CASES[name]
    ref_w, ref_iters, _ = _golden(name)
    views = _inputs(case)
    est = _cls(case["model"])(**case["kwargs"]).fit(views)
    assert est._fit_info["route"] == _route(case["kwargs"], views[0].shape[0])
    assert est._fit_info["iters"] == ref_iters
    R = np.vstack(ref_w)
    W = np.vstack(est.weights_)
    assert W.dtype == np.float64 and W.shape == R.shape
    if np.isnan(R).all():
        assert np.isnan(W).all()
        return
    err = float(np.abs(W - R).max()) / float(np.abs(R).max())
    assert err < 1e-9, f"weights differ from the reference by {err:.2e} (relative)"
    for mu, i in zip(est.means_, range(len(views))):
        assert np.allclose(mu, NPZ[f"{name}/mean{i}"], rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["dtype"] == "f32"))
def test_ey_float32_inputs(name):
    case = CASES[name]
    _, ref_iters, restated = _golden(name)
    est = _cls(case["model"])(**case["kwargs"]).fit(_inputs(case))
    W = np.vstack(est.weights_)
    assert W.dtype == np.float64
    assert est._fit_info["iters"] == ref_iters
    err = float(np.abs(W - restated).max()) / float(np.abs(restated).max())
    assert err < F32_TOL, f"float32 drift {err:.2e}"


def test_ey_divergent_case_gives_nan_without_raising():
    case = CASES["cca_two_views_diverge"]
    est = _cls("cca")(**case["kwargs"]).fit(_inputs(case))
    assert all(np.isnan(w).all() for w in est.weights_)
    assert est._fit_info["iters"] == case["kwargs"]["max_iter"]


@pytest.mark.parametrize("bs", [None, 64])
@pytest.mark.parametrize("kind", ["cca", "pls", "mcca"])
def test_ey_reruns_bit_identical(kind, bs):
    views = conftest_views("three_correlated_views")
    kw = dict(latent_dimensions=2, max_iter=200, batch_size=bs, learning_rate=2e-3, random_state=3)
    a = _cls(kind)(**kw).fit(views)
    b = _cls(kind)(**kw).fit(views)
    for x, y in zip(a.weights_, b.weights_):
        assert np.isfinite(x).all() and np.array_equal(x, y)


def test_ey_larger_problem_matches_restatement():
    """n = 20000, widths [256, 192]: both routes against the kernel-form restatements."""
    views = [(v - v.mean(axis=0)) / v.std(axis=0, ddof=1) for v in
             joint_data(n_views=2, n_samples=20000, n_features=[256, 192], latent_dimensions=4, signal_to_noise=0.5,
                        random_state=9)]
    kw = dict(latent_dimensions=8, c=0.1, learning_rate=1e-3, max_iter=60, tol=0.0, random_state=2)
    for bs in (None, 512):
        est = _cls("cca")(batch_size=bs, **kw).fit(views)
        if bs is None:
            W, it, _ = E.cov_ey_fit(views, "cca", 8, c=0.1, learning_rate=1e-3, max_iter=60, tol=0.0, random_state=2)
        else:
            W, it, _ = E.mb_ey_fit(views, "cca", 8, bs, c=0.1, learning_rate=1e-3, max_iter=60, tol=0.0,
                                   random_state=2)
        R = np.vstack(W)
        assert est._fit_info["iters"] == it == 60
        err = float(np.abs(np.vstack(est.weights_) - R).max()) / float(np.abs(R).max())
        assert err < 1e-9, f"batch {bs}: {err:.2e}"


def test_ey_one_library_call_per_chunk(monkeypatch):
    from cca_zoo_b200 import _lib
    from cca_zoo_b200.linear import _gradient

    lib = _lib.load()
    real = lib.ccab_ey_fit
    calls = {"lib": 0}

    def counted(*args):
        calls["lib"] += 1
        return real(*args)

    monkeypatch.setattr(lib, "ccab_ey_fit", counted)
    views = conftest_views("correlated_views")
    est = _cls("cca")(latent_dimensions=2, max_iter=300, tol=0.0, random_state=0).fit(views)
    assert calls["lib"] == 1 and est._fit_info["calls"] == 1
    calls["lib"] = 0
    monkeypatch.setattr(_gradient, "_CHUNK_INDEX_BYTES", 4 * 16 * 40)       # 40 steps of 16 rows per chunk
    est = _cls("pls")(latent_dimensions=2, max_iter=300, batch_size=16, tol=0.0, random_state=0).fit(views)
    assert calls["lib"] == est._fit_info["calls"] == 8
    assert est._fit_info["iters"] == 300


def test_ey_cuda_and_host_inputs_agree():
    views = conftest_views("three_correlated_views")
    for bs in (None, 32):
        kw = dict(latent_dimensions=2, max_iter=100, batch_size=bs, learning_rate=2e-3, random_state=4)
        a = _cls("mcca")(**kw).fit(views)
        b = _cls("mcca")(**kw).fit([torch.from_numpy(v).cuda() for v in views])
        for x, y in zip(a.weights_, b.weights_):
            assert np.isfinite(x).all() and np.array_equal(x, y)


@pytest.mark.parametrize("kind,bs", [("cca", 16), ("mcca", 32)])
def test_ey_initial_projections_orthonormal(kind, bs):
    """cca_zoo tests/linear/test_gradient.py:418-468: max_iter=0 returns the initial weights."""
    views = conftest_views("two_views" if kind == "cca" else "three_correlated_views")
    est = _cls(kind)(latent_dimensions=2, batch_size=bs, max_iter=0, random_state=0, center=False).fit(views)
    idx = np.random.default_rng(0).choice(views[0].shape[0], bs, replace=False)
    for v, w in zip(views, est.weights_):
        z = v[idx] @ w
        np.testing.assert_allclose(z.T @ z, np.eye(2), atol=1e-8)


def test_ey_converged_scores_match_exact_models():
    """cca_zoo tests/linear/test_gradient.py:337-382."""
    from cca_zoo_b200 import linear

    cv = conftest_views("correlated_views")
    s_ref = linear.CCA(latent_dimensions=2).fit(cv).score(cv)
    s = _cls("cca")(latent_dimensions=2, max_iter=1000, random_state=0).fit(cv).score(cv)
    np.testing.assert_allclose(sorted(s, reverse=True), sorted(s_ref, reverse=True), atol=0.05)
    s_ref = linear.PLS(latent_dimensions=2).fit(cv).score(cv)
    s = _cls("pls")(latent_dimensions=2, max_iter=1000, random_state=0).fit(cv).score(cv)
    np.testing.assert_allclose(sorted(s, reverse=True), sorted(s_ref, reverse=True), atol=0.05)
    tv = conftest_views("three_correlated_views")
    s_ref = linear.MCCA(latent_dimensions=2).fit(tv).score(tv)
    s = _cls("mcca")(latent_dimensions=2, max_iter=1000, random_state=0).fit(tv).score(tv)
    np.testing.assert_allclose(sorted(s, reverse=True), sorted(s_ref, reverse=True), atol=0.05)


def test_ey_partial_fit_and_sharded_fit_raise(monkeypatch):
    from cca_zoo_b200 import parallel

    views = conftest_views("two_views")
    with pytest.raises(NotImplementedError):
        _cls("cca")().partial_fit(views)
    monkeypatch.setattr(parallel, "is_distributed", lambda group=None: True)
    with pytest.raises(NotImplementedError):
        _cls("pls")().fit(views)


def test_ey_unsupported_shapes_raise_value_error():
    views = [np.random.default_rng(0).standard_normal((200, 40)) for _ in range(2)]
    with pytest.raises(ValueError):
        _cls("pls")(latent_dimensions=33, max_iter=2).fit(views)
    with pytest.raises(ValueError):
        _cls("cca")(latent_dimensions=5).fit([views[0], views[1][:, :3]])
