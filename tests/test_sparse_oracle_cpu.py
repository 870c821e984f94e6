"""The Gram-space restatement of the sparse / ALS estimators (oracle/sparse.py:cov_als_fit), which the CUDA
kernel implements, against the reference's golden vectors (tests/golden/reference_outputs_sparse.npz) including the
sweeps each latent dimension took; the data-space restatement (ref_als_fit) against the live reference when it is
importable."""
import json
import os

import numpy as np
import pytest

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import refshim
from oracle import sparse as S

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_sparse.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_sparse.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def _inputs(case):
    kind, args = META["datasets"][case["dataset"]]
    views = conftest_views(args["name"]) if kind == "conftest" else joint_data(**args)
    return [v.astype(np.float32) for v in views] if case["dtype"] == "f32" else views


def test_sparse_golden_covers_every_model_and_dataset():
    assert {c["model"] for c in CASES.values()} == {"pls", "pmd", "parkhomenko", "span", "admm"}
    assert {c["dataset"] for c in CASES.values()} == {"two_views", "three_views", "joint3_sparse"}
    assert any(c["dtype"] == "f32" for c in CASES.values())


@pytest.mark.parametrize("name", sorted(CASES))
def test_cov_als_fit_matches_golden(name):
    case = CASES[name]
    kw = case["kwargs"]
    views = [v.astype(np.float64) for v in _inputs(case)]
    vs, _ = S.setup_fit(views, kw.get("center", True))
    X = np.hstack(vs)
    dims = [v.shape[1] for v in views]
    W, iters = S.cov_als_fit(X.T @ X, dims, X.shape[0], case["model"], kw["latent_dimensions"], params=case["params"],
                             max_iter=kw["max_iter"], random_state=kw["random_state"])
    assert iters == [int(x) for x in NPZ[f"{name}/iters"]]
    assert float(np.abs(np.vstack(W) - NPZ[f"{name}/restated_w"]).max()) < 1e-10
    if case["dtype"] == "f64":
        for i, w in enumerate(W):
            assert float(np.abs(w - NPZ[f"{name}/w{i}"]).max()) < 1e-10


@pytest.mark.skipif(not refshim.available(), reason="the reference tree is not present")
@pytest.mark.parametrize("kind", ["pls", "pmd", "parkhomenko", "span", "admm"])
def test_ref_als_fit_matches_live_reference(kind):
    refshim.install()
    from cca_zoo import linear as ref

    cls = {"pls": ref.PLS_ALS, "pmd": ref.SCCA_PMD, "parkhomenko": ref.ParkhomenkoCCA, "span": ref.SCCA_Span,
           "admm": ref.SCCA_ADMM}[kind]
    kw = {"pmd": {"tau": 0.4}, "parkhomenko": {"tau": 0.5}, "span": {"span": 4}, "admm": {"tau": 0.1}}.get(kind, {})
    views = conftest_views("three_views")
    for center in (True, False):
        est = cls(latent_dimensions=2, center=center, max_iter=100, random_state=5, **kw).fit(views)
        params = S.als_params(kind, [v.shape[1] for v in views], tau=kw.get("tau"), span=kw.get("span"))
        W, _ = S.ref_als_fit(views, kind, 2, params=params, max_iter=100, random_state=5, center=center)
        for w, r in zip(W, est.weights_):
            assert float(np.abs(w - r).max()) < 1e-12
