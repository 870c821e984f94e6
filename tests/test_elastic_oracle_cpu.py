"""CPU checks of the ElasticCCA / SCCA_IPLS restatements (oracle/elastic.py) against each other and against the
reference's golden vectors (tests/golden/reference_outputs_elastic.npz, oracle/make_golden_elastic.py), and of the
estimators' parameter validation (no GPU needed: it runs before any kernel)."""
import json
import os

import numpy as np
import pytest

from cca_zoo_b200.datasets import conftest_views, joint_data
from oracle import elastic as E
from oracle.restatement import setup_fit

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
with open(os.path.join(_DIR, "reference_outputs_elastic.json")) as _f:
    META = json.load(_f)
NPZ = np.load(os.path.join(_DIR, "reference_outputs_elastic.npz"))
CASES = {c["name"]: c for c in META["cases"]}


def views_of(case):
    kind, args = META["datasets"][case["dataset"]]
    if kind == "joint":
        return joint_data(**args)
    return [v[:args.get("rows")] for v in conftest_views(args["name"])]


def golden(name):
    ws, i = [], 0
    while f"{name}/w{i}" in NPZ:
        ws.append(NPZ[f"{name}/w{i}"])
        i += 1
    return ws


def spread_tol(case, d):
    """max(1e-6, 10 x the reference's tol vs tol/100 spread), the spread taken over every view and every dimension up to
    d: a difference in one dimension reaches the later ones through the deflation."""
    return max(1e-6, 10.0 * max(max(s[:d + 1]) for s in case["spread"]))


def unique_dims(case, views):
    """Per view, the latent dimensions whose sub-problem minimiser is unique: alpha (1 - l1) > 0, or G_ii positive
    definite (only the first dimension: deflation makes G_ii singular)."""
    out = []
    for (a, l1), v in zip(case["params"], views):
        if a * (1.0 - l1) > 0.0:
            out.append(list(range(case["kwargs"]["latent_dimensions"])))
        else:
            out.append([0] if v.shape[0] - 1 > v.shape[1] else [])
    return out


def gram(views, center):
    vs, _ = setup_fit([np.asarray(v, np.float64) for v in views], center)
    X = np.hstack(vs)
    means = None if center else np.hstack([np.asarray(v).mean(axis=0) for v in views])
    return X.T @ X, X.shape[0], means


@pytest.mark.parametrize("name", sorted(CASES))
def test_gram_space_equals_data_space(name):
    case = CASES[name]
    views, kw = views_of(case), case["kwargs"]
    G, n, means = gram(views, kw["center"])
    Wc, ic = E.cov_elastic_fit(G, [v.shape[1] for v in views], n, case["model"], kw["latent_dimensions"],
                               params=case["params"], colmeans=means, max_iter=kw["max_iter"], tol=kw["tol"],
                               random_state=kw["random_state"])
    Wr, ir = E.ref_elastic_fit(views, case["model"], kw["latent_dimensions"], params=case["params"],
                               max_iter=kw["max_iter"], tol=kw["tol"], random_state=kw["random_state"],
                               center=kw["center"])
    stored = np.split(NPZ[f"{name}/restated_w"], np.cumsum([v.shape[1] for v in views])[:-1])
    assert ic == ir == [int(x) for x in NPZ[f"{name}/iters"]]
    for a, b in zip(Wr, stored):
        assert np.array_equal(a, b)                         # the data-space restatement still writes the goldens
    # n <= d_i: the pseudo-inverse of the rank-deficient G_ii loses a digit more to rounding
    tol = 1e-9 if min(v.shape[0] for v in views) <= max(v.shape[1] for v in views) else 1e-10
    for a, b in zip(Wc, Wr):
        assert float(np.abs(a - b).max()) < tol * max(1.0, float(np.abs(b).max()))


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if c["spread"] is not None))
def test_restatement_matches_reference_where_unique(name):
    case = CASES[name]
    views = views_of(case)
    Wr = np.split(NPZ[f"{name}/restated_w"], np.cumsum([v.shape[1] for v in views])[:-1])
    checked = 0
    for i, (w, r, dims) in enumerate(zip(Wr, golden(name), unique_dims(case, views))):
        for d in dims:
            tol = spread_tol(case, d)
            assert float(np.abs(w[:, d] - r[:, d]).max()) <= tol, (i, d)
            checked += 1
    if case["setting"] in ("enet", "ridge", "pv"):
        assert checked == len(views) * case["kwargs"]["latent_dimensions"]


def test_solver_kkt_and_minimum_norm():
    rng = np.random.default_rng(0)
    X = rng.standard_normal((6, 9))                       # n < p: X^T X singular
    y = rng.standard_normal(6)
    G, b, n = X.T @ X, X.T @ y / 6, 6
    for alpha, l1 in ((0.0, 1.0), (0.0, 0.5), (0.3, 0.0), (0.05, 0.5), (0.05, 1.0)):
        w = E.solve_penalised(G, b, n, alpha, l1, rng.standard_normal(9))
        rho = alpha / n if l1 == 0.0 else alpha * (1 - l1)
        assert E.kkt_residual(G / n + rho * np.eye(9), b, alpha * l1, w) <= 1e-12
    w = E.solve_penalised(G, b, n, 0.0, 1.0, np.zeros(9))
    assert np.allclose(w, np.linalg.pinv(X) @ y, atol=1e-12)
    assert np.all(E.solve_penalised(G, b, n, 100.0, 1.0, np.ones(9)) == 0.0)


def test_capped_coordinate_descent_is_reported():
    rng = np.random.default_rng(3)
    z = rng.standard_normal((400, 2))
    views = [z @ rng.standard_normal((2, p)) + 0.03 * rng.standard_normal((400, p)) for p in (30, 20)]
    _, iters = E.ref_elastic_fit(views, "elastic", 1, [(1e-4, 1.0)] * 2, max_iter=2, tol=0.0, random_state=0)
    assert iters == [-2]
    _, iters = E.ref_elastic_fit(views, "elastic", 1, [(1e-1, 0.5)] * 2, max_iter=2, tol=0.0, random_state=0)
    assert iters == [2]


def test_ridge_error_wording():
    from sklearn.linear_model import Ridge
    from sklearn.utils._param_validation import InvalidParameterError

    from cca_zoo_b200.linear import ElasticCCA

    with pytest.raises(InvalidParameterError) as ours:
        ElasticCCA(alpha=-1.0, l1_ratio=0.0)._validate_params()
    with pytest.raises(InvalidParameterError) as theirs:
        Ridge(alpha=-1.0).fit(np.ones((3, 2)), np.ones(3))
    assert str(ours.value) == str(theirs.value)


@pytest.mark.parametrize("cls_name", ["ElasticCCA", "SCCA_IPLS"])
@pytest.mark.parametrize("kw,msg", [({"alpha": -0.1}, "'alpha' parameter"), ({"l1_ratio": 1.5}, "'l1_ratio'"),
                                    ({"alpha": [0.1, -1.0]}, "'alpha' parameter"),
                                    ({"l1_ratio": [0.5, -0.5]}, "'l1_ratio'")])
def test_invalid_regression_parameters(cls_name, kw, msg):
    from sklearn.utils._param_validation import InvalidParameterError

    from cca_zoo_b200 import linear

    est = getattr(linear, cls_name)(**kw)
    with pytest.raises(InvalidParameterError, match=msg):
        est._validate_params()


def test_public_surface():
    from sklearn.base import clone

    from cca_zoo_b200.linear import SCCA_IPLS, ElasticCCA

    assert ElasticCCA().get_params()["l1_ratio"] == 0.5 and ElasticCCA().alpha == 0.0
    assert SCCA_IPLS().get_params()["l1_ratio"] == 1.0 and SCCA_IPLS().alpha == 0.0
    m = clone(ElasticCCA(alpha=[0.1, 0.2], l1_ratio=0.3, latent_dimensions=2, precision="f64"))
    assert m.alpha == [0.1, 0.2] and m.l1_ratio == 0.3 and m.precision == "f64"
