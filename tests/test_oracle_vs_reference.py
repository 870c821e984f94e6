"""Pin the oracle against the reference's recorded outputs (tests/golden/reference_live.npz, made by
oracle/make_golden_live.py from the unmodified reference).

This is the evidence behind the "parity pinned" line in oracle/restatement.py: each ref_* / cov_* function against
the reference estimator it restates, on the reference's own conftest fixtures, plus the data generator and the
fixture recipe.
"""
import os

import numpy as np
import pytest

from oracle import make_golden_live as L
from oracle import restatement as R

from cca_zoo_b200.datasets import conftest_views, joint_data

_G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_live.npz"))


def _ref(*parts):
    """Recorded weights_ / means_ of one reference fit."""
    k = L.key(*parts)
    ws, mus, i = [], [], 0
    while f"{k}/w{i}" in _G:
        ws.append(_G[f"{k}/w{i}"])
        i += 1
    i = 0
    while f"{k}/mean{i}" in _G:
        mus.append(_G[f"{k}/mean{i}"])
        i += 1
    assert ws, k
    return ws, mus


def _C(views, center=True):
    M, s, n = R.moments(views)
    return R.covariance_from_moments(M, s, n, center), n


@pytest.mark.parametrize("c", [0.0, 0.1, [0.2, 0.7], 1.0])
@pytest.mark.parametrize("ds", ["two_views", "correlated_views"])
def test_rcca(ds, c):
    v = conftest_views(ds)
    ref_w, _ = _ref("rcca", ds, c)
    w, mu = R.ref_rcca_fit(v, 3, c)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-12
    C, n = _C(v)
    w, _ = R.cov_rcca_fit(C, [10, 8], 3, c, n)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-9
    np.testing.assert_allclose(R.score(v, mu, w), _G[L.key("rcca", ds, c, "score")], rtol=1e-9)


@pytest.mark.parametrize("c,pca", [(0.0, True), (0.0, False), (0.3, False), ([0.1, 0.2, 0.3], True)])
def test_mcca(c, pca):
    v = conftest_views("three_views")
    ref_w, _ = _ref("mcca", c, pca)
    w, _ = R.ref_mcca_fit(v, 3, c)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-10
    C, n = _C(v)
    w, _ = R.cov_mcca_fit(C, [10, 8, 6], 3, c)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-10


@pytest.mark.parametrize("c,mu", [(0.0, None), (0.2, [1.0, 1.0, 2.0])])
def test_gcca(c, mu):
    v = conftest_views("three_views")
    ref_w, _ = _ref("gcca", c, mu)
    w, _ = R.ref_gcca_fit(v, 3, c, mu)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-10
    C, n = _C(v)
    w, _ = R.cov_gcca_fit(C, [10, 8, 6], n, 3, c, mu)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-9


def test_joint_data_generator_matches_reference():
    out = joint_data(**L.JOINT_ARGS)
    assert len(out) == L.JOINT_ARGS["n_views"]
    for i, a in enumerate(out):
        assert np.array_equal(a, _G[L.key("joint_data", i)])


def test_conftest_fixture_recipe_matches_reference_file():
    """The fixture recipe in cca_zoo_b200.datasets must be the one in the reference's tests/conftest.py."""
    for name in L.FIXTURES:
        views = conftest_views(name)
        assert L.key("fixture", name, len(views)) not in _G
        for i, a in enumerate(views):
            assert np.array_equal(a, _G[L.key("fixture", name, i)])


@pytest.mark.parametrize("c,center,nv", [(0.0, True, 2), (0.2, True, 3), ([0.1, 0.3], False, 2)])
def test_partialcca(c, center, nv):
    v = conftest_views("three_views")[:nv]
    Z = L.partial_confounds(v)
    ref_w, _ = _ref("partial", c, center, nv)
    ref_betas = [_G[L.key("partial", c, center, nv, f"beta{i}")] for i in range(nv)]
    w, _, betas = R.ref_partialcca_fit(v, Z, 2, c, center=center)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-12
    M, s, n = R.moments(v + [Z])
    w, betas = R.cov_partialcca(M, s, n, [x.shape[1] for x in v], 3, 2, c, center=center)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-9
    for a, b in zip(betas, ref_betas):
        np.testing.assert_allclose(a, b, atol=1e-12)


@pytest.mark.parametrize("c,mu,nv", [(0.0, 0.0, 2), (0.5, 0.0, 2), ([0.3, 0.6, 0.0], [0.5, 2.0, 1.0], 3)])
def test_grcca(c, mu, nv):
    v = conftest_views("three_views")[:nv]
    gs = L.grcca_groups(v)
    ref_w, _ = _ref("grcca", c, mu, nv)
    w, _ = R.ref_grcca_fit(v, gs, 2, c, mu)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-10
    C, n = _C(v)
    w = R.cov_grcca(C, [x.shape[1] for x in v], gs, 2, c, mu)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-9


@pytest.mark.parametrize("model", ["MCCA", "MCCA_pca", "GCCA", "GCCA_w"])
def test_center_false_semantics(model):
    """np.cov centres inside MCCA / GCCA even when ``center=False``; GCCA mixes in raw second moments."""
    v = [x + 1.3 for x in conftest_views("three_views")]
    ref_w, ref_mu = _ref("center", model)
    M, s, n = R.moments(v)
    C, Cu = R.covariance_from_moments(M, s, n, True), R.covariance_from_moments(M, s, n, False)
    dims = [10, 8, 6]
    if model.startswith("MCCA"):
        w, _ = R.ref_mcca_fit(v, 3, 0.1, center=False)
        wc, _ = R.cov_mcca_fit(C, dims, 3, 0.1)
    else:
        vw = [1.0, 2.0, 0.5] if model.endswith("w") else None
        w, _ = R.ref_gcca_fit(v, 3, 0.1, vw, center=False)
        wc, _ = R.cov_gcca_fit(C, dims, n, 3, 0.1, vw, second_moment=Cu)
    assert R.max_rel_err_per_vector(w, ref_w) < 1e-9
    assert R.max_rel_err_per_vector(wc, ref_w) < 1e-8
    assert all(np.all(np.asarray(m) == 0) for m in ref_mu)


def test_ridge_keeps_the_null_directions_of_a_rank_deficient_view():
    v = conftest_views("two_views")
    v = [v[0], np.hstack([v[1], v[1][:, :1]])]          # 9 columns of rank 8
    ref_w, _ = _ref("ridge_rank_deficient")
    assert ref_w[0].shape == (10, 9)                    # nothing dropped: (1-c) lam + c >= c
    C, n = _C(v)
    w, sv = R.cov_rcca_fit(C, [10, 9], 9, 0.2, n)
    assert w[0].shape == (10, 9) and sv[-1] < 1e-7     # the 9th singular value is the null direction
    assert R.max_rel_err_per_vector([x[:, :8] for x in w], [x[:, :8] for x in ref_w]) < 1e-9
