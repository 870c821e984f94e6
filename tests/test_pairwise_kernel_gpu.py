"""ccab_pairwise_kernel against sklearn.metrics.pairwise_kernels in float64, every metric, X is Y and X != Y, at
shapes that hit every tile edge (64-row tiles, 16-feature chunks), column-slice views whose leading dimension exceeds
d, and float32 input.  The exact-sum metrics agree to 1e-13 of max|K|; rbf to its cancellation bound
gamma eps (|x|^2 + |y|^2).  Also: the rbf diagonal is exactly 1 when X is Y, zero rows give zeros for cosine, sklearn's
ValueError on negative chi2 input, and reruns are bit-identical."""
import numpy as np
import pytest
import torch
from sklearn.metrics import pairwise_kernels

from cca_zoo_b200 import ops

pytestmark = pytest.mark.gpu

METRICS = ["linear", "poly", "polynomial", "rbf", "sigmoid", "cosine", "laplacian", "chi2", "additive_chi2"]
PARAMS = dict(gamma=0.3, degree=2.5, coef0=1.5)
EPS = np.finfo(np.float64).eps


def _data(n, d, seed, nonneg):
    x = np.random.default_rng(seed).standard_normal((n, d)) * 0.5
    return np.abs(x) + 0.1 if nonneg else x


def _params(metric, d):
    gamma = PARAMS["gamma"] / d if metric not in ("linear", "cosine", "additive_chi2") else 1.0
    return dict(gamma=gamma, degree=PARAMS["degree"], coef0=PARAMS["coef0"])


def _check(metric, x, y, K, p):
    want = pairwise_kernels(x, Y=y, metric=metric, filter_params=True, **p)
    scale = max(float(np.abs(want).max()), 1e-300)
    err = np.abs(K - want)
    if metric == "rbf":
        yy = x if y is None else y
        bound = p["gamma"] * EPS * ((x * x).sum(1)[:, None] + (yy * yy).sum(1)[None, :]) * 16 + 1e-13 * scale
        assert (err <= bound).all(), float((err / bound).max())
    else:
        assert err.max() <= 1e-13 * scale, float(err.max() / scale)


@pytest.mark.parametrize("metric", METRICS)
@pytest.mark.parametrize("nx,ny", [(1, 1), (63, 65), (64, 64), (65, 1000), (1000, 63)])
@pytest.mark.parametrize("d", [1, 257])
def test_pairwise_kernel_matches_sklearn(metric, nx, ny, d):
    nonneg = "chi2" in metric
    x, y = _data(nx, d, 0, nonneg), _data(ny, d, 1, nonneg)
    p = _params(metric, d)
    X, Y = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    _check(metric, x, y, ops.pairwise_kernel(X, Y, metric, **p).cpu().numpy(), p)
    _check(metric, x, None, ops.pairwise_kernel(X, None, metric, **p).cpu().numpy(), p)


@pytest.mark.parametrize("metric", METRICS)
def test_pairwise_kernel_strided_and_float32(metric):
    nonneg = "chi2" in metric
    base = _data(130, 300, 2, nonneg)
    p = _params(metric, 257)
    B = torch.from_numpy(base).cuda()
    X, Y = B[:65, 3:260], B[65:, 40:297]                      # leading dimension 300 > d = 257
    assert X.stride(0) == 300
    _check(metric, base[:65, 3:260], base[65:, 40:297], ops.pairwise_kernel(X, Y, metric, **p).cpu().numpy(), p)
    x32 = base[:, :257].astype(np.float32)
    K = ops.pairwise_kernel(torch.from_numpy(x32).cuda(), None, metric, **p)
    _check(metric, x32.astype(np.float64), None, K.cpu().numpy(), p)


def test_rbf_diagonal_cosine_zero_rows_and_bitwise_reruns():
    x = _data(200, 33, 3, False)
    x[7] = 0.0
    X = torch.from_numpy(x).cuda()
    K = ops.pairwise_kernel(X, None, "rbf", gamma=0.7)
    assert (torch.diagonal(K) == 1.0).all()
    C = ops.pairwise_kernel(X, None, "cosine")
    assert (C[7] == 0).all() and (C[:, 7] == 0).all()
    for metric in METRICS:
        xx = np.abs(x) if "chi2" in metric else x
        T = torch.from_numpy(xx).cuda()
        a = ops.pairwise_kernel(T, None, metric, **_params(metric, 33))
        b = ops.pairwise_kernel(T, None, metric, **_params(metric, 33))
        assert torch.equal(a, b)


def test_chi2_rejects_negative_input():
    X = torch.from_numpy(_data(10, 4, 4, False)).cuda()
    for metric in ("chi2", "additive_chi2"):
        with pytest.raises(ValueError, match="negative"):
            ops.pairwise_kernel(X, None, metric)
    with pytest.raises(ValueError, match="unknown kernel"):
        ops.pairwise_kernel(X, None, "precomputed")
