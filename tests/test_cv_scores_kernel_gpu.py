"""ccab_cv_scores (the held-out scoring of GridSearchCV's moment route) against its float64 torch restatement
(tests/fake_ops_cv.py): view counts 2, 3 and 5 with ragged widths (1, and widths that cross the 64-row tiles of the
GEMM), G k_max crossing the 64-column tiles, candidates narrower than k_max, a zero-variance variate, n = 2, two calls
bit for bit, and the argument errors raised before any launch."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from cca_zoo_b200 import _lib, ops

from . import fake_ops_cv

pytestmark = pytest.mark.gpu

CASES = [
    # (dims, G, k_of, n)
    ([1, 7], 3, [1, 1, 1], 50),
    ([10, 8], 5, [2, 1, 2, 2, 1], 120),
    ([65, 1, 130], 9, [3, 1, 2, 3, 3, 1, 2, 3, 3], 400),
    ([3, 64, 5, 129, 2], 20, [4] * 10 + [1, 2, 3, 4] * 2 + [2, 2], 1000),
    ([33, 31], 40, [2] * 40, 2),
]


def _problem(dims, G, k_of, n, seed=0, zero_variate=False):
    rng = np.random.default_rng(seed)
    D, k_max = sum(dims), max(k_of)
    X = rng.standard_normal((max(n, D + 3), D)) @ rng.standard_normal((D, D)) / np.sqrt(D)
    C = np.cov(X[:max(n, 2)].T) if n > 2 else np.cov(X[:2].T)
    W = np.zeros((D, G * k_max))
    for b, k in enumerate(k_of):
        W[:, b * k_max:b * k_max + k] = rng.standard_normal((D, k))
    if zero_variate:
        W[: dims[0], 0] = 0.0                     # view 0's first variate of candidate 0 has zero variance
    return torch.from_numpy(np.ascontiguousarray(C)).cuda(), torch.from_numpy(W).cuda()


@pytest.mark.parametrize("case", range(len(CASES)))
def test_matches_restatement(case):
    dims, G, k_of, n = CASES[case]
    C, W = _problem(dims, G, k_of, n, seed=case)
    corr, score = ops.cv_scores(C, dims, n, W, k_of)
    rc, rs = fake_ops_cv.cv_scores(C, dims, n, W, k_of)
    torch.testing.assert_close(corr, rc, rtol=1e-11, atol=1e-12)
    torch.testing.assert_close(score, rs, rtol=1e-11, atol=1e-12)
    k_max = max(k_of)
    for b, k in enumerate(k_of):
        assert bool((corr[b, k:] == 0).all())
    assert corr.shape == (G, k_max)


def test_zero_variance_guard():
    dims, k_of = [6, 5, 4], [2, 2]
    C, W = _problem(dims, 2, k_of, 80, zero_variate=True)
    corr, score = ops.cv_scores(C, dims, 80, W, k_of)
    rc, rs = fake_ops_cv.cv_scores(C, dims, 80, W, k_of)
    assert torch.isfinite(corr).all()
    torch.testing.assert_close(corr, rc, rtol=1e-11, atol=1e-12)
    torch.testing.assert_close(score, rs, rtol=1e-11, atol=1e-12)


def test_repeated_calls_are_bit_identical():
    dims, G, k_of, n = CASES[3]
    C, W = _problem(dims, G, k_of, n, seed=7)
    a = ops.cv_scores(C, dims, n, W, k_of)
    b = ops.cv_scores(C, dims, n, W, k_of)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_argument_errors_raise_before_any_launch():
    dims, k_of = [4, 3], [2, 1]
    C, W = _problem(dims, 2, k_of, 30)
    lib = _lib.load()
    before = lib.ccab_launch_count()
    bad = [
        lambda: ops.cv_scores(C[:4, :4], [4], 30, W[:4], k_of),                 # one view
        lambda: ops.cv_scores(C, [1] * 9, 30, W, k_of),                         # more than MAX_VIEWS
        lambda: ops.cv_scores(C, dims, 30, W, [3, 1]),                          # k_of > k_max
        lambda: ops.cv_scores(C, dims, 30, W, [0, 1]),
        lambda: ops.cv_scores(C, [4, 4], 30, W, k_of),                          # sizes disagree
        lambda: ops.cv_scores(C, dims, 1, W, k_of),                             # n < 2
        lambda: ops.cv_scores(C.float(), dims, 30, W, k_of),
        lambda: ops.cv_scores(C, dims, 30, W[:, :3], k_of),                     # G k_max columns
    ]
    for f in bad:
        with pytest.raises(ValueError):
            f()
    d = _lib.i64_array(dims)
    kk = torch.tensor(k_of, dtype=torch.int32, device="cuda")
    out = torch.empty(8, dtype=torch.float64, device="cuda")
    ws = torch.empty(16, dtype=torch.uint8, device="cuda")                       # far too small
    rc = lib.ccab_cv_scores(2, d, C.data_ptr(), 7, 30.0, W.data_ptr(), 4, 2, 2, kk.data_ptr(), out.data_ptr(),
                            out.data_ptr(), ws.data_ptr(), ws.numel(), None)
    assert rc < 0 and "workspace" in _lib.last_error()
    assert lib.ccab_cv_scores_workspace_bytes(1, d, 2, 2) == 0
    assert lib.ccab_launch_count() == before
