"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.pairwise_kernel`` and
``column_sums``, the companion of tests/fake_ops.py for ``cca_zoo_b200.nonparametric._kcca``.  The kernel matrices
come from sklearn's pairwise_kernels (the reference's own call), with the binding's contract: float64 output, sklearn's
ValueError on negative chi2 input, an unknown metric refused.  Nothing in the package imports this module;
``install(monkeypatch)`` swaps it in for one test (after ``fake_ops.install``).  ``CALLS`` counts the kernel calls and
the eigensolves."""
from __future__ import annotations

import torch
from sklearn.metrics import pairwise_kernels

from cca_zoo_b200.ops import KCCA_MAX_ORDER, KCCA_MAX_SAMPLES, KCCA_MAX_VIEWS  # noqa: F401
from tests import fake_ops

CALLS = {"kernel": 0, "syevj": 0}
_SYEVJ = fake_ops.syevj
_METRICS = ("linear", "poly", "polynomial", "rbf", "sigmoid", "cosine", "laplacian", "chi2", "additive_chi2")


def pairwise_kernel(X, Y=None, metric="linear", gamma=1.0, degree=1.0, coef0=1.0):
    if metric not in _METRICS:
        raise ValueError(f"unknown kernel {metric!r}")
    CALLS["kernel"] += 1
    x = X.to(torch.float64).numpy()
    y = None if Y is None else Y.to(torch.float64).numpy()
    K = pairwise_kernels(x, Y=y, metric=metric, gamma=gamma, degree=degree, coef0=coef0, filter_params=True)
    return torch.from_numpy(K)


def column_sums(view):
    return view.to(torch.float64).sum(dim=0)


def syevj(A, shift=0.0, return_info=False):
    CALLS["syevj"] += 1
    out = _SYEVJ(A, shift=shift, return_info=return_info)
    if return_info:
        out[2]["converged"] = True
    return out


def install(monkeypatch):
    """Route KCCA's library calls through this module (and tests/fake_ops.py) for one test."""
    import sys

    from cca_zoo_b200.nonparametric import _kcca

    me = sys.modules[__name__]
    for name in ("pairwise_kernel", "column_sums", "syevj", "KCCA_MAX_VIEWS", "KCCA_MAX_SAMPLES", "KCCA_MAX_ORDER"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    monkeypatch.setattr(_kcca, "ops", fake_ops)
    CALLS.update(kernel=0, syevj=0)
