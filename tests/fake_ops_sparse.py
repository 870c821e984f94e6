"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.als_fit`` (the sparse / ALS estimators),
the companion of tests/fake_ops.py for ``cca_zoo_b200.linear._iterative``.  It runs the Gram-space restatement
(oracle/sparse.py:cov_als_fit) with the same contract as the kernel binding: ``(n_total - 1) cov`` is the Gram matrix,
``init`` holds the k x D initial weights, the result is (W as D x k float64 numpy, sweeps per dimension).  Nothing in
the package imports this module; ``install(monkeypatch)`` swaps it in for one test (after ``fake_ops.install``)."""
from __future__ import annotations

import numpy as np
import torch


def als_fit(cov, dims, n_total, kind, params, init, max_iter, tol, mu=1.0):
    from oracle import sparse as S

    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    init = np.asarray(init, dtype=np.float64)
    starts = [[init[d, off[i]:off[i + 1]] for i in range(len(dims))] for d in range(init.shape[0])]
    G = cov.to(torch.float64).numpy() * (n_total - 1)
    W, iters = S.cov_als_fit(G, dims, n_total, kind, init.shape[0], params=list(params), mu=mu, init=starts,
                             max_iter=max_iter, tol=tol)
    return np.vstack(W), iters


def install(monkeypatch):
    """Route the sparse / ALS estimators' library call through this module for the duration of one test."""
    import sys

    from cca_zoo_b200.linear import _iterative

    monkeypatch.setattr(_iterative, "ops", sys.modules[__name__])
