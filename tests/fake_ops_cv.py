"""TEST INFRASTRUCTURE ONLY: a float64 torch restatement of ``ops.cv_scores`` (the held-out scoring of GridSearchCV's
moment route), used as the CPU stand-in of the kernel and as the reference the kernel test compares against."""
from __future__ import annotations

import numpy as np
import torch

from .fake_ops import covariance  # noqa: F401  (the test covariance of a split, as ops.covariance)


def cv_scores(C, dims, n, W, k_of):
    dims = [int(p) for p in dims]
    m, G = len(dims), len(k_of)
    if not 2 <= m <= 8:
        raise ValueError(f"cv_scores takes 2 to 8 views, got {m}")
    k_max = int(W.shape[1]) // G
    if any(not 1 <= int(k) <= k_max for k in k_of):
        raise ValueError(f"every candidate width must lie in 1..{k_max}, got {list(k_of)}")
    if not n >= 2:
        raise ValueError("at least 2 held-out samples are needed")
    C, W = C.to(torch.float64), W.to(torch.float64)
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    blk = [slice(int(off[i]), int(off[i + 1])) for i in range(m)]
    S = torch.stack([torch.stack([(W[blk[i]] * (C[blk[i], blk[l]] @ W[blk[l]])).sum(dim=0) for l in range(m)])
                     for i in range(m)])                                      # m x m x G k_max
    norms = torch.sqrt(torch.stack([S[i, i] for i in range(m)]) * (n - 1))
    den = torch.where(norms > 1e-12, norms, torch.ones_like(norms)) / np.sqrt(n - 1)
    R = S / (den[:, None] * den[None, :])
    corr = ((R.sum(dim=(0, 1)) - sum(R[i, i] for i in range(m))) / (m * (m - 1))).reshape(G, k_max)
    kk = torch.tensor([int(k) for k in k_of], device=corr.device)
    corr = torch.where(torch.arange(k_max, device=corr.device)[None, :] < kk[:, None], corr, torch.zeros_like(corr))
    return corr, corr.sum(dim=1) / kk.to(torch.float64)


def install(monkeypatch):
    """Route the grid search's scoring call through this module for the duration of one test."""
    import sys

    from cca_zoo_b200.model_selection import _search

    monkeypatch.setattr(_search, "ops", sys.modules[__name__])
