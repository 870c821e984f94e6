"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.row_norm4_sum`` / ``ccar3_admm``, the
companion of tests/fake_ops.py for ``cca_zoo_b200.linear._ccar3``.  It runs the float64 restatement of
oracle/ccar3.py with the binding's contract.  Nothing in the package imports this module; ``install(monkeypatch)``
swaps it in for one test (after ``fake_ops.install``).  ``CALLS`` counts the calls."""
from __future__ import annotations

import numpy as np
import torch

from cca_zoo_b200.ops import CCAR3_MAX_P, CCAR3_MAX_Q
from tests import fake_ops

CALLS = {"norm4": 0, "admm": 0}


def row_norm4_sum(Y, mean):
    CALLS["norm4"] += 1
    d = Y.to(torch.float64) - mean.to(torch.float64)
    return ((d * d).sum(dim=1) ** 2).sum().reshape(1)


def ccar3_admm(M, B0, kappa, rho, tol, max_iter):
    from oracle import ccar3 as O

    CALLS["admm"] += 1
    p, q = B0.shape
    if not (1 <= p <= CCAR3_MAX_P and 1 <= q <= CCAR3_MAX_Q):
        raise ValueError("ccar3_admm: problem out of range")
    Z, U, it, primal, dual, stopped = O.admm_inverse(M.numpy(), B0.numpy(), kappa, rho, tol, max_iter)
    info = np.array([it, primal, dual, float(stopped)])
    return torch.from_numpy(Z), torch.from_numpy(U), torch.from_numpy(info)


def install(monkeypatch):
    """Route CCAR3's library calls through this module (and tests/fake_ops.py) for one test."""
    import sys

    from cca_zoo_b200.linear import _ccar3

    me = sys.modules[__name__]
    for name in ("row_norm4_sum", "ccar3_admm", "CCAR3_MAX_P", "CCAR3_MAX_Q"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    monkeypatch.setattr(_ccar3, "ops", fake_ops)
    CALLS.update(norm4=0, admm=0)
