"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.gfa_fit``, the companion of
tests/fake_ops.py for ``cca_zoo_b200.probabilistic._gfa``.  It runs the Gram-form steps of oracle/gfa.py with the same
contract as the binding: a fit handle whose ``run(n)`` does up to n iterations, ``stopped()`` and ``result()`` (the
decoded state).  Nothing in the package imports this module; ``install(monkeypatch)`` swaps it in for one test (after
``fake_ops.install``)."""
from __future__ import annotations

import numpy as np
import torch

from tests import fake_ops

CALLS = {"run": 0}
GFA_MAX_K = 64
GFA_ARD_ALPHA_0 = GFA_TAU_ALPHA_0 = 1e-14


class GfaFit:
    def __init__(self, dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=True):
        from oracle import gfa as O

        if XtZ0.shape[1] > GFA_MAX_K:
            raise ValueError("ccab_gfa_fit supports 1 <= k <= 64")
        self.O = O
        self.G = G.to(torch.float64).numpy()
        self.Xz0 = XtZ0.to(torch.float64).numpy()
        self.tol, self.drop_k = float(tol), bool(drop_k)
        self.st = O.gram_state(n_samples, [int(d) for d in dims], XtZ0.shape[1], z0tz0, datavar, y_const)
        self.st["prunes"] = 0

    def run(self, n_steps):
        CALLS["run"] += 1
        for _ in range(int(n_steps)):
            k = self.st["k"]
            self.O.gram_step(self.st, self.G, self.Xz0, self.tol, self.drop_k)
            self.st["prunes"] += int(self.st["k"] != k)

    def stopped(self):
        return self.st["stop"]

    def result(self):
        return dict(self.st, alpha=np.asarray(self.st["alpha"]), b_ard=np.asarray(self.st["b_ard"]))


def gfa_fit(dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=True):
    return GfaFit(dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=drop_k)


def install(monkeypatch):
    """Route GFA's library calls through this module (and tests/fake_ops.py) for one test."""
    import sys

    from cca_zoo_b200.probabilistic import _gfa

    me = sys.modules[__name__]
    for name in ("gfa_fit", "GFA_MAX_K", "GFA_ARD_ALPHA_0", "GFA_TAU_ALPHA_0"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    monkeypatch.setattr(_gfa, "ops", fake_ops)
