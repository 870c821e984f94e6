"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.ey_fit`` (the Eckart-Young gradient
estimators), the companion of tests/fake_ops.py for ``cca_zoo_b200.linear._gradient``.  It runs the kernel forms of
oracle/ey.py (``cov_step`` / ``mb_step``) with the same contract as the binding: a fit handle whose ``run(n_steps,
idx)`` takes the row indices of the chunk, ``stopped()`` and ``result()`` -> (W as D x k float64 numpy, steps).
Nothing in the package imports this module; ``install(monkeypatch)`` swaps it in for one test (after
``fake_ops.install``)."""
from __future__ import annotations

import numpy as np
import torch

from tests import fake_ops

CALLS = {"run": 0}


class EyFit:
    def __init__(self, dims, init, c, learning_rate, momentum, tol, cov=None, views=None, batch=0):
        from oracle import ey as E

        self.E = E
        self.dims = [int(d) for d in dims]
        off = np.concatenate([[0], np.cumsum(self.dims)]).astype(int)
        init = np.asarray(init, dtype=np.float64)
        if init.shape[1] > 32:
            raise ValueError("ccab_ey_fit supports 1 <= k <= 32")
        self.st = E.new_state([init[off[i]:off[i + 1]] for i in range(len(self.dims))])
        self.hyper = (float(c), float(learning_rate), float(momentum), float(tol))
        self.cov = None if cov is None else cov.to(torch.float64).numpy()
        self.views = None if views is None else [v.to(torch.float64).numpy() for v in views]
        self.batch = int(batch)

    def run(self, n_steps, idx=None):
        CALLS["run"] += 1
        for s in range(int(n_steps)):
            if self.cov is not None:
                self.E.cov_step(self.st, self.cov, self.dims, *self.hyper)
            else:
                self.E.mb_step(self.st, self.views, idx[s].numpy().astype(np.int64), *self.hyper)

    def stopped(self):
        return self.st["stop"]

    def result(self):
        return np.vstack(self.st["W"]), self.st["steps"]


def ey_fit(dims, init, c, learning_rate, momentum, tol, cov=None, views=None, batch=0):
    return EyFit(dims, init, c, learning_rate, momentum, tol, cov=cov, views=views, batch=batch)


def column_sums(view):
    return view.to(torch.float64).sum(dim=0)


def install(monkeypatch):
    """Route the EY estimators' library calls through this module (and tests/fake_ops.py) for one test."""
    import sys

    from cca_zoo_b200.linear import _gradient

    me = sys.modules[__name__]
    for name in ("ey_fit", "column_sums"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    monkeypatch.setattr(_gradient, "ops", fake_ops)
