"""TEST INFRASTRUCTURE ONLY: the torch-CPU stand-in for ``cca_zoo_b200.ops.tcca_moment`` and
``tcca_moment_adjoint``, the companion of tests/fake_ops.py for ``TCCALoss`` (cca_zoo_b200/deep/objectives.py).  It
runs the float64 restatement of oracle/tccaloss.py with the binding's contracts: M as the p_1 x prod_{i>1} p_i
unfolding, the adjoint scaled by ``scale`` times the device scalar.  Nothing in the package imports this module;
``install(monkeypatch)`` swaps it in for one test (it installs tests/fake_ops.py as well).  ``CALLS`` counts the
calls of each."""
from __future__ import annotations

import torch

from cca_zoo_b200.ops import TCCA_MAX_ENTRIES, TCCA_MAX_VIEWS  # noqa: F401
from tests import fake_ops

CALLS = {"moment": 0, "adjoint": 0}


def tcca_moment(Z, nsplit=0):
    from oracle import tccaloss as O

    CALLS["moment"] += 1
    H = [z.to(torch.float64).numpy() for z in Z]
    return torch.from_numpy(O.moment(H).reshape(H[0].shape[1], -1).copy())


def tcca_moment_adjoint(M, H, scale=1.0, scale_dev=None):
    from oracle import tccaloss as O

    CALLS["adjoint"] += 1
    Hn = [h.to(torch.float64).numpy() for h in H]
    f = scale * (1.0 if scale_dev is None else float(scale_dev.reshape(-1)[0]))
    T = M.to(torch.float64).numpy().reshape([h.shape[1] for h in Hn])
    return [torch.from_numpy(f * y) for y in O.adjoint(T, Hn)]


def install(monkeypatch):
    """Route TCCALoss's library calls through this module and tests/fake_ops.py for one test."""
    import sys

    fake_ops.install(monkeypatch)
    me = sys.modules[__name__]
    for name in ("tcca_moment", "tcca_moment_adjoint", "TCCA_MAX_VIEWS", "TCCA_MAX_ENTRIES"):
        monkeypatch.setattr(fake_ops, name, getattr(me, name), raising=False)
    CALLS.update(moment=0, adjoint=0)
