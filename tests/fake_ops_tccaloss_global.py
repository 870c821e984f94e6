"""TEST INFRASTRUCTURE ONLY: the entry points of the global-batch ``TCCALoss`` on top of the torch-CPU stand-ins
(tests/fake_ops.py, tests/fake_ops_global.py), with the contracts of ``cca_zoo_b200.ops``: ``tcca_moment`` with its
``scale`` (default 1/n) and ``out`` arguments, and ``tcca_moment_adjoint`` scaled by ``scale`` times the device
scalar, both from the float64 restatement of oracle/tccaloss.py.  ``install(monkeypatch)`` routes the objectives
through them for one test, logs every call in the call log of tests/fake_ops_global.py, and returns that log."""
from __future__ import annotations

import sys

import torch

from cca_zoo_b200.ops import TCCA_MAX_ENTRIES, TCCA_MAX_VIEWS  # noqa: F401
from tests import fake_ops as F
from tests import fake_ops_global as FG


def tcca_moment(Z, nsplit=0, scale=None, out=None):
    from oracle import tccaloss as O

    H = [z.to(torch.float64).numpy() for z in Z]
    n = H[0].shape[0]
    f = 1.0 / max(n, 1) if scale is None else float(scale)
    M = torch.from_numpy((O.moment(H) * (n * f)).reshape(H[0].shape[1], -1).copy())
    if out is None:
        return M
    out.copy_(M.reshape(out.shape))
    return out


def tcca_moment_adjoint(M, H, scale=1.0, scale_dev=None):
    from oracle import tccaloss as O

    Hn = [h.to(torch.float64).numpy() for h in H]
    f = scale * (1.0 if scale_dev is None else float(scale_dev.reshape(-1)[0]))
    T = M.to(torch.float64).contiguous().numpy().reshape([h.shape[1] for h in Hn])
    return [torch.from_numpy(f * y) for y in O.adjoint(T, Hn)]


def install(monkeypatch):
    """Route the objectives through the stand-ins, with every ops call logged; returns the log."""
    log = FG.install(monkeypatch)
    me = sys.modules[__name__]
    for name in ("TCCA_MAX_VIEWS", "TCCA_MAX_ENTRIES"):
        monkeypatch.setattr(F, name, getattr(me, name), raising=False)
    for name in ("tcca_moment", "tcca_moment_adjoint"):
        monkeypatch.setattr(F, name, FG._logged(name, getattr(me, name)), raising=False)
    return log
