"""TEST INFRASTRUCTURE ONLY: the global-batch entry points of ``cca_zoo_b200.ops`` on top of the torch-CPU stand-in
(tests/fake_ops.py), with a call log, so that the host logic of ``global_batch=True`` -- one exchange per forward,
no read-back when the local shard is wide enough, the collective route decisions -- runs on a CPU-only machine.
``install(monkeypatch)`` routes the objectives through it for one test and returns the call log."""
from __future__ import annotations

import sys

import torch

from tests import fake_ops as F


class Calls(list):
    """Names of the ops calls in order, plus the number of host read-backs (``.item()`` / ``.tolist()``)."""

    def names(self):
        return [c for c in self]


LOG = Calls()


def _logged(name, fn):
    def wrapper(*a, **k):
        LOG.append(name)
        return fn(*a, **k)
    return wrapper


def moments_size(dims):
    _, Dp = F._layout(dims)
    return Dp * Dp + Dp


def _blocks(saved, d1, d2):
    s = saved.to(torch.float64)
    G11 = s[:d1 * d1].reshape(d1, d1)
    P = s[d1 * d1:d1 * d1 + d1 * d2].reshape(d1, d2)
    G22 = s[d1 * d1 + d1 * d2:d1 * d1 + d1 * d2 + d2 * d2].reshape(d2, d2)
    tail = s[d1 * d1 + d1 * d2 + d2 * d2:]
    return G11, P, G22, tail


def ccaloss_fwd_moments(mom, n_dev, d1, d2, eps, dtype):
    flags = torch.zeros(3, dtype=torch.int32)
    if not bool(torch.isfinite(mom).all()):
        flags[2] = 1
    C, mean = F.covariance(mom, [d1, d2], n_dev, True, torch.float64)
    S11 = C[:d1, :d1] + eps * torch.eye(d1, dtype=torch.float64)
    S22 = C[d1:, d1:] + eps * torch.eye(d2, dtype=torch.float64)
    S12 = C[:d1, d1:]
    for i, S in enumerate((S11, S22)):
        L, info = torch.linalg.cholesky_ex(S)
        if int(info) != 0 or bool((L.diagonal() ** 2 <= 0.25 * eps).any()):
            flags[i] = 1
    A1, A2 = torch.linalg.inv(S11), torch.linalg.inv(S22)
    P = A1 @ S12 @ A2
    saved = torch.cat([(P @ S12.T @ A1).reshape(-1), P.reshape(-1), (A2 @ S12.T @ P).reshape(-1), mean,
                       n_dev.to(torch.float64).reshape(1)]).to(dtype)
    return (-(P * S12).sum()).reshape(1).to(dtype), saved, flags


def ccaloss_bwd_global(z1, z2, saved, grad_out):
    d1, d2 = z1.shape[1], z2.shape[1]
    G11, P, G22, tail = _blocks(saved, d1, d2)
    mu1, mu2, N = tail[:d1], tail[d1:d1 + d2], float(tail[-1])
    x1, x2 = z1.to(torch.float64) - mu1, z2.to(torch.float64) - mu2
    s = 2.0 / (N - 1) * float(grad_out.reshape(-1)[0])
    return ((x1 @ G11 - x2 @ P.T) * s).to(z1.dtype), ((x2 @ G22 - x1 @ P) * s).to(z1.dtype)


def row_sub_scale_(A, r, s):
    A.sub_(r.to(A.dtype).reshape(1, -1)).mul_(s.to(A.dtype).reshape(1, 1))
    return A


def install(monkeypatch):
    """Route the objectives through the stand-in, with every ops call and read-back logged; returns the log."""
    from cca_zoo_b200.deep import objectives

    F.install(monkeypatch)
    me = sys.modules[__name__]
    for name in ("moments_size", "ccaloss_fwd_moments", "ccaloss_bwd_global", "row_sub_scale_"):
        monkeypatch.setattr(F, name, getattr(me, name), raising=False)
    LOG.clear()
    for name in ("moments", "covariance", "ccaloss_fwd", "ccaloss_bwd", "ccaloss_fwd_moments", "ccaloss_bwd_global",
                 "syevj", "potrf_inv_", "row_sub_scale_"):
        monkeypatch.setattr(F, name, _logged(name, getattr(F, name)), raising=False)
    count = objectives._global_count
    monkeypatch.setattr(objectives, "_global_count", _logged("read_n", count))
    return LOG
