"""The Eckart-Young gradient estimators on the GPU (mirrors cca_zoo/linear/gradient/): CCA_EY, PLS_EY and MCCA_EY.

The reference minimises the EY loss ``L = -2 tr(C_ey - c V) + tr(Vb Vb)`` (cca_zoo/linear/gradient/_cca_ey.py:212-225)
by momentum steps on mini-batches of ``bs`` rows (cca_zoo/linear/gradient/_base.py:113-130).  Two routes here, both
ONE library call (``ccab_ey_fit``) per chunk of steps, every step inside one persistent kernel:

  * full batch (``batch_size`` None or >= n): every quantity of a step is a function of the centred block covariance,
    so the fit is the usual moment pass followed by steps whose cost does not depend on n.  The reference's per-step
    permutations change nothing and are not drawn.
  * mini-batch: the rows of each step are gathered on the device straight from the raw views (float32 or float64, in
    place); the row indices are drawn on the host in the reference's order, one chunk at a time, while the previous
    chunk runs.  The stop flag is read back once per chunk, never per step.

The arithmetic is float64 throughout (the reference's float64 initial weights upcast every product).  ``partial_fit``
and the sharded fit are not supported: the reference has neither for this family, and the CCA initialisation takes
rows of one global permutation.
"""
from __future__ import annotations

from numbers import Real
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval

from .. import ops, parallel
from .._base import BaseModel
from .._validation import validate_views

#: bytes of row indices drawn on the host per chunk of mini-batch steps
_CHUNK_INDEX_BYTES = 4 << 20


def _householder_r(z):
    return np.linalg.qr(z, mode="r")


class CCA_EY(BaseModel):
    r"""Eckart-Young CCA, ridge-blended with PLS_EY by ``c`` (cca_zoo/linear/gradient/_cca_ey.py).

    ``c = 0`` is plain CCA_EY, ``c = 1`` PLS_EY's loss.  Initial weights give orthonormal projections of one batch
    (cca_zoo/_utils/_ey.py:173-184).  ``_fit_info`` records the ``route`` ("covariance" or "minibatch"), ``iters``
    (steps taken) and ``calls`` (library calls).  Gradient descent on the unregularised loss (``c = 0``) can diverge to
    NaN weights when a batch barely outnumbers the features; as in the reference this returns NaN weights and does not
    raise."""

    _solve_in_float64 = True
    _covariance_always_centred = True     # the gradient and the objective centre within the batch
    _wants_second_moment = True           # uncentred initialisation: z0 of the raw views
    _projection_init: ClassVar[bool] = True
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "c": [Interval(Real, 0, 1, closed="both")],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c: float = 0.0, learning_rate: float = 1e-2,
                 max_iter: int = 1000, batch_size: int | None = None, tol: float = 1e-6, momentum: float = 0.9,
                 random_state: int | None = None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.c = c
        self.learning_rate = learning_rate
        self.max_iter = max_iter
        self.batch_size = batch_size
        self.tol = tol
        self.momentum = momentum
        self.random_state = random_state

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        self._validate_params()
        if parallel.is_distributed():
            raise NotImplementedError(f"{type(self).__name__} has no sharded fit: its initialisation draws rows of one "
                                      "global permutation")
        validated = validate_views(views)
        n = int(validated[0].shape[0])
        dims = [int(v.shape[1]) for v in validated]
        ks = {min(int(self.latent_dimensions), p) for p in dims}
        if len(ks) != 1:
            raise ValueError(f"latent_dimensions = {self.latent_dimensions} gives a different number of components per "
                             f"view for widths {dims}")
        k = ks.pop()
        bs = n if self.batch_size is None else min(int(self.batch_size), n)
        rng = np.random.default_rng(self.random_state)
        if bs == n:
            W, iters, calls = self._fit_covariance(validated, n, k, rng)
            route = "covariance"
        else:
            W, iters, calls = self._fit_minibatch(validated, n, dims, k, bs, rng)
            route = "minibatch"
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        self.weights_ = [np.ascontiguousarray(W[off[i]:off[i + 1]]) for i in range(len(dims))]
        self._fit_info = {"route": route, "iters": iters, "calls": calls}
        return self

    def partial_fit(self, views, y=None, solve: bool = True):
        raise NotImplementedError(f"{type(self).__name__} has no partial_fit (neither has the reference); use fit "
                                  "with batch_size for mini-batch steps")

    def _solve(self, C, dims, n_total):
        raise NotImplementedError("the EY estimators iterate in ccab_ey_fit, not on a solved covariance")

    def _hyper(self):
        return float(self.c), float(self.learning_rate), float(self.momentum), float(self.tol)

    # ------------------------------------------------------------------ full batch: the covariance route
    def _fit_covariance(self, validated, n, k, rng):
        device = self._device()
        mom, n_local, dims, in_dtype = self._local_moments(validated, device)
        self._partial = None
        C, dims, n = self._covariance_stage(mom, n_local, dims, in_dtype, True)
        perm = rng.choice(n, n, replace=False) if self._projection_init else None
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        init = []
        for i, p in enumerate(dims):
            w0, _ = np.linalg.qr(rng.standard_normal((p, k)))
            if self._projection_init:
                R = self._init_r_covariance(validated[i], i, w0, perm, C, off, n)
                w0 = w0 @ np.linalg.solve(R, np.eye(k))
            init.append(w0)
        fit = ops.ey_fit(dims, np.vstack(init), *self._hyper(), cov=C)
        fit.run(int(self.max_iter))
        W, iters = fit.result()
        return W, iters, 1

    def _rows(self, view, rows, i):
        """Rows of view i (host float64), centred when ``center``."""
        sel = view[torch.as_tensor(rows, device=view.device)] if isinstance(view, torch.Tensor) else view[rows]
        x = sel.detach().cpu().to(torch.float64).numpy() if isinstance(sel, torch.Tensor) else np.asarray(sel, np.float64)
        return x - np.asarray(self.means_[i], dtype=np.float64) if self.center else x

    def _init_r_covariance(self, view, i, w0, perm, C, off, n):
        """R of qr(views_[i][perm] @ w0) without the n x k product: Householder QR gives the same R (signs included) for
        z0 and for the 2k x k stack [z0[:k]; chol(z0^T z0 - z0[:k]^T z0[:k])^T], and z0^T z0 = w0^T (n - 1) C_ii w0
        (the raw second moment when ``center=False``)."""
        k = w0.shape[1]
        if n >= 2 * k:
            sl = slice(int(off[i]), int(off[i + 1]))
            M = C if self.center else self._second_moment
            w = torch.from_numpy(np.ascontiguousarray(w0)).to(C.device)
            G = ops.gemm(w, ops.gemm(M[sl, sl], w), transa=True).cpu().numpy() * (n - 1)
            head = self._rows(view, perm[:k], i) @ w0
            try:
                L = np.linalg.cholesky(0.5 * ((G - head.T @ head) + (G - head.T @ head).T))
            except np.linalg.LinAlgError:
                L = None
            if L is not None:
                return _householder_r(np.vstack([head, L.T]))
        return _householder_r(self._rows(view, perm, i) @ w0)

    # ------------------------------------------------------------------ mini-batch route
    def _fit_minibatch(self, validated, n, dims, k, bs, rng):
        device = self._device()
        views = []
        for v in validated:
            t = v if isinstance(v, torch.Tensor) and v.is_cuda else self._to_device(v, device)
            if t.dtype not in (torch.float32, torch.float64):
                t = t.to(torch.float64)
            if t.stride(1) != 1:
                t = t.contiguous()
            views.append(t)
        if len({v.dtype for v in views}) > 1:
            views = [v.to(torch.float64) for v in views]
        sums = [ops.column_sums(v) for v in views]
        if not all(bool(torch.isfinite(s).all()) for s in sums):
            raise ValueError("Input contains NaN or infinity.")
        self.n_views_, self.n_features_in_, self.n_samples_ = len(dims), dims, n
        np_dtype = np.float32 if views[0].dtype == torch.float32 else np.float64
        if self.center:
            self.means_ = [(s / n).cpu().numpy().astype(np_dtype) for s in sums]
        else:
            self.means_ = [np.zeros(p) for p in dims]
        self._partial = None

        idx0 = rng.choice(n, bs, replace=False) if self._projection_init else None
        init = []
        for i, p in enumerate(dims):
            w0, _ = np.linalg.qr(rng.standard_normal((p, k)))
            if self._projection_init:
                rows = views[i][torch.as_tensor(idx0, device=device)].to(torch.float64)
                z0 = ops.gemm(rows, torch.from_numpy(np.ascontiguousarray(w0)).to(device)).cpu().numpy()
                if self.center:
                    z0 = z0 - np.asarray(self.means_[i], dtype=np.float64) @ w0
                w0 = w0 @ np.linalg.solve(_householder_r(z0), np.eye(k))
            init.append(w0)
        fit = ops.ey_fit(dims, np.vstack(init), *self._hyper(), views=views, batch=bs)

        max_iter = int(self.max_iter)
        chunk = max(1, min(max_iter, _CHUNK_INDEX_BYTES // (4 * bs)))
        pinned = [torch.empty((chunk, bs), dtype=torch.int32, pin_memory=torch.cuda.is_available()) for _ in range(2)]
        dev_idx = torch.empty((chunk, bs), dtype=torch.int32, device=device)

        def draw(buf, steps):
            arr = buf.numpy()
            for s in range(steps):                       # the reference's draw per step, in order
                arr[s] = rng.choice(n, bs, replace=False)

        done, calls, cur = 0, 0, 0
        while done < max_iter:
            steps = min(chunk, max_iter - done)
            draw(pinned[cur], steps)                     # overlaps the previous chunk on the device
            if calls and fit.stopped():                  # one small read-back per chunk
                break
            dev_idx[:steps].copy_(pinned[cur][:steps], non_blocking=True)
            fit.run(steps, dev_idx)
            calls += 1
            done += steps
            cur ^= 1
        W, iters = fit.result()
        return W, iters, calls


class PLS_EY(CCA_EY):
    r"""Stochastic Eckart-Young PLS: CCA_EY with ``c`` fixed at 1 and orthonormal initial weights
    (cca_zoo/linear/gradient/_pls_ey.py)."""

    _wants_second_moment = False
    _projection_init = False

    def __init__(self, latent_dimensions: int = 1, center: bool = True, learning_rate: float = 1e-2,
                 max_iter: int = 1000, batch_size: int | None = None, tol: float = 1e-6, momentum: float = 0.9,
                 random_state: int | None = None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, c=1.0, learning_rate=learning_rate,
                         max_iter=max_iter, batch_size=batch_size, tol=tol, momentum=momentum,
                         random_state=random_state, precision=precision, device=device)


class MCCA_EY(CCA_EY):
    r"""Eckart-Young multiview CCA (cca_zoo/linear/gradient/_mcca_ey.py): CCA_EY, whose loss is already defined for any
    number of views."""
