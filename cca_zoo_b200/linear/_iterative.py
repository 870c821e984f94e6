"""The sparse / ALS estimators on the GPU (mirrors cca_zoo/linear/_iterative.py): PLS_ALS, SCCA_PMD, ParkhomenkoCCA,
SCCA_Span and SCCA_ADMM.

The reference runs each as a Python loop of tall ``n x d`` mat-vecs with a data-space deflation between latent
dimensions.  Every step of that loop is a function of the block Gram matrix ``G = [X_1..X_m]^T [X_1..X_m]``
(``(n - 1) C`` for the covariance the moment pass produces, centred or not following ``center``):

  * target of view i: ``X_i^T t = sum_{j != i} G_ij w_j`` and ``||t||^2 = w_{-i}^T G w_{-i}``;
  * deflation ``X_i <- X_i (I - w_i a_i^T / s_i)``, ``a_i = G_ii w_i``, ``s_i = w_i^T a_i``: a congruence of G.

So a fit is the usual moment pass, then ONE library call (``ccab_als_fit``) that iterates all latent dimensions on the
``D x D`` matrix on the device.  ``partial_fit``, streamed host input and the sharded fit come from ``BaseModel``.

One intended divergence: float32 views iterate in float64 (the reference iterates in float32), like the
covariance stage of MCCA / GCCA here.
"""
from __future__ import annotations

from numbers import Integral, Real
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval

from .. import ops
from .._base import BaseModel
from .._validation import perview_parameter


class _BaseIterative(BaseModel):
    """ALS loop with deflation for each latent dimension (cca_zoo/linear/_iterative.py:38-135).

    ``max_iter`` sweeps at most per dimension; a dimension stops when ``max_i ||w_i - w_i_prev|| < tol``.  The initial
    weights come from ``np.random.default_rng(random_state)`` in the reference's order.  ``_fit_info["iters"]`` holds
    the sweeps each dimension took."""

    _solve_in_float64 = True
    _kind: ClassVar[str] = "pls"
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "max_iter": [Interval(Integral, 0, None, closed="left")],
        "tol": [Interval(Real, None, None, closed="neither")],
        "random_state": [None, Integral, np.random.Generator],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, max_iter: int = 500, tol: float = 1e-6,
                 random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.max_iter = max_iter
        self.tol = tol
        self.random_state = random_state

    def fit(self, views, y=None):
        C, dims, n_total = self._fit_device(views)
        return self._finish(self._solve(C, dims, n_total))

    def _view_params(self, dims):
        """Per-view parameter of the model's update (see ccab_als_fit)."""
        return [0.0] * len(dims)

    _mu = 1.0

    def _solve(self, C, dims, n_total):
        k = int(self.latent_dimensions)
        rng = np.random.default_rng(self.random_state)
        init = np.empty((k, int(sum(dims))))
        for d in range(k):                       # cca_zoo/linear/_iterative.py:86-89: per dimension, per view
            ws = [rng.standard_normal(p) for p in dims]
            init[d] = np.concatenate([w / np.linalg.norm(w) for w in ws])
        W, iters = ops.als_fit(C, dims, n_total, self._kind, self._view_params(dims), init, int(self.max_iter),
                               float(self.tol), mu=float(self._mu))
        self._fit_info = {"route": "als", "iters": iters}
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        return [torch.from_numpy(np.ascontiguousarray(W[off[i]:off[i + 1]])) for i in range(len(dims))]


class PLS_ALS(_BaseIterative):
    r"""PLS by alternating power steps, :math:`w_i \leftarrow X_i^\top \bar t_{\neg i} / \|\cdot\|`
    (cca_zoo/linear/_iterative.py:166-223)."""

    _kind = "pls"


class SCCA_PMD(_BaseIterative):
    r"""Sparse CCA by penalised matrix decomposition (cca_zoo/linear/_iterative.py:231-380): each update soft-thresholds
    at the level found by 50 bisection halvings so that :math:`\|w_i\|_1 \le \tau_i \sqrt{p_i}`."""

    _kind = "pmd"
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_BaseIterative._parameter_constraints, "tau": [Real, list]}

    def __init__(self, latent_dimensions: int = 1, center: bool = True, tau=1.0, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, max_iter=max_iter, tol=tol,
                         random_state=random_state, precision=precision, device=device)
        self.tau = tau

    def _view_params(self, dims):
        return [float(t) for t in perview_parameter("tau", self.tau, 1.0, len(dims))]


class ParkhomenkoCCA(_BaseIterative):
    r"""Sparse CCA by soft-thresholding power steps at a fixed :math:`\tau_i` (cca_zoo/linear/_iterative.py:839-930)."""

    _kind = "parkhomenko"
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_BaseIterative._parameter_constraints, "tau": [Real, list]}

    def __init__(self, latent_dimensions: int = 1, center: bool = True, tau=0.1, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, max_iter=max_iter, tol=tol,
                         random_state=random_state, precision=precision, device=device)
        self.tau = tau

    def _view_params(self, dims):
        return [float(t) for t in perview_parameter("tau", self.tau, 0.1, len(dims))]


class SCCA_Span(_BaseIterative):
    r"""SpanCCA: power steps that keep the ``span`` entries of largest magnitude, ties included
    (cca_zoo/linear/_iterative.py:631-722).  The default span is the width of view 0 for every view."""

    _kind = "span"
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_BaseIterative._parameter_constraints, "span": [None, Interval(Integral, 1, None, closed="left"), list]}

    def __init__(self, latent_dimensions: int = 1, center: bool = True, span=None, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, max_iter=max_iter, tol=tol,
                         random_state=random_state, precision=precision, device=device)
        self.span = span

    def _view_params(self, dims):
        default = dims[0]
        span = self.span if self.span is not None else default
        return [int(s) for s in perview_parameter("span", span, default, len(dims))]


class SCCA_ADMM(_BaseIterative):
    r"""Sparse CCA by ADMM (cca_zoo/linear/_iterative.py:388-514): a proximal gradient step on :math:`w_i`, soft
    thresholding at :math:`\tau_i / \mu` projected onto the unit ball for :math:`z_i`, a dual step; every target
    comes from the weights at the start of the iteration."""

    _kind = "admm"
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_BaseIterative._parameter_constraints, "tau": [Real, list],
        "mu": [Interval(Real, 0, None, closed="neither")]}

    def __init__(self, latent_dimensions: int = 1, center: bool = True, tau=0.1, mu: float = 1.0, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, max_iter=max_iter, tol=tol,
                         random_state=random_state, precision=precision, device=device)
        self.tau = tau
        self.mu = mu

    @property
    def _mu(self):
        return self.mu

    def _view_params(self, dims):
        return [float(t) for t in perview_parameter("tau", self.tau, 0.1, len(dims))]
