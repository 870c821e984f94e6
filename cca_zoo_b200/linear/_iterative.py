"""The sparse / ALS estimators on the GPU (mirrors cca_zoo/linear/_iterative.py): PLS_ALS, SCCA_PMD, ParkhomenkoCCA,
SCCA_Span, SCCA_ADMM, and the elastic-net regressions ElasticCCA and SCCA_IPLS.

The reference runs each as a Python loop of tall ``n x d`` mat-vecs with a data-space deflation between latent
dimensions.  Every step of that loop is a function of the block Gram matrix ``G = [X_1..X_m]^T [X_1..X_m]``
(``(n - 1) C`` for the covariance the moment pass produces, centred or not following ``center``):

  * target of view i: ``X_i^T t = sum_{j != i} G_ij w_j`` and ``||t||^2 = w_{-i}^T G w_{-i}``;
  * deflation ``X_i <- X_i (I - w_i a_i^T / s_i)``, ``a_i = G_ii w_i``, ``s_i = w_i^T a_i``: a congruence of G.

ElasticCCA and SCCA_IPLS refit sklearn's Ridge (``l1_ratio == 0``), Lasso (``== 1``) or ElasticNet on the view for
every update.  Those regressions are functions of G too.  With ``y = t / ||t||`` (ElasticCCA: ``t`` sums ALL views'
scores, view i with its current weights; SCCA_IPLS: the others), ``X_i^T y = sum_j G_ij w_j / ||t||`` and the
sub-problem of view i is

  ``min_w 1/2 w^T Q_i w - b_i^T w + lam_i ||w||_1``,  ``Q_i = G_ii / n + alpha_i (1 - l1_i) I``,  ``b_i = X_i^T y / n``,
  ``lam_i = alpha_i l1_i``

(Ridge, whose penalty is not divided by n: ``(G_ii + alpha I) w = X_i^T y``).  ``Q_i`` only changes at deflation, so its eigendecomposition is computed
once per latent dimension.  Each sub-problem is solved to a KKT residual of ``1e-12 max(1, ||b_i||_inf)``: by the
eigendecomposition when ``lam_i = 0`` (the minimum-norm solution when ``Q_i`` is singular, as Ridge's SVD fallback;
eigenvalues below a cut that follows the accuracy of the moments count as zero), by coordinate descent otherwise (at
most 1000 sweeps, sklearn's ``max_iter``; a descent that stops above the bound raises a ``ConvergenceWarning``).  SCCA_IPLS divides by the score's population std
``sqrt(w^T G_ii w / n - (s_i^T w / n)^2)``, ``s_i`` the column sums: zero when centred (deflation keeps the columns
centred), otherwise carried through the deflation as ``s_i^T <- s_i^T (I - w a^T / s)``.

So a fit is the usual moment pass, then ONE library call (``ccab_als_fit``) that iterates all latent dimensions on the
``D x D`` matrix on the device.  ``partial_fit``, streamed host input and the sharded fit come from ``BaseModel``.

One intended divergence: float32 views iterate in float64 (the reference iterates in float32), like the
covariance stage of MCCA / GCCA here.  ElasticCCA / SCCA_IPLS add one: on a singular ``G_ii`` at ``alpha = 0`` (from
the second latent dimension on, or whenever ``n <= d_i``) they return the minimum-norm least-squares weights, where
the reference's Lasso / ElasticNet coordinate descent keeps a path-dependent null-space component.  From the second
dimension on (``n > d_i``) the scores of the deflated views agree with the reference's; for ``n <= d_i`` the
reference's solver does not converge, and the two are not compared.
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


class _BaseRegression(_BaseIterative):
    """ElasticCCA / SCCA_IPLS: per-view ``alpha`` and ``l1_ratio`` (cca_zoo/linear/_iterative.py:938-982).

    The reference declares no constraints for them; sklearn's regressors reject a negative ``alpha`` or an
    ``l1_ratio`` outside [0, 1] with ``InvalidParameterError`` once the first update runs.  Here the same error, with
    the regressor's wording, is raised before any kernel runs."""

    _default_l1: ClassVar[float] = 1.0
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_BaseIterative._parameter_constraints, "alpha": [Real, list], "l1_ratio": [Real, list]}

    def __init__(self, latent_dimensions: int = 1, center: bool = True, alpha=0.0, l1_ratio=1.0, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, max_iter=max_iter, tol=tol,
                         random_state=random_state, precision=precision, device=device)
        self.alpha = alpha
        self.l1_ratio = l1_ratio

    # relative eigenvalue cut of the alpha l1 = 0 solves: the null space of a singular G_ii is only as exact as the
    # moments (float64 or exact accumulation: ~1e-16; 3xTF32 float32 moments: ~1e-7 per entry; single-pass TF32: ~1e-3)
    _RCOND = {"exact": 1e-12, "tf32x3": 1e-5, "tf32x3b": 1e-5, "tf32": 1e-3}

    @property
    def _mu(self):
        if getattr(self, "_in_dtype", torch.float64) == torch.float64:
            return 1e-12
        return self._RCOND[self.precision]

    def _covariance_stage(self, mom, n_local, dims, in_dtype, *args, **kwargs):
        self._in_dtype = in_dtype
        return super()._covariance_stage(mom, n_local, dims, in_dtype, *args, **kwargs)

    def _regression_params(self, m):
        """[alpha_0, l1_0, alpha_1, l1_1, ...], each pair checked against the constraints of the sklearn regressor the
        reference builds for it (cca_zoo/linear/_iterative.py:957-981), with that regressor's error."""
        from sklearn.linear_model import ElasticNet, Lasso, Ridge
        from sklearn.utils._param_validation import validate_parameter_constraints

        alpha = perview_parameter("alpha", self.alpha, 0.0, m)
        l1 = perview_parameter("l1_ratio", self.l1_ratio, self._default_l1, m)
        out = []
        for a, r in zip(alpha, l1):
            reg, given = (Ridge, {"alpha": a}) if r == 0.0 else (
                (Lasso, {"alpha": a}) if r == 1.0 else (ElasticNet, {"alpha": a, "l1_ratio": r}))
            validate_parameter_constraints(reg._parameter_constraints, given, caller_name=reg.__name__)
            out += [float(a), float(r)]
        return out

    def _validate_params(self):
        super()._validate_params()
        if isinstance(self.alpha, list) and isinstance(self.l1_ratio, list) and len(self.alpha) != len(self.l1_ratio):
            raise ValueError("alpha and l1_ratio give different numbers of views")
        m = len(self.alpha) if isinstance(self.alpha, list) else (
            len(self.l1_ratio) if isinstance(self.l1_ratio, list) else 1)
        self._regression_params(m)

    def _view_params(self, dims):
        params = self._regression_params(len(dims))
        if self._kind == "ipls":
            means = self._column_means if not self.center else np.zeros(int(sum(dims)))
            params += [float(x) for x in means]
        return params


class ElasticCCA(_BaseRegression):
    r"""Elastic-net CCA (cca_zoo/linear/_iterative.py:730-831): each view is regressed by Ridge / Lasso / ElasticNet
    on the normalised sum of ALL views' scores (its own included, Gauss-Seidel order); the coefficients are used as
    they come.  Defaults ``alpha=0``, ``l1_ratio=0.5``."""

    _kind = "elastic"
    _default_l1 = 0.5

    def __init__(self, latent_dimensions: int = 1, center: bool = True, alpha=0.0, l1_ratio=0.5, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, alpha=alpha, l1_ratio=l1_ratio,
                         max_iter=max_iter, tol=tol, random_state=random_state, precision=precision, device=device)


class SCCA_IPLS(_BaseRegression):
    r"""Iterative penalised least squares (cca_zoo/linear/_iterative.py:522-623): each view is regressed on the
    normalised sum of the OTHER views' scores, then divided by the population std of its score.  Defaults
    ``alpha=0``, ``l1_ratio=1``."""

    _kind = "ipls"
    _default_l1 = 1.0
    _wants_column_means = True

    def __init__(self, latent_dimensions: int = 1, center: bool = True, alpha=0.0, l1_ratio=1.0, max_iter: int = 500,
                 tol: float = 1e-6, random_state=None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, alpha=alpha, l1_ratio=l1_ratio,
                         max_iter=max_iter, tol=tol, random_state=random_state, precision=precision, device=device)
