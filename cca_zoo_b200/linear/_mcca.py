"""MCCA on the GPU (mirrors cca_zoo/linear/_mcca.py)."""
from __future__ import annotations

from numbers import Real
from typing import Any, ClassVar

from sklearn.utils._param_validation import Interval, StrOptions

from .. import ops
from ..ops import mcca_fit_workspace_bytes   # a host query of the library: needs no device
from .._base import BaseModel
from .._solvers import mcca_weights
from .._validation import perview_parameter, validate_views
from ._rcca import RIDGE_PARAMETER

#: cca_zoo/_utils/_param_constraints.py:22 (POSITIVE_EPS)
POSITIVE_EPS: list[Any] = [Interval(Real, 0, None, closed="neither")]


class MCCA(BaseModel):
    r"""Multiset CCA for two or more views (cca_zoo/linear/_mcca.py:16-135).

    Solves :math:`A v = \lambda B v` with :math:`A` the between-view block covariance and
    :math:`B` the ridge-regularised block-diagonal within-view covariance, eigenvectors normalised
    to :math:`v^\top B v = 1`.  ``pca`` is accepted for signature compatibility: the reference's PCA
    pre-rotation is an exact change of basis (identical weights for full-column-rank views), which
    the covariance form here subsumes -- the per-view eigendecompositions ARE that rotation.

    As in the reference (np.cov upcasts, SURVEY.md §7.3-7) the eigen-stage runs in float64 and
    ``weights_`` are float64 even for float32 views.
    """

    _solve_in_float64 = True
    _covariance_always_centred = True      # np.cov in _build_A / _build_B, PCA in the pca=True branch
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "c": RIDGE_PARAMETER,
        "pca": ["boolean"],
        "eps": POSITIVE_EPS,
        "solver": [StrOptions({"auto", "eigen", "cholesky"})],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.0, pca: bool = True,
                 eps: float = 1e-6, precision: str = "tf32x3b", device=None, solver: str = "auto") -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.c = c
        self.pca = pca
        self.eps = eps
        self.solver = solver

    def fit(self, views, y=None):
        self._validate_params()
        validated = validate_views(views)
        device = self._device()
        mom, n_local, dims, in_dtype = self._local_moments(validated, device)
        self._partial = None
        return self._fit_moments(mom, n_local, dims, in_dtype)

    def _device_fit_plan(self, dims, n_local, in_dtype):
        """Device-side fit (csrc/fit.cu: mcca_fit) for plain MCCA on large, well-posed problems; subclasses that
        rebuild A / B (GRCCA, PartialCCA) assemble on the host and never get here.  Declined when the library refuses
        the block width p in the solve dtype (its workspace query answers 0)."""
        if type(self) is not MCCA or self.solver == "eigen":
            return None
        D = int(sum(dims))
        if self.solver == "auto" and not (D >= 512 and n_local > max(dims)):
            return None
        k = min(int(self.latent_dimensions), D)
        p = min(D, max(2 * k, k + 32))
        c_ = [float(x) for x in perview_parameter("c", self.c, 0.0, len(dims))]
        if 4 * k > D or max(c_) > 0.9 or mcca_fit_workspace_bytes(dims, k, p, self._solve_dtype(in_dtype)) == 0:
            return None
        eps = float(self.eps)

        def call(mom, dims_, n_host, n_dev, solve_dtype, iters):
            # np.cov centres regardless of `center` (cca_zoo/linear/_mcca.py:150,166)
            return ops.mcca_fit(mom, dims_, n_host, n_dev, True, c_, eps, k, p, iters, solve_dtype)

        return {"call": call, "k": k, "iters": [32, 60]}

    def _solve(self, C, dims, n_total):
        c_ = perview_parameter("c", self.c, 0.0, self.n_views_)
        return mcca_weights(C, dims, self.latent_dimensions, [float(x) for x in c_], float(self.eps),
                            solver=self.solver)
