"""rCCA / CCA / PLS on the GPU (mirrors cca_zoo/linear/_rcca.py, _cca.py, _pls.py)."""
from __future__ import annotations

import os

from numbers import Real
from typing import Any, ClassVar

from sklearn.utils._param_validation import Interval, StrOptions

from .._base import BaseModel
from .. import ops
from ..ops import rcca_fit_workspace_bytes   # a host query of the library: needs no device
from .._solvers import rcca_weights
from .._validation import perview_parameter, validate_views

#: cca_zoo/_utils/_param_constraints.py:18 (RIDGE_PARAMETER)
RIDGE_PARAMETER: list[Any] = [Interval(Real, 0, 1, closed="both"), "array-like"]


class rCCA(BaseModel):
    r"""Regularised CCA (canonical ridge) for exactly two views.

    Same estimator as ``cca_zoo.linear.rCCA`` (cca_zoo/linear/_rcca.py:16-101): maximise
    :math:`w_1^\top X_1^\top X_2 w_2` s.t. :math:`w_i^\top((1-c_i) X_i^\top X_i + c_i I) w_i = 1`.
    The reference whitens each view with a tall SVD and takes the SVD of the whitened
    cross-covariance; here the same weights come from the block covariance (one tensor-core pass over
    the data) and small Jacobi eigen/singular-value solves on the device.

    Args:
        latent_dimensions: number of latent dimensions (default 1).
        center: subtract column means (default True).
        c: ridge parameter(s) in [0, 1]; scalar or ``[c1, c2]``.
        precision: covariance arithmetic for float32 inputs: ``"tf32x3b"`` (default: 3xTF32 with the two cross terms
            as bf16 tensor-core MMAs, float32-grade at 2/3 of the tensor work), ``"tf32x3"`` (all three terms in
            TF32: ~2.5x smaller covariance error, 1.3x slower), ``"tf32"`` (single tensor-core pass) or ``"exact"``
            (CUDA-core FMA).
        device: CUDA device (default: current).
        solver: ``"eigen"`` mirrors the reference step by step (eigendecomposition of each view's
            covariance, Jacobi SVD of the whitened cross-covariance); ``"cholesky"`` whitens with Cholesky
            factors and extracts the leading ``latent_dimensions`` singular triplets by subspace iteration
            (identical weights, much less work when ``latent_dimensions << n_features``); ``"auto"`` picks
            the latter for large full-rank problems and falls back to ``"eigen"`` otherwise.
    """

    _requires_two_views = True
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "c": RIDGE_PARAMETER,
        "solver": [StrOptions({"auto", "eigen", "cholesky"})],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.0, precision: str = "tf32x3b",
                 device=None, solver: str = "auto") -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.c = c
        self.solver = solver

    def fit(self, views, y=None):
        """Fit on a list of exactly two ``(n_samples, n_features_i)`` arrays (numpy or torch)."""
        self._validate_params()
        validated = validate_views(views)
        device = self._device()
        mom, n_local, dims, in_dtype = self._local_moments(validated, device)
        self._partial = None
        if len(dims) != 2:
            raise ValueError(
                f"rCCA requires exactly 2 views, got {len(dims)}. "
                "Use MCCA for more than 2 views."
            )
        return self._fit_moments(mom, n_local, dims, in_dtype)

    def _device_fit_plan(self, dims, n_local, in_dtype):
        """The device-side fit (csrc/fit.cu: Cholesky whitening + subspace iteration, everything on the stream) is
        taken for large, well-posed problems: ``solver`` allows it, k is small against the widths (4k <= min d_i) and
        the library takes the iterated block width p in the solve dtype (its workspace query answers 0 otherwise: the
        single-CTA Ritz solve bounds p).  Whether n > max d_i holds for the TOTAL sample count, and whether the blocks
        are positive definite, is decided on the device (status word)."""
        if self.solver == "eigen":
            return None
        if self.solver == "auto" and not (min(dims) >= 256 and n_local > max(dims)):
            return None
        k = min(int(self.latent_dimensions), dims[0], dims[1])
        over = int(os.environ.get("CCAB_FIT_OVERSAMPLE", "0")) or max(16, k // 4)
        p = min(min(dims), k + over)
        if 4 * k > min(dims) or rcca_fit_workspace_bytes(dims, k, p, self._solve_dtype(in_dtype)) == 0:
            return None
        first = int(os.environ.get("CCAB_FIT_ITERS", "0")) or 6
        c_ = [float(x) for x in perview_parameter("c", self.c, 0.0, 2)]
        center = bool(self.center)

        def call(mom, dims_, n_host, n_dev, solve_dtype, iters):
            return ops.rcca_fit(mom, dims_, n_host, n_dev, center, c_, k, p, iters, solve_dtype)

        return {"call": call, "k": k, "iters": [first, 20]}

    def _solve(self, C, dims, n_total):
        c_ = perview_parameter("c", self.c, 0.0, 2)
        return rcca_weights(C, dims, n_total, self.latent_dimensions, [float(x) for x in c_], solver=self.solver)


class CCA(rCCA):
    """Canonical Correlation Analysis: ``rCCA`` with ``c=0`` (cca_zoo/linear/_cca.py:10-76)."""

    def __init__(self, latent_dimensions: int = 1, center: bool = True, precision: str = "tf32x3b",
                 device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, c=0.0, precision=precision,
                         device=device, solver="auto")


class PLS(rCCA):
    """Partial Least Squares: ``rCCA`` with ``c=1`` (cca_zoo/linear/_pls.py:10-77)."""

    def __init__(self, latent_dimensions: int = 1, center: bool = True, precision: str = "tf32x3b",
                 device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, c=1.0, precision=precision,
                         device=device, solver="auto")
