"""TCCA (tensor CCA) on the GPU (mirrors cca_zoo/linear/_tcca.py).

The reference whitens each view, builds the n x p_1 x ... x p_m array of per-sample outer products and only then
averages over the samples (3 views of 128 features at n = 1e5 would be 1.7 TB), then runs tensorly's ``parafac`` on
the averaged tensor.  A fit here is:

  1. the moment pass, with the covariance always centred (the reference whitens with ``np.cov``);
  2. the symmetric whiteners S_i = V (lambda + floor)^-1/2 V^T of (1 - c_i) cov_i + c_i I, from ``syevj``;
  3. Z_i = (X_i - mu_i) S_i, one DMMA GEMM per view with the mean term preloaded (mu_i = 0 for ``center=False``);
  4. the cross-moment tensor M = Z_1^T KR(Z_2, ..., Z_m) / n as one contraction over the samples (``ccab_tcca_moment``);
  5. tensorly's default CP-ALS on M (``ccab_tcca_fit``): the start from the leading eigenvectors of every unfolding
     Gram, the random start columns drawn on the host in tensorly's order, then up to 100 iterations enqueued at once;
  6. weights_i = S_i F_i, copied back with the state block in one transfer.

``partial_fit`` and the sharded fit are not supported: the whiteners must be known before the contraction pass.
"""
from __future__ import annotations

from numbers import Integral, Real
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval

from .. import ops, parallel
from .._base import BaseModel
from .._validation import perview_parameter, validate_views
from ._rcca import RIDGE_PARAMETER


def random_start_columns(dims, k: int, random_state):
    """tensorly's random start columns (``initialize_cp``, init='svd'): ``rng.random_sample((p_j, k - p_j))`` for every
    mode with p_j < k, in mode order, from one ``RandomState(random_state)`` (numpy's global one for None)."""
    rng = np.random.mtrand._rand if random_state is None else np.random.RandomState(random_state)
    return [rng.random_sample((p, k - p)) if p < k else None for p in dims]


class TCCA(BaseModel):
    r"""Tensor CCA (cca_zoo/linear/_tcca.py): CP decomposition of the cross-moment tensor of the whitened views.

    Same arguments, defaults and fitted attributes as the reference (``weights_`` -- always float64 --, ``means_``,
    ``n_views_``, ``n_features_in_``, ``n_samples_``), plus ``precision`` (arithmetic of the moment pass for float32
    views) and ``device``.  Limits: at most 8 views, ``latent_dimensions`` at most 64, and at most 2^25 tensor entries
    (the product of the view widths).  The iteration count and the reconstruction errors are in ``_fit_info``."""

    _solve_in_float64 = True
    _covariance_always_centred = True     # the whitening uses np.cov, which always centres
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "c": RIDGE_PARAMETER,
        "eps": [Interval(Real, 0, None, closed="neither")],
        "random_state": [None, Interval(Integral, 0, None, closed="left")],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.0, eps: float = 1e-6,
                 random_state: int | None = None, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.c = c
        self.eps = eps
        self.random_state = random_state

    def _check_limits(self, dims):
        k = int(self.latent_dimensions)
        if k > ops.TCCA_MAX_K:
            raise ValueError(f"latent_dimensions = {k}: TCCA supports at most {ops.TCCA_MAX_K} latent dimensions")
        if len(dims) > ops.TCCA_MAX_VIEWS:
            raise ValueError(f"TCCA supports at most {ops.TCCA_MAX_VIEWS} views, got {len(dims)}")
        entries = int(np.prod(dims, dtype=np.int64))
        if entries > ops.TCCA_MAX_ENTRIES:
            raise ValueError(f"the cross-moment tensor of widths {list(dims)} has {entries} entries; TCCA supports at "
                             f"most 2^25 = {ops.TCCA_MAX_ENTRIES} (the product of the view widths)")
        for j, p in enumerate(dims):
            if entries // p < min(k, p):
                raise ValueError(f"the mode-{j} unfolding of the tensor ({p} x {entries // p}) has fewer than "
                                 f"min(latent_dimensions, {p}) = {min(k, p)} singular vectors for the SVD start")

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        self._validate_params()
        if parallel.is_distributed():
            raise NotImplementedError("TCCA has no sharded fit: the whiteners must be known before the contraction pass")
        validated = validate_views(views)
        dims = [int(v.shape[1]) for v in validated]
        self._check_limits(dims)
        k = int(self.latent_dimensions)
        c_ = [float(x) for x in perview_parameter("c", self.c, 0.0, len(dims))]
        device = self._device()
        dev_views = [self._to_device(v, device) for v in validated]
        if len({v.dtype for v in dev_views}) > 1:
            dev_views = [v.to(torch.float64) for v in dev_views]
        mom, n_local, dims, in_dtype = self._local_moments(dev_views, device)
        self._partial = None
        C, dims, n = self._covariance_stage(mom, n_local, dims, in_dtype, True)
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        S = [self._whitener(C[off[i]:off[i + 1], off[i]:off[i + 1]], c_[i]) for i in range(len(dims))]
        Z = [self._whitened(v, s, i) for i, (v, s) in enumerate(zip(dev_views, S))]
        M = ops.tcca_moment(Z)
        del Z
        rand = random_start_columns(dims, k, self.random_state)
        state = ops.tcca_fit(M, dims, k, ops.TCCA_MAX_ITER, rand=rand)
        lay = ops.tcca_layout(dims, k)
        W = torch.empty(int(off[-1]) * k, dtype=torch.float64, device=device)
        for i, s in enumerate(S):
            F = state[lay["F"][i]:lay["F"][i] + dims[i] * k].view(dims[i], k)
            ops.gemm(s, F, out=W[off[i] * k:off[i + 1] * k].view(dims[i], k))
        host = torch.cat([state, W]).cpu().numpy()              # the one copy back of the fit
        st = ops.decode_tcca_state(host[:lay["total"]], dims, k)
        if st["singular"]:
            raise np.linalg.LinAlgError("Singular matrix")
        Wh = host[lay["total"]:]
        self.weights_ = [Wh[off[i] * k:off[i + 1] * k].reshape(dims[i], k).copy() for i in range(len(dims))]
        self._fit_info = {"iters": st["iters"], "stop": st["stop"], "rec": st["rec"]}
        return self

    def _whitener(self, Cii, c):
        """V (lambda + floor)^-1/2 V^T from the eigendecomposition of the view's covariance block, with the
        reference's regularisation (1 - c) cov + c I and its floor: if lambda_min < eps, add eps - lambda_min."""
        lam, Vt = ops.syevj(Cii.contiguous())
        lam = lam * (1.0 - c) + c
        lmin = lam.min()
        lam = torch.where(lmin < self.eps, lam + (self.eps - lmin), lam)
        return ops.gemm(Vt, ops.scale(Vt, rows=lam, rows_pow=-0.5), transa=True)

    def _whitened(self, v, S, i):
        """Z_i = (X_i - mu_i) S_i in float64 (n x p_i): the mean term preloaded into the output (the caller's view is
        not modified; float32 views are upcast once)."""
        X = v if v.dtype == torch.float64 else v.to(torch.float64)
        if not self.center:
            return ops.gemm(X, S)
        mu = torch.from_numpy(np.asarray(self.means_[i], dtype=np.float64)).to(X.device).view(1, -1)
        Z = ops.gemm(mu, S, alpha=-1.0).expand(X.shape[0], -1).contiguous()
        return ops.gemm(X, S, beta=1.0, out=Z)

    def partial_fit(self, views, y=None, solve: bool = True):
        raise NotImplementedError("TCCA has no partial_fit: the whiteners must be known before the contraction pass")

    def _solve(self, C, dims, n_total):
        raise NotImplementedError("TCCA decomposes the cross-moment tensor in ccab_tcca_fit, not a solved covariance")
