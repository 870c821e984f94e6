"""KTCCA (kernel tensor CCA) on the GPU (mirrors cca_zoo/nonparametric/_ktcca.py).

The reference whitens every kernel matrix with invsqrt_i = inv(sqrtm((1 - c_i) K_i^2 + c_i K_i + s_i I)) (each floored
at eps on its own), builds the n x n x ... x n array of per-sample outer products of the rows of K_i invsqrt_i (one
n-wide mode per view plus the sample axis), averages it over the samples and runs tensorly's ``parafac``; weights_i =
invsqrt_i F_i.  In the eigenbasis K_i = V_i^T diag(lambda_i) V_i (V_i: the eigenvectors as rows) a fit here is:

  1. K_i = k_i(X_i, X_i) in float64 (``ccab_pairwise_kernel``) and lambda_i, V_i from ``syevj``, as in KCCA;
  2. the per-view floor on the host: f_i = c_i lambda + (1 - c_i) lambda^2, s_i = eps - min f_i if min f_i < eps,
     h_i = (f_i + s_i)^-1/2;
  3. Z_i = V_i^T diag(lambda_i h_i) V_i = K_i invsqrt_i, one DMMA GEMM per view;
  4. M = Z_1^T KR(Z_2, ..., Z_m) / n, the sample mean of the outer products, as one contraction (``ccab_tcca_moment``;
     like the reference, nothing is centred);
  5. tensorly's default CP-ALS on M (``ccab_tcca_fit``), its random start columns drawn on the host in tensorly's
     order, as TCCA does;
  6. weights_i = V_i^T diag(h_i) (V_i F_i), two thin GEMMs, copied back with the state block in one transfer
     (invsqrt_i is never formed).

``transform`` computes k_i(train_views_i, X) and, like the reference, does not centre the new views.  ``partial_fit``
and the sharded fit are not supported: every K_i needs all the rows.
"""
from __future__ import annotations

from numbers import Integral
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval

from .. import ops
from ..linear._tcca import random_start_columns
from ._kcca import _KernelModel, eigenbases, kernel_matrices


def tensor_scales(lams, c, eps: float):
    """Step 2 on the host, per view: (lambda_i h_i, h_i, min f_i)."""
    out = []
    for lam, ci in zip(lams, c):
        f = ci * lam + (1.0 - ci) * lam * lam
        fm = float(f.min())
        h = 1.0 / np.sqrt(f + (eps - fm if fm < eps else 0.0))
        out.append((lam * h, h, fm))
    return [o[0] for o in out], [o[1] for o in out], [o[2] for o in out]


class KTCCA(_KernelModel):
    r"""Kernel tensor CCA (cca_zoo/nonparametric/_ktcca.py): CP decomposition of the cross-moment tensor of the
    whitened kernel matrices, each whitened in its own eigenbasis.

    Same arguments, defaults and fitted attributes as the reference (``weights_`` -- float64 n x k per view --,
    ``train_views_`` -- the centred float64 training views, kept on the device --, ``means_``, ``n_views_``,
    ``n_features_in_``, ``n_samples_``), plus ``device``.  The iteration count and the reconstruction errors are in
    ``_fit_info``.  Limits: at most 8 views, ``latent_dimensions`` at most 64 and n^m <= 2^25 tensor entries (n <= 5792
    for two views, n <= 322 for three)."""

    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **_KernelModel._parameter_constraints,
        "random_state": [None, Interval(Integral, 0, None, closed="left")],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.1, kernel="linear", gamma=None,
                 degree=1.0, coef0=1.0, kernel_params=None, eps: float = 1e-3, random_state: int | None = None,
                 device=None) -> None:
        self.latent_dimensions = latent_dimensions
        self.center = center
        self.c = c
        self.kernel = kernel
        self.gamma = gamma
        self.degree = degree
        self.coef0 = coef0
        self.kernel_params = kernel_params
        self.eps = eps
        self.random_state = random_state
        self.device = device

    def _check_limits(self, m: int, n: int):
        k = int(self.latent_dimensions)
        if k > ops.TCCA_MAX_K:
            raise ValueError(f"latent_dimensions = {k}: KTCCA supports at most {ops.TCCA_MAX_K} latent dimensions")
        if m > ops.TCCA_MAX_VIEWS:
            raise ValueError(f"KTCCA supports at most {ops.TCCA_MAX_VIEWS} views, got {m}")
        entries = n ** m
        if entries > ops.TCCA_MAX_ENTRIES:
            raise ValueError(f"the cross-moment tensor of {m} views at n = {n} has n^{m} = {entries} entries; KTCCA "
                             f"supports at most 2^25 = {ops.TCCA_MAX_ENTRIES}")
        if entries // n < min(k, n):
            raise ValueError(f"the unfoldings of the tensor ({n} x {entries // n}) have fewer than "
                             f"min(latent_dimensions, {n}) = {min(k, n)} singular vectors for the SVD start")

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        X, c_, _, device = self._setup_kernel_fit(views)
        m, n = self.n_views_, self.n_samples_
        k = int(self.latent_dimensions)
        dims = [n] * m

        K, knorm = kernel_matrices(X, self._kernel_args)
        lams, V, sweeps = eigenbases(K, knorm)
        del K
        lam_h = torch.cat(lams).cpu().numpy()
        d, h, fmin = tensor_scales([lam_h[i * n:(i + 1) * n] for i in range(m)], c_, float(self.eps))
        Z = [ops.gemm(ops.scale(Vi, rows=torch.from_numpy(di).to(device)), Vi, transa=True) for Vi, di in zip(V, d)]
        M = ops.tcca_moment(Z)
        del Z
        state = ops.tcca_fit(M, dims, k, ops.TCCA_MAX_ITER, rand=random_start_columns(dims, k, self.random_state))
        lay = ops.tcca_layout(dims, k)
        W = torch.empty(m * n * k, dtype=torch.float64, device=device)
        for i, (Vi, hi) in enumerate(zip(V, h)):
            F = state[lay["F"][i]:lay["F"][i] + n * k].view(n, k)
            VF = ops.scale(ops.gemm(Vi, F), rows=torch.from_numpy(hi).to(device))
            ops.gemm(Vi, VF, transa=True, out=W[i * n * k:(i + 1) * n * k].view(n, k))
        host = torch.cat([state, W]).cpu().numpy()              # the one copy back of the fit
        st = ops.decode_tcca_state(host[:lay["total"]], dims, k)
        if st["singular"]:
            raise np.linalg.LinAlgError("Singular matrix")
        Wh = host[lay["total"]:]
        self.weights_ = [Wh[i * n * k:(i + 1) * n * k].reshape(n, k).copy() for i in range(m)]
        self._fit_info = {"iters": st["iters"], "stop": st["stop"], "rec": st["rec"], "kernel_sweeps": sweeps,
                          "fmin": fmin}
        return self
