"""KGCCA (kernel generalised CCA) on the GPU (mirrors cca_zoo/nonparametric/_kgcca.py).

The reference builds Q = sum_i mu_i K_i (c_i K_i + (1 - c_i) K_i^2 + s_i I)^-1 K_i (n x n), with each B_i floored at
eps on its own, takes the top-k eigenvectors T of Q and returns weights_i = pinv(K_i) T.  Every term of Q is a function
of K_i, so in the eigenbasis K_i = V_i^T diag(lambda_i) V_i (V_i: the eigenvectors as rows) a fit here is:

  1. K_i = k_i(X_i, X_i) in float64 (``ccab_pairwise_kernel``) and lambda_i, V_i from ``syevj``, as in KCCA;
  2. the per-view floor on the host: f_i = c_i lambda + (1 - c_i) lambda^2, s_i = eps - min f_i if min f_i < eps;
  3. Q = sum_i mu_i V_i^T diag(lambda_i^2 / (f_i + s_i)) V_i, m DMMA GEMMs accumulating into one n x n matrix (K_i^2
     and B_i^-1 are never formed);
  4. the top-k eigenvectors T of Q from ``syevj`` with the shift ||Q||_inf (k clamped to n);
  5. weights_i = V_i^T diag(lambda_i^+) (V_i T), with lambda^+ = 1 / lambda where |lambda| > n eps_mach max|lambda_i|
     and 0 elsewhere: the minimum-norm solution.  numpy's pinv cuts at 1e-15 sigma_max and so inverts noise-level
     eigenvalues of a rank-deficient K_i; its weights carry that noise in K_i's null space (DESIGN.md §2a).

``transform`` computes k_i(train_views_i, X) and, like the reference, does not centre the new views.  ``partial_fit``
and the sharded fit are not supported: every K_i needs all the rows.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from ._kcca import _KernelModel, _syevj, eigenbases, kernel_matrices


def gcca_scales(lams, c, mu, eps: float, n: int):
    """Steps 2 and 5 on the host, per view: (mu_i lambda^2 / (f_i + s_i), lambda^+, min f_i)."""
    g, pinv, fmin = [], [], []
    for lam, ci, mi in zip(lams, c, mu):
        f = ci * lam + (1.0 - ci) * lam * lam
        fm = float(f.min())
        s = eps - fm if fm < eps else 0.0
        g.append(mi * lam * lam / (f + s))
        keep = np.abs(lam) > n * np.finfo(np.float64).eps * float(np.abs(lam).max())
        pinv.append(np.where(keep, 1.0 / np.where(keep, lam, 1.0), 0.0))
        fmin.append(fm)
    return g, pinv, fmin


class KGCCA(_KernelModel):
    r"""Kernel generalised CCA (cca_zoo/nonparametric/_kgcca.py), solved in the eigenbasis of each kernel matrix.

    Same arguments, defaults and fitted attributes as the reference (``weights_`` -- float64 n x k per view --,
    ``train_views_`` -- the centred float64 training views, kept on the device --, ``means_``, ``n_views_``,
    ``n_features_in_``, ``n_samples_``), plus ``device``.  ``weights_`` are the minimum-norm dual coefficients (a clean
    pseudo-inverse of each kernel matrix).  Limits: at most 8 views and n <= 8192."""

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.1, kernel="linear", gamma=None,
                 degree=1.0, coef0=1.0, kernel_params=None, view_weights=None, eps: float = 1e-6,
                 device=None) -> None:
        self.latent_dimensions = latent_dimensions
        self.center = center
        self.c = c
        self.kernel = kernel
        self.gamma = gamma
        self.degree = degree
        self.coef0 = coef0
        self.kernel_params = kernel_params
        self.view_weights = view_weights
        self.eps = eps
        self.device = device

    def _check_limits(self, m: int, n: int):
        if m > ops.KCCA_MAX_VIEWS:
            raise ValueError(f"KGCCA supports at most {ops.KCCA_MAX_VIEWS} views, got {m}")
        if n > ops.KCCA_MAX_SAMPLES:
            raise ValueError(f"KGCCA supports at most n = {ops.KCCA_MAX_SAMPLES} samples (each kernel matrix is "
                             f"n x n), got n = {n}")

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        X, c_, (mu,), device = self._setup_kernel_fit(views, [("view_weights", self.view_weights, 1.0)])
        m, n = self.n_views_, self.n_samples_
        mu = [float(x) for x in mu]
        k = min(int(self.latent_dimensions), n)

        K, knorm = kernel_matrices(X, self._kernel_args)
        lams, V, sweeps = eigenbases(K, knorm)
        del K
        lam_h = torch.cat(lams).cpu().numpy()
        g, pinv, fmin = gcca_scales([lam_h[i * n:(i + 1) * n] for i in range(m)], c_, mu, float(self.eps), n)
        Q = torch.zeros((n, n), dtype=torch.float64, device=device)
        for Vi, gi in zip(V, g):
            ops.gemm(ops.scale(Vi, rows=torch.from_numpy(gi).to(device)), Vi, transa=True, beta=1.0, out=Q)
        _, Tt, q_sweeps = _syevj(Q, float(Q.abs().sum(dim=1).max().item()), "the kernel GCCA matrix Q")
        del Q
        Tt = Tt[:k]                                                            # k x n, rows
        W = torch.empty((m * n, k), dtype=torch.float64, device=device)
        for i, (Vi, pi) in enumerate(zip(V, pinv)):
            VT = ops.scale(ops.gemm(Vi, Tt, transb=True), rows=torch.from_numpy(pi).to(device))
            ops.gemm(Vi, VT, transa=True, out=W[i * n:(i + 1) * n])
        Wh = W.cpu().numpy()                                                   # the one copy back of the weights
        self.weights_ = [Wh[i * n:(i + 1) * n].copy() for i in range(m)]
        self._fit_info = {"kernel_sweeps": sweeps, "sweeps": q_sweeps, "fmin": fmin}
        return self
