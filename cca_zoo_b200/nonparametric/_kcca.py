"""KCCA (kernel CCA) on the GPU (mirrors cca_zoo/nonparametric/_kcca.py).

The reference builds the m kernel matrices K_i (n x n), the (m n)^2 matrix A = (cov(hstack K) - blockdiag cov K_i) / m
with np.cov, B = blockdiag(c_i K_i + (1 - c_i) K_i^2) floored at eps, and solves the generalised eigenproblem (A, B) of
order m n.  B_i is a polynomial in K_i, so in the eigenbasis K_i = U_i diag(lambda_i) U_i^T the whole problem whitens
without forming A, B or K_i^2.  A fit here is:

  1. K_i = k_i(X_i, X_i) in float64 (``ccab_pairwise_kernel``: DMMA tiles for the inner-product metrics, FMA tiles for
     the distance metrics); float32 views are upcast once;
  2. lambda_i, U_i from ``syevj`` with the shift ||K_i||_inf (kernels may be indefinite);
  3. the reference's floor on the host from the eigenvalues alone: f_i = c_i lambda + (1 - c_i) lambda^2,
     s = eps - min f if min f < eps, beta_i = (f_i + s) / m;
  4. D_i = lambda_i beta_i^-1/2 / sqrt(m (n - 1)); columns with |D| <= n eps_mach max|D| are dropped (they only carry
     rounding noise into A);
  5. T_ij = D_i (U_i^T U_j - (U_i^T 1)(U_j^T 1)^T / n) D_j for i != j (the centring term preloaded into the GEMM),
     T_ii = 0;
  6. the top-k eigenvectors Y of T from ``syevj`` with the shift ||T||_inf;
  7. weights_i = U_i diag(beta_i^-1/2) Y_i, which gives v^T (B / m) v = 1 as the reference's ``eigh`` does.

``transform`` computes k_i(train_views_i, X) with the same kernel and, like the reference, does not centre the new
views.  ``partial_fit`` and the sharded fit are not supported: every K_i needs all the rows.
"""
from __future__ import annotations

from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils.validation import check_is_fitted

from .. import ops, parallel
from .._base import BaseModel
from .._validation import perview_parameter, validate_views

#: sklearn.metrics.pairwise.KERNEL_PARAMS: the parameters each metric takes (``filter_params=True`` drops the rest)
KERNEL_PARAMS = {"additive_chi2": (), "chi2": ("gamma",), "cosine": (), "linear": (),
                 "poly": ("gamma", "degree", "coef0"), "polynomial": ("gamma", "degree", "coef0"), "rbf": ("gamma",),
                 "laplacian": ("gamma",), "sigmoid": ("gamma", "coef0")}
#: metrics whose sklearn function resolves gamma=None to 1 / n_features
_GAMMA_DEFAULT = ("poly", "polynomial", "rbf", "laplacian", "sigmoid")


def kernel_arguments(kernel, gamma, degree, coef0, kernel_params, n_features: int):
    """(metric, gamma, degree, coef0) as ``pairwise_kernels(..., filter_params=True, **kernel_params)`` resolves them
    for one view.  A ``kernel_params`` key that duplicates gamma, degree or coef0 raises the reference's TypeError;
    other keys are dropped, as ``filter_params`` drops them (no metric takes any other parameter)."""
    if callable(kernel) or not isinstance(kernel, str) or kernel not in KERNEL_PARAMS:
        raise ValueError(f"kernel {kernel!r} is not supported: KCCA computes the kernels {sorted(KERNEL_PARAMS)} "
                         "(callables and 'precomputed' are not supported)")
    for key in ("gamma", "degree", "coef0"):
        if key in (kernel_params or {}):
            raise TypeError(f"sklearn.metrics.pairwise.pairwise_kernels() got multiple values for keyword argument "
                            f"'{key}'")
    takes = KERNEL_PARAMS[kernel]
    if "gamma" in takes and gamma is None:
        if kernel not in _GAMMA_DEFAULT:       # chi2_kernel multiplies by gamma: None fails in numpy (a TypeError)
            raise TypeError(f"the {kernel!r} kernel needs a numeric gamma, got None")
        gamma = 1.0 / n_features
    return (kernel, float(gamma) if "gamma" in takes else 1.0, float(degree) if "degree" in takes else 1.0,
            float(coef0) if "coef0" in takes else 1.0)


def eigenbasis_scales(lams, c, eps: float, n: int):
    """Steps 3 and 4 on the host: per view (beta, D, keep) from the eigenvalues ``lams`` of the kernel matrices."""
    m = len(lams)
    f = [ci * lam + (1.0 - ci) * lam * lam for ci, lam in zip(c, lams)]
    fmin = min(float(x.min()) for x in f)
    s = eps - fmin if fmin < eps else 0.0
    beta = [(x + s) / m for x in f]
    D = [lam / np.sqrt(b) / np.sqrt(m * (n - 1.0)) for lam, b in zip(lams, beta)]
    cut = n * np.finfo(np.float64).eps * max(float(np.abs(x).max()) for x in D)
    return beta, D, [np.abs(x) > cut for x in D]


def kernel_matrices(X, args):
    """Step 1: the kernel matrices of the (centred, float64) views and their inf-norms, read back once.  A kernel
    matrix with a non-finite entry raises numpy's LinAlgError, as the reference's eigvalsh of B does."""
    K = [ops.pairwise_kernel(x, None, *a) for x, a in zip(X, args)]
    knorm = torch.stack([Ki.abs().sum(dim=1).max() for Ki in K]).cpu().numpy()
    for i, v in enumerate(knorm):
        if not np.isfinite(v):
            raise np.linalg.LinAlgError(f"Eigenvalues did not converge: the kernel matrix of view {i} ({args[i][0]}) "
                                        "has non-finite entries")
    return K, knorm


def _syevj(A, shift, what):
    lam, evt, info = ops.syevj(A, shift=float(shift), return_info=True)
    if not info["converged"]:
        raise np.linalg.LinAlgError(f"the eigensolver of {what} did not converge in {info['sweeps']} sweeps")
    return lam, evt, info["sweeps"]


def eigenbases(K, knorm):
    """Step 2: (eigenvalues, eigenvectors as rows, sweeps) of every kernel matrix, shifted by its inf-norm."""
    out = [_syevj(Ki, s, "a kernel matrix") for Ki, s in zip(K, knorm)]
    return [o[0] for o in out], [o[1] for o in out], [o[2] for o in out]


def whitened_matrix(Uk, dk):
    """Step 5: T (R x R) from the kept eigenvectors ``Uk`` (rows, r_i x n) and the column scales ``dk``."""
    n, r = int(Uk[0].shape[1]), [int(u.shape[0]) for u in Uk]
    off = np.concatenate([[0], np.cumsum(r)]).astype(int)
    ones = torch.ones((n, 1), dtype=torch.float64, device=Uk[0].device)
    s1 = [ops.gemm(u, ones) for u in Uk]                                   # U_i^T 1  (r_i x 1)
    T = torch.zeros((int(off[-1]), int(off[-1])), dtype=torch.float64, device=Uk[0].device)
    for i in range(len(Uk)):
        for j in range(i + 1, len(Uk)):
            blk = T[off[i]:off[i + 1], off[j]:off[j + 1]]
            ops.gemm(s1[i], s1[j], transb=True, alpha=-1.0 / n, out=blk)   # the centring term, preloaded
            ops.gemm(Uk[i], Uk[j], transb=True, beta=1.0, out=blk)
            ops.scale(blk, rows=dk[i], cols=dk[j], out=blk)
            T[off[j]:off[j + 1], off[i]:off[i + 1]].copy_(blk.T)
    return T


def top_eigenvectors(T):
    """Step 6: the eigenvectors of T as rows, descending, from syevj shifted by ||T||_inf; and the sweeps."""
    _, Yt, sweeps = _syevj(T, float(T.abs().sum(dim=1).max().item()), "the whitened kernel matrix")
    return Yt, sweeps


class _KernelModel(BaseModel):
    """The part KCCA, KGCCA and KTCCA share: the fit preamble (parameters, limits, per-view kernel arguments, the
    device upload, centring) and the kernel-space methods (``transform`` and ``pairwise_correlations`` evaluate the
    kernel against ``train_views_``).  ``partial_fit`` and the sharded fit are refused: every kernel matrix needs all
    the rows."""

    _solve_in_float64 = True
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = dict(BaseModel._parameter_constraints)   # none of its own

    def _check_limits(self, m: int, n: int):
        raise NotImplementedError

    def _setup_kernel_fit(self, views, extra=()):
        """Validate, upload and centre the views; set ``means_``, ``train_views_``, ``n_views_``, ``n_features_in_``,
        ``n_samples_`` and the resolved kernel arguments.  ``extra`` names further per-view parameters as (name,
        value, default).  Returns (float64 device views, per-view c, the per-view ``extra`` lists, device).  Every
        parameter and limit error is raised before anything is uploaded."""
        self._validate_params()
        if parallel.is_distributed():
            raise NotImplementedError(f"{type(self).__name__} has no sharded fit: every kernel matrix needs all the rows")
        validated = validate_views(views)
        m, n = len(validated), int(validated[0].shape[0])
        dims = [int(v.shape[1]) for v in validated]
        self._check_limits(m, n)
        c_ = [float(x) for x in perview_parameter("c", self.c, 0.1, m)]
        kernel_ = perview_parameter("kernel", self.kernel, "linear", m)
        gamma_ = perview_parameter("gamma", self.gamma, None, m)
        degree_ = perview_parameter("degree", self.degree, 1.0, m)
        coef0_ = perview_parameter("coef0", self.coef0, 1.0, m)
        kp_ = perview_parameter("kernel_params", self.kernel_params, {}, m)
        args = [kernel_arguments(kernel_[i], gamma_[i], degree_[i], coef0_[i], kp_[i], dims[i]) for i in range(m)]
        extra_ = [perview_parameter(name, value, default, m) for name, value, default in extra]
        device = self._device()

        X = [self._to_device(v, device).to(torch.float64) for v in validated]
        if any(isinstance(v, torch.Tensor) for v in validated):
            if not bool(torch.stack([torch.isfinite(x).all() for x in X]).all().item()):
                raise ValueError("Input contains NaN or infinity.")
        if self.center:
            mu = [ops.column_sums(x) / n for x in X]
            X = [x - u.view(1, -1) for x, u in zip(X, mu)]
            means = torch.cat(mu).cpu().numpy()
            off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
            self.means_ = [means[off[i]:off[i + 1]].copy() for i in range(m)]
        else:
            X = [x.clone() for x in X]                  # train_views_ never aliases the caller's tensors
            self.means_ = [np.zeros(p) for p in dims]
        self.n_views_, self.n_features_in_, self.n_samples_ = m, dims, n
        self.train_views_ = X
        self._kernel_args = args
        return X, c_, extra_, device

    # ------------------------------------------------------------------ kernel transform
    def transform(self, views):
        """k_i(train_views_i, X_i)^T weights_i per view; the new views are not centred (as in the reference)."""
        check_is_fitted(self)
        validated = validate_views(views)
        device = self.train_views_[0].device
        out = []
        for i, v in enumerate(validated):
            Xt = self._to_device(v, device).to(torch.float64)
            Kt = ops.pairwise_kernel(self.train_views_[i], Xt, *self._kernel_args[i])     # n_train x n_test
            W = torch.from_numpy(np.ascontiguousarray(self.weights_[i])).to(device)
            out.append(ops.gemm(Kt, W, transa=True).cpu().numpy())
        return out

    def pairwise_correlations(self, views):
        """(n_views, n_views, k) Pearson correlations of the kernel variates (cca_zoo/_base.py:153-174)."""
        T = np.stack(self.transform(views), axis=0)
        T = T - T.mean(axis=1, keepdims=True)
        norms = np.sqrt((T**2).sum(axis=1, keepdims=True))
        T_norm = T / np.where(norms > 1e-12, norms, 1.0)
        return np.einsum("isd,jsd->ijd", T_norm, T_norm)

    def partial_fit(self, views, y=None, solve: bool = True):
        raise NotImplementedError(f"{type(self).__name__} has no partial_fit: every kernel matrix needs all the rows")

    def _solve(self, C, dims, n_total):
        raise NotImplementedError(f"{type(self).__name__} solves its kernel eigenproblem in fit, not from a block "
                                  "covariance")


class KCCA(_KernelModel):
    r"""Kernel CCA (cca_zoo/nonparametric/_kcca.py), solved in the eigenbasis of each kernel matrix.

    Same arguments, defaults and fitted attributes as the reference (``weights_`` -- float64 n x k per view --,
    ``train_views_`` -- the centred float64 training views, kept on the device --, ``means_``, ``n_views_``,
    ``n_features_in_``, ``n_samples_``), plus ``device``.  Kernels: the metric names of sklearn's
    ``PAIRWISE_KERNEL_FUNCTIONS``.  Limits: at most 8 views, n <= 8192 and m n <= 16384."""

    def __init__(self, latent_dimensions: int = 1, center: bool = True, c=0.1, kernel="linear", gamma=None,
                 degree=1.0, coef0=1.0, kernel_params=None, eps: float = 1e-3, device=None) -> None:
        self.latent_dimensions = latent_dimensions
        self.center = center
        self.c = c
        self.kernel = kernel
        self.gamma = gamma
        self.degree = degree
        self.coef0 = coef0
        self.kernel_params = kernel_params
        self.eps = eps
        self.device = device

    def _check_limits(self, m: int, n: int):
        if m > ops.KCCA_MAX_VIEWS:
            raise ValueError(f"KCCA supports at most {ops.KCCA_MAX_VIEWS} views, got {m}")
        if n > ops.KCCA_MAX_SAMPLES:
            raise ValueError(f"KCCA supports at most n = {ops.KCCA_MAX_SAMPLES} samples (each kernel matrix is n x n), "
                             f"got n = {n}")
        if m * n > ops.KCCA_MAX_ORDER:
            raise ValueError(f"KCCA supports n_views * n_samples <= {ops.KCCA_MAX_ORDER} (the order of the "
                             f"eigenproblem), got {m} * {n} = {m * n}")

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        X, c_, _, device = self._setup_kernel_fit(views)
        m, n = self.n_views_, self.n_samples_
        k = min(int(self.latent_dimensions), m * n)

        K, knorm = kernel_matrices(X, self._kernel_args)
        lams, U, sweeps = eigenbases(K, knorm)
        del K
        lam_h = torch.cat(lams).cpu().numpy()
        beta, D, keep = eigenbasis_scales([lam_h[i * n:(i + 1) * n] for i in range(m)], c_, float(self.eps), n)
        idx = [np.flatnonzero(kp) for kp in keep]
        r = [len(ix) for ix in idx]
        if k > sum(r):
            raise ValueError(f"latent_dimensions = {k} exceeds the {sum(r)} kernel eigendirections that carry signal "
                             f"(per view {r})")
        Uk = [u.index_select(0, torch.from_numpy(ix).to(device)) for u, ix in zip(U, idx)]   # r_i x n, rows
        del U
        dk = [torch.from_numpy(np.ascontiguousarray(Di[ix])).to(device) for Di, ix in zip(D, idx)]
        bk = [torch.from_numpy(np.ascontiguousarray(b[ix])).to(device) for b, ix in zip(beta, idx)]
        T = whitened_matrix(Uk, dk)
        Yt, top_sweeps = top_eigenvectors(T)
        del T
        off = np.concatenate([[0], np.cumsum(r)]).astype(int)
        Y = Yt[:k].T.contiguous()                                             # R x k
        W = torch.empty((m * n, k), dtype=torch.float64, device=device)
        for i in range(m):
            ops.gemm(ops.scale(Uk[i], rows=bk[i], rows_pow=-0.5), Y[off[i]:off[i + 1]], transa=True,
                     out=W[i * n:(i + 1) * n])
        Wh = W.cpu().numpy()                                                   # the one copy back of the weights
        self.weights_ = [Wh[i * n:(i + 1) * n].copy() for i in range(m)]
        self._fit_info = {"kernel_sweeps": sweeps, "sweeps": top_sweeps, "ranks": r}
        return self
