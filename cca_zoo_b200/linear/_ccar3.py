"""CCAR3 (CCA by reduced-rank regression) on the GPU (mirrors cca_zoo/linear/_ccar3.py).

Every step of the reference's fit is a function of the 1/n block moments S (centred when ``center``, raw otherwise)
and of one more scalar:

  1. the moment pass (``_local_moments``, so badly centred columns are still accumulated shifted);
  2. with ``ledoit_wolf``, sklearn's shrinkage from Y's centred covariance S_c: mu = tr(S_c) / q, ||S_c||_F^2 and
     sum_s ||y_s - ybar||^4 (``ccab_row_norm4_sum``), giving Sy = (1 - s) S_c + s mu I; otherwise Sy = S_yy;
  3. Sy^-1/2 from one ``syevj`` with the reference's absolute cut (eigenvalues <= 1e-4 map to 0);
  4. M = (Sx + (rho + eps) I)^-1 (or (Sx + eps I)^-1 for ``highdim=False``) from ``potrf_inv``;
  5. B0 = M Sxy Sy^-1/2 (X^T Y~ / n = Sxy Sy^-1/2);
  6. ``highdim``: the row-sparse ADMM (``ccab_ccar3_admm``, one persistent kernel, no host synchronisation until it
     ends), which returns Z with its exact zero rows; otherwise B = B0;
  7. the SVD of B (``gesvj``), V0 = Sy^-1/2 Vt0[:r]^T;
  8. U0^T Sx U0, V0^T S_yy V0 and U0^T Sxy V0 on the device (S_yy the plain second moment, never the shrunk one).

The r x r tail (the whitening with its eigen fallback, the sign alignment and the sort) runs in float64 numpy after
the one copy back, line for line as in the reference.  Float32 views are read in float32 by the moment pass
(``precision``) and everything after it, the ADMM included, runs in float64, where the reference keeps float32 for
its products of the data: the same intended divergence as the ALS family.

``partial_fit`` and the sharded fit are not supported: the fourth-power sum of the Ledoit-Wolf term needs the global
mean before its pass.
"""
from __future__ import annotations

from numbers import Integral, Real
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval

from .. import ops, parallel
from .._base import BaseModel
from .._validation import validate_views

SQRT_INV_CUT = 1e-4       # cca_zoo/linear/_ccar3.py:_sqrt_inv_psd threshold (absolute)


def ledoit_wolf_shrinkage(fro2: float, trace: float, norm4: float, n: int, q: int):
    """(shrinkage, mu) of sklearn's ledoit_wolf_shrinkage from the centred 1/n covariance S_c of Y: its squared
    Frobenius norm, its trace and sum_s ||y_s - ybar||^4.  One column: no shrinkage, as in sklearn."""
    mu = trace / q
    if q == 1:
        return 0.0, mu
    beta = 1.0 / (q * n) * (norm4 / n - fro2)
    delta = (fro2 - 2.0 * mu * trace + q * mu ** 2) / q
    beta = min(beta, delta)
    return (0.0 if beta == 0 else beta / delta), mu


def whiten_factor(G, ridge):
    """W with W^T G W = I (cca_zoo/linear/_ccar3.py:_whiten_factor): inv(chol(sym(G) + ridge I))^T, or the eigen
    route with eigenvalues floored at ridge when the Cholesky fails."""
    p = G.shape[0]
    G = (G + G.T) / 2 + ridge * np.eye(p)
    try:
        L = np.linalg.cholesky(G)
        return np.asarray(np.linalg.inv(L).T)
    except np.linalg.LinAlgError:
        vals, vecs = np.linalg.eigh(G)
        vals = np.maximum(vals, ridge)
        return np.asarray((vecs * (1.0 / np.sqrt(vals))) @ vecs.T)


def rrr_tail(U0, V0, GX, GY, P, r, ridge):
    """Whitened, sign-aligned, sorted and padded weights from the thin products (cca_zoo/linear/_ccar3.py:101-125):
    U0 (p x r_eff), V0 (q x r_eff), GX = U0^T Sx U0, GY = V0^T S_yy V0, P = U0^T Sxy V0."""
    p, q, r_eff = U0.shape[0], V0.shape[0], U0.shape[1]
    Wx, Wy = whiten_factor(GX, ridge), whiten_factor(GY, ridge)
    U, V = U0 @ Wx, V0 @ Wy
    cor = np.diag(Wx.T @ P @ Wy).copy()
    neg = cor < 0
    V[:, neg] *= -1
    cor[neg] *= -1
    order = np.argsort(-cor)
    U, V = U[:, order], V[:, order]
    if r_eff < r:
        U = np.hstack([U, np.zeros((p, r - r_eff))])
        V = np.hstack([V, np.zeros((q, r - r_eff))])
    return U, V


class CCAR3(BaseModel):
    r"""CCA via reduced-rank regression (cca_zoo/linear/_ccar3.py), with the row-group-lasso ADMM on the device.

    Same arguments, defaults and fitted attributes as the reference (``weights_`` -- always float64 --, ``means_``,
    ``n_views_``, ``n_features_in_``, ``n_samples_``), plus ``precision`` (arithmetic of the moment pass for float32
    views) and ``device``.  Exactly two views.  Limits: at most 16384 features in X (M is p x p float64) and, for
    ``highdim=True``, at most 512 in Y.  The route (``admm`` / ``closed_form``), the ADMM iterations and final
    residuals, the Ledoit-Wolf shrinkage and the effective rank are in ``_fit_info``."""

    _solve_in_float64 = True
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "lambda_": [Interval(Real, 0, None, closed="left")],
        "highdim": ["boolean"],
        "ledoit_wolf": ["boolean"],
        "rho": [Interval(Real, 0, None, closed="neither")],
        "max_iter": [Interval(Integral, 1, None, closed="left")],
        "tol": [Interval(Real, 0, None, closed="neither")],
        "eps": [Interval(Real, 0, None, closed="neither")],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, lambda_: float = 0.0, highdim: bool = True,
                 ledoit_wolf: bool = True, rho: float = 1.0, max_iter: int = 10_000, tol: float = 1e-4,
                 eps: float = 1e-8, precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.lambda_ = lambda_
        self.highdim = highdim
        self.ledoit_wolf = ledoit_wolf
        self.rho = rho
        self.max_iter = max_iter
        self.tol = tol
        self.eps = eps

    def _check_limits(self, dims):
        p, q = dims
        if p > ops.CCAR3_MAX_P:
            raise ValueError(f"X has {p} features; CCAR3 supports at most {ops.CCAR3_MAX_P} (M = (Sx + (rho + eps) "
                             f"I)^-1 is p x p float64)")
        if self.highdim and q > ops.CCAR3_MAX_Q:
            raise ValueError(f"Y has {q} features; the CCAR3 ADMM (highdim=True) supports at most {ops.CCAR3_MAX_Q}")

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        self._validate_params()
        if parallel.is_distributed():
            raise NotImplementedError("CCAR3 has no sharded fit: the Ledoit-Wolf term needs the global mean before "
                                      "its pass over Y")
        validated = validate_views(views)
        if len(validated) != 2:
            raise ValueError(f"CCAR3 requires exactly 2 views, got {len(validated)}. Use MCCA for more than 2 views.")
        dims = [int(v.shape[1]) for v in validated]
        self._check_limits(dims)
        k = int(self.latent_dimensions)
        device = self._device()
        dev_views = [self._to_device(v, device) for v in validated]
        if len({v.dtype for v in dev_views}) > 1:
            dev_views = [v.to(torch.float64) for v in dev_views]
        mom, n_local, dims, in_dtype = self._local_moments(dev_views, device)
        self._partial = None
        C, dims, n = self._covariance_stage(mom, n_local, dims, in_dtype, True)
        p, q = dims
        S = C * ((n - 1) / n)                                   # the 1/n moments of the reference
        Sx, Sxy, Syy = S[:p, :p], S[:p, p:], S[p:, p:]

        shrinkage = None
        if self.ledoit_wolf:
            Cc, mean = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
            Sc = (Cc[p:, p:] * ((n - 1) / n)).contiguous()
            norm4 = ops.row_norm4_sum(dev_views[1], mean[p:])
            h = torch.cat([ops.frobenius_norm(Sc), norm4, Sc.diagonal()]).cpu().numpy()
            shrinkage, mu = ledoit_wolf_shrinkage(float(h[0]) ** 2, float(h[2:].sum()), float(h[1]), n, q)
            Sy = Sc * (1.0 - shrinkage)
            Sy.diagonal().add_(shrinkage * mu)
        else:
            Sy = Syy.contiguous()
        lam, Vt = ops.syevj(Sy)
        f = torch.where(lam > SQRT_INV_CUT, lam.abs().rsqrt(), torch.zeros_like(lam))
        Sinv = ops.gemm(Vt, ops.scale(Vt, rows=f), transa=True)      # Sy^-1/2
        R = ops.gemm(Sxy, Sinv)                                        # X^T Y~ / n

        ridge = (self.rho + self.eps) if self.highdim else self.eps
        A = Sx.contiguous().clone()
        A.diagonal().add_(ridge)
        Linv, pinfo = ops.potrf_inv_(A)
        Minv = ops.gemm(Linv, Linv, transa=True)
        B0 = ops.gemm(Minv, R)
        if self.highdim:
            B, _, admm = ops.ccar3_admm(Minv, B0, self.lambda_ / self.rho, self.rho, self.tol, self.max_iter)
        else:
            B, admm = B0, torch.zeros(4, dtype=torch.float64, device=B0.device)
        h = torch.cat([admm, ops.frobenius_norm(B), pinfo.to(torch.float64).to(B.device)]).cpu().numpy()
        if h[5] != 0:
            raise np.linalg.LinAlgError(f"Sx + {ridge:g} I is not numerically positive definite")
        r_eff = min(k, p, q)
        self._fit_info = {"route": "admm" if self.highdim else "closed_form", "iters": int(h[0]),
                          "primal": float(h[1]), "dual": float(h[2]), "stopped": bool(h[3]), "shrinkage": shrinkage,
                          "r_eff": r_eff}
        if h[4] == 0:
            self.weights_ = [np.zeros((p, k)), np.zeros((q, k))]
            return self

        if p >= q:
            _, Vt0, U0t = ops.gesvj(B.T.contiguous())     # G = B: right vectors = rows of Vt0, left = rows of U0^T
        else:
            _, U0t, Vt0 = ops.gesvj(B)                    # G = B^T: the roles swap
        U0t, Vt0 = U0t[:r_eff].contiguous(), Vt0[:r_eff].contiguous()
        V0 = ops.gemm(Sinv, Vt0, transb=True)                           # q x r
        GX = ops.gemm(U0t, ops.gemm(Sx, U0t, transb=True))
        GY = ops.gemm(V0, ops.gemm(Syy, V0), transa=True)
        P = ops.gemm(U0t, ops.gemm(Sxy, V0))
        parts = [U0t, V0, GX, GY, P]
        host = torch.cat([t.reshape(-1) for t in parts]).cpu().numpy()
        at, out = 0, []
        for t in parts:
            out.append(host[at:at + t.numel()].reshape(tuple(t.shape)))
            at += t.numel()
        U0t_h, V0_h, GX_h, GY_h, P_h = out
        U, V = rrr_tail(U0t_h.T, V0_h, GX_h, GY_h, P_h, k, self.eps)
        self.weights_ = [np.ascontiguousarray(U), np.ascontiguousarray(V)]
        return self

    def partial_fit(self, views, y=None, solve: bool = True):
        raise NotImplementedError("CCAR3 has no partial_fit: the Ledoit-Wolf term needs the global mean before its "
                                  "pass over Y")

    def _solve(self, C, dims, n_total):
        raise NotImplementedError("CCAR3 solves its reduced-rank regression from the moments in fit")
