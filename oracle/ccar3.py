"""CCAR3 restated in float64 numpy (TEST INFRASTRUCTURE ONLY): the reference's data-space fit
(cca_zoo/linear/_ccar3.py) and, step for step, the moment form that cca_zoo_b200.linear.CCAR3 runs on the device,
including the inverse-form ADMM of ccab_ccar3_admm.  Neither needs the reference tree or sklearn's LedoitWolf."""
from __future__ import annotations

import numpy as np

from cca_zoo_b200.linear._ccar3 import SQRT_INV_CUT, ledoit_wolf_shrinkage, rrr_tail, whiten_factor


def sqrt_inv_psd(S, threshold=SQRT_INV_CUT):
    vals, vecs = np.linalg.eigh(S)
    f = np.where(vals > threshold, 1.0 / np.sqrt(np.abs(vals)), 0.0)
    return (vecs * f) @ vecs.T


def ledoit_wolf_data(Y):
    """sklearn's LedoitWolf().fit(Y).covariance_ in data space (Y centred first; one column: no shrinkage)."""
    n, q = Y.shape
    X = Y - Y.mean(axis=0)
    S = X.T @ X / n
    if q == 1:
        return S, 0.0
    X2 = X ** 2
    mu = np.trace(S) / q
    beta_ = np.sum(X2.T @ X2)
    delta_ = np.sum(S ** 2)
    beta = 1.0 / (q * n) * (beta_ / n - delta_)
    delta = (delta_ - 2.0 * mu * np.trace(S) + q * mu ** 2) / q
    beta = min(beta, delta)
    s = 0.0 if beta == 0 else beta / delta
    out = (1 - s) * S
    out.flat[::q + 1] += s * mu
    return out, s


def admm_ref(X, Yt, lam, rho, max_iter, tol, ridge, trace=None):
    """_admm_row_sparse_rrr in data space (two triangular solves of order p per iteration)."""
    n, p = X.shape
    Sx = X.T @ X / n
    L = np.linalg.cholesky(Sx + (rho + ridge) * np.eye(p))
    prod = X.T @ Yt / n
    U = np.zeros_like(prod)
    Z = np.zeros_like(prod)
    it = 0
    for it in range(1, max_iter + 1):
        B = np.linalg.solve(L.T, np.linalg.solve(L, prod + rho * (Z - U)))
        Z_old = Z
        Z = B + U
        nrm = np.linalg.norm(Z, axis=1)
        s = np.zeros_like(nrm)
        nz = nrm > 0
        s[nz] = np.maximum(0.0, 1.0 - (lam / rho) / nrm[nz])
        Z = Z * s[:, None]
        U = U + B - Z
        primal = np.linalg.norm(Z - B) / np.sqrt(p)
        dual = np.linalg.norm(Z_old - Z) / np.sqrt(p)
        if trace is not None:
            trace.append(dict(primal=primal, dual=dual, rownorm=nrm))
        if max(primal, dual) < tol:
            break
    return Z, it


def admm_inverse(M, B0, kappa, rho, tol, max_iter, trace=None):
    """The inverse form ccab_ccar3_admm runs: B = B0 + rho M (Z - U).  Returns (Z, U, iterations, primal, dual,
    stopped); ``trace`` (a list) receives every iteration's residuals and the row norms of B + U."""
    p = B0.shape[0]
    Z = np.zeros_like(B0)
    U = np.zeros_like(B0)
    primal = dual = 0.0
    stopped = False
    it = 0
    while it < max_iter:
        B = B0 + rho * (M @ (Z - U))
        Z_old = Z
        Zn = B + U
        nrm = np.linalg.norm(Zn, axis=1)
        s = np.where(nrm > 0, np.maximum(0.0, 1.0 - kappa / np.where(nrm > 0, nrm, 1.0)), 0.0)
        Z = Zn * s[:, None]
        U = U + B - Z
        primal = np.linalg.norm(Z - B) / np.sqrt(p)
        dual = np.linalg.norm(Z_old - Z) / np.sqrt(p)
        it += 1
        if trace is not None:
            trace.append(dict(primal=primal, dual=dual, rownorm=nrm))
        if max(primal, dual) < tol:
            stopped = True
            break
    return Z, U, it, primal, dual, stopped


def ref_ccar3_fit(views, k=1, center=True, lambda_=0.0, highdim=True, ledoit_wolf=True, rho=1.0, max_iter=10_000,
                  tol=1e-4, eps=1e-8, info=None):
    """The reference's fit in data space.  Returns (weights, means)."""
    X, Y = [np.asarray(v, dtype=np.float64) for v in views]
    means = [X.mean(axis=0), Y.mean(axis=0)]
    if center:
        X, Y = X - means[0], Y - means[1]
    n, p = X.shape
    q = Y.shape[1]
    Sy = ledoit_wolf_data(Y)[0] if ledoit_wolf else Y.T @ Y / n
    Si = sqrt_inv_psd(Sy)
    Yt = Y @ Si
    if highdim:
        B, it = admm_ref(X, Yt, lambda_, rho, max_iter, tol, eps)
    else:
        B, it = np.linalg.solve(X.T @ X / n + eps * np.eye(p), X.T @ Yt / n), 0
    if info is not None:
        info["iters"] = it
    if not np.any(B):
        return [np.zeros((p, k)), np.zeros((q, k))], means
    r = min(k, p, q)
    U0, _, Vt0 = np.linalg.svd(B, full_matrices=False)
    U0 = U0[:, :r]
    V0 = Si @ Vt0[:r].T
    XU0, YV0 = X @ U0, Y @ V0
    U, V = rrr_tail(U0, V0, XU0.T @ XU0 / n, YV0.T @ YV0 / n, XU0.T @ YV0 / n, k, eps)
    return [U, V], means


def moment_ccar3_fit(views, k=1, center=True, lambda_=0.0, highdim=True, ledoit_wolf=True, rho=1.0, max_iter=10_000,
                     tol=1e-4, eps=1e-8, info=None):
    """The device algorithm from the 1/n block moments.  Returns (weights, means); ``info`` receives iterations,
    residuals, the stop flag, the shrinkage, r_eff and the ADMM trace."""
    X, Y = [np.asarray(v, dtype=np.float64) for v in views]
    n, p = X.shape
    q = Y.shape[1]
    means = [X.mean(axis=0), Y.mean(axis=0)]
    D = np.hstack([X - means[0], Y - means[1]]) if center else np.hstack([X, Y])
    S = D.T @ D / n
    Sx, Sxy, Syy = S[:p, :p], S[:p, p:], S[p:, p:]
    shrink = None
    if ledoit_wolf:
        Yc = Y - means[1]
        Sc = Yc.T @ Yc / n
        norm4 = float(np.sum(np.sum(Yc ** 2, axis=1) ** 2))
        shrink, mu = ledoit_wolf_shrinkage(float(np.sum(Sc ** 2)), float(np.trace(Sc)), norm4, n, q)
        Sy = Sc * (1 - shrink) + shrink * mu * np.eye(q)
    else:
        Sy = Syy
    Si = sqrt_inv_psd(Sy)
    R = Sxy @ Si
    ridge = rho + eps if highdim else eps
    M = np.linalg.inv(Sx + ridge * np.eye(p))
    B0 = M @ R
    trace = []
    if highdim:
        B, _, it, primal, dual, stopped = admm_inverse(M, B0, lambda_ / rho, rho, tol, max_iter, trace)
    else:
        B, it, primal, dual, stopped = B0, 0, 0.0, 0.0, False
    r = min(k, p, q)
    if info is not None:
        info.update(iters=it, primal=primal, dual=dual, stopped=stopped, shrinkage=shrink, r_eff=r, trace=trace, B=B,
                    U=None)
    if not np.any(B):
        return [np.zeros((p, k)), np.zeros((q, k))], means
    U0, sig, Vt0 = np.linalg.svd(B, full_matrices=False)
    if info is not None:
        info["sigma"] = sig
    U0 = U0[:, :r]
    V0 = Si @ Vt0[:r].T
    U, V = rrr_tail(U0, V0, U0.T @ Sx @ U0, V0.T @ Syy @ V0, U0.T @ Sxy @ V0, k, eps)
    return [U, V], means


__all__ = ["admm_inverse", "admm_ref", "ledoit_wolf_data", "moment_ccar3_fit", "ref_ccar3_fit", "sqrt_inv_psd",
           "whiten_factor"]
