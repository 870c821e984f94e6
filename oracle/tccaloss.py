"""Float64 restatement of the deep tensor-CCA objective (cca_zoo/deep/objectives.py:223-289, ``TCCALoss``) and of
its analytic gradient, in the two whitenings ``cca_zoo_b200.deep.TCCALoss`` uses.

For views z_i (n x k_i): Zc_i = z_i - mean, S_i = Zc_i^T Zc_i / (n - 1) + eps I, H_i = Zc_i W_i,
M = (1/n) sum_s H_1[s] x ... x H_m[s] and loss = -||M||_F.  With Gamma_i = dL/dH_i = -Y_i / (n ||M||),
Y_i = KR_{j != i}(H_j) M_(i)^T (0 when ||M|| = 0):

* ``chol_form``: W_i = R_i = L_i^-T with S_i = L_i L_i^T.  ||M|| is invariant under an orthogonal change of basis in
  every mode and S_i^1/2 R_i is orthogonal, so the loss is the reference's whenever its eigenvalue clamp is inactive.
  dL/dz_i = center((Gamma_i - H_i (H_i^T Gamma_i) / (n - 1)) R_i^T).
* ``eigen_form``: W_i = V f(Lam) V^T with S_i = V Lam V^T and f(l) = max(l, eps)^-1/2: the reference literally.
  With B = sym(Zc_i^T Gamma_i) and F the divided differences of f (F_aa = f'(l_a), 0 where the clamp is active),
  dL/dz_i = center(Gamma_i W_i + 2/(n - 1) Zc_i V (F o V^T B V) V^T).  Where S_i has a repeated eigenvalue the
  reference's eigh backward is NaN; this form gives the finite limit.

``gram_norm`` gives ||M|| without M: ||M||^2 = 1^T (G_1 o ... o G_m) 1 / n^2 with G_i = H_i H_i^T.
"""
from __future__ import annotations

import string

import numpy as np


def moment(H):
    """M (k_1 x ... x k_m) = mean over the samples of the outer products of the rows of H."""
    n = H[0].shape[0]
    T = H[0]
    for h in H[1:]:
        T = (T[..., None] * h.reshape((n,) + (1,) * (T.ndim - 1) + (h.shape[1],)))
    return T.mean(axis=0)


def adjoint(M, H):
    """[Y_i]: Y_i[s, a] = sum_{idx, idx_i = a} M[idx] prod_{j != i} H_j[s, idx_j]."""
    m = len(H)
    letters = string.ascii_letters[:m]
    out = []
    for i in range(m):
        ops = [M] + [H[j] for j in range(m) if j != i]
        spec = letters + "," + ",".join("z" + letters[j] for j in range(m) if j != i) + "->z" + letters[i]
        out.append(np.einsum(spec, *ops, optimize=True))
    return out


def _center(x):
    return x - x.mean(axis=0)


def _gammas(M, H, n):
    nrm = float(np.linalg.norm(M.reshape(-1)))
    if nrm == 0.0:
        return nrm, [np.zeros_like(h) for h in H]
    return nrm, [-y / (n * nrm) for y in adjoint(M, H)]


def chol_form(zs, eps):
    """(loss, [dL/dz_i], {"H", "R"}) by Cholesky whitening."""
    zs = [np.asarray(z, dtype=np.float64) for z in zs]
    n = zs[0].shape[0]
    H, R = [], []
    for z in zs:
        Zc = _center(z)
        S = Zc.T @ Zc / (n - 1) + eps * np.eye(z.shape[1])
        Ri = np.linalg.inv(np.linalg.cholesky(S)).T
        H.append(Zc @ Ri)
        R.append(Ri)
    M = moment(H)
    nrm, Gam = _gammas(M, H, n)
    grads = [_center(g - h @ (h.T @ g) / (n - 1)) @ r.T for g, h, r in zip(Gam, H, R)]
    return -nrm, grads, {"H": H, "R": R, "M": M}


def divided_differences(lam, eps):
    """F_ab = (f(l_a) - f(l_b)) / (l_a - l_b), F_aa = f'(l_a), f(l) = max(l, eps)^-1/2 (f' = 0 where clamped)."""
    lam = np.asarray(lam, dtype=np.float64)
    s = np.sqrt(np.maximum(lam, eps))
    f = 1.0 / s
    la, lb = lam[:, None], lam[None, :]
    both = (la > eps) & (lb > eps)
    d = la - lb
    with np.errstate(divide="ignore", invalid="ignore"):
        mixed = np.where(d != 0.0, (f[:, None] - f[None, :]) / np.where(d != 0.0, d, 1.0), 0.0)
    return np.where(both, -1.0 / (s[:, None] * s[None, :] * (s[:, None] + s[None, :])), mixed)


def eigen_form(zs, eps):
    """(loss, [dL/dz_i], {"H", "W"}) with the reference's clamp(eigh(S_i), min=eps) whitening."""
    zs = [np.asarray(z, dtype=np.float64) for z in zs]
    n = zs[0].shape[0]
    H, W, parts = [], [], []
    for z in zs:
        Zc = _center(z)
        S = Zc.T @ Zc / (n - 1) + eps * np.eye(z.shape[1])
        lam, V = np.linalg.eigh(S)
        Wi = (V / np.sqrt(np.maximum(lam, eps))) @ V.T
        H.append(Zc @ Wi)
        W.append(Wi)
        parts.append((Zc, lam, V))
    M = moment(H)
    nrm, Gam = _gammas(M, H, n)
    grads = []
    for g, Wi, (Zc, lam, V) in zip(Gam, W, parts):
        B = Zc.T @ g
        B = 0.5 * (B + B.T)
        X = V @ (divided_differences(lam, eps) * (V.T @ B @ V)) @ V.T
        grads.append(_center(g @ Wi + 2.0 / (n - 1) * Zc @ X))
    return -nrm, grads, {"H": H, "W": W, "M": M}


def gram_norm(H):
    """||M||_F from the sample Grams: sqrt(1^T (G_1 o ... o G_m) 1) / n, M never formed."""
    n = H[0].shape[0]
    P = H[0] @ H[0].T
    for h in H[1:]:
        P *= h @ h.T
    return float(np.sqrt(max(P.sum(), 0.0))) / n
