"""Float64 numpy restatements of GFA (Group Factor Analysis, cca_zoo/probabilistic/_gfa.py).

TEST INFRASTRUCTURE ONLY: the step-for-step reference of the ``ccab_gfa_fit`` kernel (csrc/gfa.cu).

Two forms of the same variational loop:

  * ``ref_gfa_fit``: the data-space loop of the reference, restated without the posterior sampling, and recording the
    two statistics that steer it (the relative change of z and the pruning statistic mean(z^2, 0)).
  * ``cov_gfa_fit``: the Gram form the kernel iterates.  From the first Z update on, z = X B with
    B = [tau_1 W_1; ...; tau_m W_m] cov_z (D x k), so every later quantity is a function of G = X^T X (centred when
    ``center``) and of GB:  X_m^T z = (GB)_m,  z^T z = B^T G B,  sum z o (X_m W_m) = sum (GB)_m o W_m,
    mean(z^2, 0) = diag(B^T G B) / n  and  ||z - z'||^2 = tr((B - B')^T (GB - GB')).  Only the first W update reads
    the random z0, through X^T z0.

``gram_state`` / ``gram_step`` are the kernel's phases on a state dictionary that mirrors the device state block
(header counters, B, GB, their previous values, W, cov_w, ww, cov_z, zz, alpha, b_ard, tau, b_tau and the original
index of every active column).
"""
from __future__ import annotations

import numpy as np

ARD_ALPHA_0 = 1e-14
ARD_BETA_0 = 1e-14
TAU_ALPHA_0 = 1e-14
TAU_BETA_0 = 1e-14
INIT_TAU = 1e3
DROP_TOL = 1e-7
PATIENCE = 1000


def _inv_spd(A):
    L = np.linalg.cholesky(A)
    Li = np.linalg.solve(L, np.eye(A.shape[0]))
    return Li.T @ Li


# ---------------------------------------------------------------------------------------------------- data space
def ref_gfa_fit(views, k, center=True, max_iter=10000, tol=1e-4, drop_k=True, random_state=0):
    """The reference's loop on the (centred) views.  Returns a dict with the final z, cov_z, W, cov_w, alpha, b_ard,
    tau, b_tau, a_ard, a_tau, n_iter, k and the statistics ``rel`` (every relative change of z that was compared with
    tol) and ``drop`` (every mean(z^2, 0) entry that was compared with the pruning threshold)."""
    X = [np.asarray(v, dtype=np.float64) for v in views]
    if center:
        X = [x - x.mean(axis=0) for x in X]
    rng = np.random.default_rng(random_state)
    m, n = len(X), X[0].shape[0]
    d = [x.shape[1] for x in X]
    z = rng.standard_normal((n, k))
    cov_z = np.eye(k)
    w = [np.zeros((p, k)) for p in d]
    cov_w = [np.eye(k) for _ in range(m)]
    tau = np.full(m, INIT_TAU)
    datavar = np.array([np.var(x, axis=0, ddof=1).sum() for x in X])
    alpha = [np.full(k, k * d[i] / max(datavar[i] - 1.0 / tau[i], 1e-8)) for i in range(m)]
    y_const = np.array([np.sum(x ** 2) for x in X])
    a_ard = ARD_ALPHA_0 + np.array(d) / 2.0
    a_tau = TAU_ALPHA_0 + n * np.array(d) / 2.0
    ww = [w[i].T @ w[i] + d[i] * cov_w[i] for i in range(m)]
    zz = z.T @ z + n * cov_z
    b_ard = [np.full(k, ARD_BETA_0) for _ in range(m)]
    b_tau = np.full(m, TAU_BETA_0)
    prev_z, n_iter, stable = None, max_iter, 0
    rels, drops = [], []
    for it in range(max_iter):
        for i in range(m):
            tmp = 1.0 / np.sqrt(alpha[i])
            inner = np.outer(tmp, tmp) * zz + np.eye(k) / tau[i]
            cov_w[i] = (1.0 / tau[i]) * np.outer(tmp, tmp) * _inv_spd(inner)
            w[i] = X[i].T @ z @ cov_w[i] * tau[i]
            ww[i] = w[i].T @ w[i] + d[i] * cov_w[i]
        prec = np.eye(k)
        for i in range(m):
            prec = prec + tau[i] * ww[i]
        cov_z = _inv_spd(prec)
        rhs = np.zeros((n, k))
        for i in range(m):
            rhs = rhs + X[i] @ w[i] * tau[i]
        z = rhs @ cov_z
        zz = z.T @ z + n * cov_z
        for i in range(m):
            b_ard[i] = ARD_BETA_0 + np.diag(ww[i]) / 2.0
            alpha[i] = a_ard[i] / b_ard[i]
        for i in range(m):
            b_tau[i] = TAU_BETA_0 + (y_const[i] + np.sum(ww[i] * zz) - 2.0 * np.sum(z * (X[i] @ w[i]))) / 2.0
            tau[i] = a_tau[i] / b_tau[i]
        pruned = False
        if drop_k:
            stat = np.mean(z ** 2, axis=0)
            drops.extend(stat.tolist())
            keep = np.where(stat > DROP_TOL)[0]
            if 0 < len(keep) != k:
                pruned, k = True, len(keep)
                z, cov_z, zz = z[:, keep], cov_z[np.ix_(keep, keep)], zz[np.ix_(keep, keep)]
                for i in range(m):
                    w[i], cov_w[i], ww[i] = w[i][:, keep], cov_w[i][np.ix_(keep, keep)], ww[i][np.ix_(keep, keep)]
                    alpha[i], b_ard[i] = alpha[i][keep], b_ard[i][keep]
        if pruned:
            stable = 0
        elif prev_z is not None and prev_z.shape == z.shape:
            rel = np.linalg.norm(z - prev_z) / max(np.linalg.norm(prev_z), 1e-300)
            rels.append(rel)
            stable = stable + 1 if rel < tol else 0
        prev_z = z.copy()
        if stable >= PATIENCE:
            n_iter = it + 1
            break
    return dict(z=z, cov_z=cov_z, W=w, cov_w=cov_w, alpha=np.array(alpha), b_ard=b_ard, tau=tau, b_tau=b_tau,
                a_ard=a_ard, a_tau=a_tau, n_iter=n_iter, k=k, rel=np.array(rels), drop=np.array(drops))


# ---------------------------------------------------------------------------------------------------- Gram form
def gram_inputs(views, k, center=True, random_state=0):
    """(G, n, dims, X^T z0, z0^T z0, datavar, y_const) exactly as the package forms them (float64)."""
    X = [np.asarray(v, dtype=np.float64) for v in views]
    mu = [x.mean(axis=0) for x in X]
    Xc = [x - u for x, u in zip(X, mu)]
    Xg = np.hstack(Xc if center else X)
    n = Xg.shape[0]
    G = Xg.T @ Xg
    G = 0.5 * (G + G.T)
    z0 = np.random.default_rng(random_state).standard_normal((n, k))
    Xz0 = Xg.T @ z0
    dims = [x.shape[1] for x in X]
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    Cc = np.hstack(Xc)
    datavar = np.array([float(np.sum(Cc[:, off[i]:off[i + 1]] ** 2)) / (n - 1) for i in range(len(dims))])
    return G, n, dims, Xz0, z0.T @ z0, datavar


def gram_state(n, dims, k, z0tz0, datavar, y_const):
    """The state block the host writes before the first call: k active columns, tau = 1e3, alpha from the data
    variance, zz = z0^T z0 + n I."""
    m, D = len(dims), int(sum(dims))
    tau = np.full(m, INIT_TAU)
    alpha = np.array([np.full(k, k * dims[i] / max(datavar[i] - 1.0 / tau[i], 1e-8)) for i in range(m)])
    return dict(iters=0, k=k, stable=0, stop=False, rel=None, n=float(n), dims=list(dims),
                y_const=np.asarray(y_const, dtype=np.float64),
                a_ard=ARD_ALPHA_0 + np.array(dims) / 2.0, a_tau=TAU_ALPHA_0 + n * np.array(dims) / 2.0,
                tau=tau, b_tau=np.full(m, TAU_BETA_0), alpha=alpha, b_ard=np.full((m, k), ARD_BETA_0),
                cov_w=np.array([np.eye(k)] * m), ww=np.zeros((m, k, k)), cov_z=np.eye(k),
                zz=z0tz0 + n * np.eye(k), B=np.zeros((D, k)), GB=np.zeros((D, k)), B_prev=np.zeros((D, k)),
                GB_prev=np.zeros((D, k)), W=np.zeros((D, k)), index=np.arange(k))


def y_constants(G, dims):
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    return np.array([float(np.trace(G[off[i]:off[i + 1], off[i]:off[i + 1]])) for i in range(len(dims))])


def gram_step(st, G, Xz0, tol, drop_k=True):
    """One iteration of the kernel on ``st`` (in place); a stopped state does not move."""
    if st["stop"]:
        return st
    dims, n = st["dims"], st["n"]
    m, k = len(dims), st["k"]
    off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
    XZ = Xz0[:, st["index"]] if st["iters"] == 0 else st["GB"]
    # W update
    W = np.zeros_like(XZ)
    for i in range(m):
        tmp = 1.0 / np.sqrt(st["alpha"][i])
        T = np.outer(tmp, tmp)
        st["cov_w"][i] = (1.0 / st["tau"][i]) * T * _inv_spd(T * st["zz"] + np.eye(k) / st["tau"][i])
        sl = slice(off[i], off[i + 1])
        W[sl] = st["tau"][i] * (XZ[sl] @ st["cov_w"][i])
        st["ww"][i] = W[sl].T @ W[sl] + dims[i] * st["cov_w"][i]
    # Z update and the ARD update
    prec = np.eye(k)
    for i in range(m):
        prec = prec + st["tau"][i] * st["ww"][i]
        st["b_ard"][i] = ARD_BETA_0 + np.diag(st["ww"][i]) / 2.0
        st["alpha"][i] = st["a_ard"][i] / st["b_ard"][i]
    st["cov_z"] = _inv_spd(prec)
    TW = W.copy()
    for i in range(m):
        TW[off[i]:off[i + 1]] *= st["tau"][i]
    st["B_prev"], st["GB_prev"] = st["B"], st["GB"]
    st["B"] = TW @ st["cov_z"]
    st["GB"] = G @ st["B"]
    st["W"] = W
    BtGB = st["B"].T @ st["GB"]
    BtGB = np.triu(BtGB) + np.triu(BtGB, 1).T
    st["zz"] = BtGB + n * st["cov_z"]
    # tau update
    for i in range(m):
        sl = slice(off[i], off[i + 1])
        cross = float(np.sum(st["GB"][sl] * W[sl]))
        st["b_tau"][i] = TAU_BETA_0 + (st["y_const"][i] + float(np.sum(st["ww"][i] * st["zz"])) - 2.0 * cross) / 2.0
        st["tau"][i] = st["a_tau"][i] / st["b_tau"][i]
    # pruning
    pruned = False
    st["rel"], st["drop_stat"] = None, np.diag(BtGB) / n
    if drop_k:
        keep = np.where(st["drop_stat"] > DROP_TOL)[0]
        if 0 < len(keep) != k:
            pruned = True
            st["k"] = k = len(keep)
            ix = np.ix_(keep, keep)
            for key in ("B", "GB", "W"):
                st[key] = st[key][:, keep]
            st["cov_z"], st["zz"], st["index"] = st["cov_z"][ix], st["zz"][ix], st["index"][keep]
            st["cov_w"] = np.array([c[ix] for c in st["cov_w"]])
            st["ww"] = np.array([c[ix] for c in st["ww"]])
            st["alpha"], st["b_ard"] = st["alpha"][:, keep], st["b_ard"][:, keep]
    # stopping rule
    if pruned:
        st["stable"] = 0
    elif st["iters"] > 0:
        num = float(np.sum((st["B"] - st["B_prev"]) * (st["GB"] - st["GB_prev"])))
        den = float(np.sum(st["B_prev"] * st["GB_prev"]))
        with np.errstate(invalid="ignore"):
            rel = np.sqrt(num) / max(np.sqrt(den), 1e-300)
        st["rel"] = rel
        st["stable"] = st["stable"] + 1 if rel < tol else 0
    st["iters"] += 1
    if st["stable"] >= PATIENCE:
        st["stop"] = True
    return st


def cov_gfa_fit(views, k, center=True, max_iter=10000, tol=1e-4, drop_k=True, random_state=0):
    """The Gram form of the whole fit.  Returns (state, statistics) with ``state`` as after the last iteration and
    ``statistics`` = (every relative change compared with tol, every pruning statistic compared with 1e-7)."""
    G, n, dims, Xz0, z0tz0, datavar = gram_inputs(views, k, center, random_state)
    st = gram_state(n, dims, k, z0tz0, datavar, y_constants(G, dims))
    rels, drops = [], []
    for _ in range(max_iter):
        gram_step(st, G, Xz0, tol, drop_k)
        if st["rel"] is not None:
            rels.append(st["rel"])
        if drop_k:
            drops.extend(st["drop_stat"].tolist())
        if st["stop"]:
            break
    return st, (np.array(rels), np.array(drops))


def weights(st):
    off = np.concatenate([[0], np.cumsum(st["dims"])]).astype(int)
    return [st["W"][off[i]:off[i + 1]].copy() for i in range(len(st["dims"]))]
