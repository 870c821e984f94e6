"""CPU restatement (numpy, float64 unless the views say otherwise) of the sparse / ALS estimators of the reference
(cca_zoo/linear/_iterative.py): PLS_ALS, SCCA_PMD, ParkhomenkoCCA, SCCA_Span, SCCA_ADMM.

TEST INFRASTRUCTURE ONLY -- the checker of csrc/als.cu, in the two forms of oracle/restatement.py:

* ``ref_als_fit`` -- the reference's data-space loop, restated;
* ``cov_als_fit`` -- the Gram-space form the CUDA kernel implements, validated against the reference by
  ``oracle/make_golden_sparse.py`` and ``tests/test_sparse_oracle_cpu.py``.
"""
from __future__ import annotations

import numpy as np

from .restatement import block_slices, perview, setup_fit

ALS_KINDS = ("pls", "pmd", "parkhomenko", "span", "admm")


def als_params(kind, dims, tau=None, span=None):
    """Per-view parameter of each model with the reference's defaults: PMD tau (1.0), Parkhomenko / ADMM tau (0.1),
    Span span (the width of view 0 for every view, cca_zoo/linear/_iterative.py:690-692)."""
    m = len(dims)
    if kind == "pmd":
        return [float(t) for t in perview(tau, 1.0, m)]
    if kind in ("parkhomenko", "admm"):
        return [float(t) for t in perview(tau, 0.1, m)]
    if kind == "span":
        return [int(s) for s in perview(dims[0] if span is None else span, dims[0], m)]
    return [0.0] * m


def als_init(dims, k, random_state):
    """Initial weights of every dimension, drawn up front in the reference's order (one standard normal vector per view
    per dimension from ``np.random.default_rng(random_state)``, unit norm): a list of k lists of m vectors."""
    rng = np.random.default_rng(random_state)
    out = []
    for _ in range(k):
        ws = [rng.standard_normal(p) for p in dims]
        out.append([w / np.linalg.norm(w) for w in ws])
    return out


def _soft(x, t):
    return np.sign(x) * np.maximum(np.abs(x) - t, 0.0)


def _unit(x, rec=None):
    nrm = np.linalg.norm(x)
    if rec is not None:
        rec["norm"] = float(nrm)
    return x / nrm if nrm > 1e-12 else x


def tau_gap(x, t):
    """min ||x_r| - t|: how far the soft-threshold support decision |x_r| > t is from flipping."""
    return float(np.abs(np.abs(x) - t).min())


def _als_post(kind, raw, param, rec=None):
    """Per-view update from X_i^T t / ||t|| (the _update_weight of each Gauss-Seidel model).  ``rec`` (a dict) receives
    the quantities its decisions turn on."""
    if kind == "parkhomenko":
        if rec is not None:
            rec["tau_gap"] = tau_gap(raw, param)
        return _unit(_soft(raw, param), rec)
    if kind == "span":
        if param < raw.size:
            srt = np.sort(np.abs(raw))
            thr = srt[-param]
            if rec is not None:
                rec.update(thr=float(thr), gap=float(thr - srt[-param - 1]))
            raw = np.where(np.abs(raw) >= thr, raw, 0.0)
        return _unit(raw, rec)
    if kind == "pmd":
        bound = param
        l1 = np.abs(raw).sum()
        if rec is not None:
            rec.update(l1=float(l1), bound=float(bound))
        if l1 <= bound:
            return _unit(raw, rec)
        lo, hi = 0.0, float(np.abs(raw).max())
        for _ in range(50):
            mid = (lo + hi) / 2.0
            if np.abs(_soft(raw, mid)).sum() > bound:
                lo = mid
            else:
                hi = mid
        if rec is not None:
            rec.update(thr=(lo + hi) / 2.0, tau_gap=tau_gap(raw, (lo + hi) / 2.0))
        return _unit(_soft(raw, (lo + hi) / 2.0), rec)
    return _unit(raw, rec)


def update_record(trace, it, i, raw, tn):
    """The record of one view update appended to ``trace`` (None without a trace): the raw target X_i^T t and ||t||."""
    if trace is None:
        return None
    rec = {"sweep": it, "view": i, "raw": np.array(raw, dtype=np.float64), "tn": float(tn)}
    trace.append(rec)
    return rec


def _als_loop(kind, dims, w, params, mu, n, max_iter, tol, cross, gram_ii, trace=None):
    """The iteration of one latent dimension, shared by the data-space and the Gram-space restatements.

    ``cross(w, i)`` -> (X_i^T t, ||t||) with t = sum_{j != i} X_j w_j;  ``gram_ii(i)`` -> X_i^T X_i.
    Returns (sweeps, deltas).  ``trace`` (a list) receives one record per view update (update_record, plus what
    the post-processing decides on)."""
    m = len(dims)
    deltas = []
    if kind == "admm":
        z = [wi.copy() for wi in w]
        eta = [np.zeros_like(wi) for wi in w]
    for it in range(max_iter):
        w_prev = [wi.copy() for wi in w]
        if kind == "admm":
            raws = [cross(w, i) for i in range(m)]
            for i in range(m):
                raw, tn = raws[i]
                rec = update_record(trace, it, i, raw, tn)
                if tn > 1e-12:
                    raw = raw / tn
                Gii = gram_ii(i)
                g = Gii @ w[i] - raw + mu * (w[i] - z[i] + eta[i])
                w[i] = w[i] - g / (np.linalg.norm(Gii) / n + mu)
                z[i] = _soft(w[i] + eta[i], params[i] / mu)
                zn = np.linalg.norm(z[i])
                if rec is not None:
                    rec.update(zn=float(zn), tau_gap=tau_gap(w[i] + eta[i], params[i] / mu))
                if zn > 1.0:
                    z[i] = z[i] / zn
                eta[i] = eta[i] + w[i] - z[i]
            for i in range(m):
                w[i] = z[i].copy()
        else:
            for i in range(m):
                raw, tn = cross(w, i)
                rec = update_record(trace, it, i, raw, tn)
                if tn > 1e-12:
                    raw = raw / tn
                w[i] = _als_post(kind, raw, params[i] * np.sqrt(dims[i]) if kind == "pmd" else params[i], rec)
        delta = max(np.linalg.norm(w[i] - w_prev[i]) for i in range(m))
        deltas.append(delta)
        if delta < tol:
            break
    return len(deltas), deltas


def cov_als_fit(G, dims, n, kind, latent_dimensions=1, params=None, mu=1.0, init=None, max_iter=500, tol=1e-6,
                random_state=None, return_info=False, trace=None):
    """The sparse / ALS models on the block Gram matrix G = [X_1..X_m]^T [X_1..X_m] ((n - 1) C of the covariance the
    package computes, for either value of ``center``): the form csrc/als.cu iterates.

      X_i^T t = sum_{j != i} G_ij w_j,   ||t||^2 = w_{-i}^T G w_{-i},
      deflation G <- Q^T G Q,  Q_i = I - w_i a_i^T / s_i

    Returns (weights per view (d_i x k), sweeps per dimension) and, with ``return_info``, the per-sweep convergence
    deltas of every dimension.  ``trace`` (a list) receives one record per dimension (dimension_record)."""
    G = np.array(G, dtype=np.float64)
    dims = [int(p) for p in dims]
    m, k = len(dims), int(latent_dimensions)
    sl = block_slices(dims)
    params = als_params(kind, dims) if params is None else params
    init = als_init(dims, k, random_state) if init is None else init
    W = [np.zeros((p, k)) for p in dims]
    iters, info = [], []

    def cross(w, i):
        u = sum(G[:, sl[j]] @ w[j] for j in range(m) if j != i)
        tn2 = sum(float(w[j] @ u[sl[j]]) for j in range(m) if j != i)
        return u[sl[i]], np.sqrt(max(tn2, 0.0))

    for d in range(k):
        w = [v.copy() for v in init[d]]
        updates = None if trace is None else []
        sweeps, deltas = _als_loop(kind, dims, w, params, mu, n, max_iter, tol, cross, lambda i: G[sl[i], sl[i]],
                                   updates)
        iters.append(sweeps)
        info.append(deltas)
        for i in range(m):
            W[i][:, d] = w[i]
        if trace is not None:
            trace.append(dimension_record(G, sl, w, updates, deltas))
        if d + 1 < k:
            D = G.shape[0]
            E, F = np.zeros((D, m)), np.zeros((D, m))
            for i in range(m):
                a = G[sl[i], sl[i]] @ w[i]
                s = float(w[i] @ a)
                E[sl[i], i] = w[i]
                if s > 1e-12:
                    F[sl[i], i] = a / s
            Y = G @ E
            S = E.T @ Y
            G = G - Y @ F.T - F @ Y.T + F @ S @ F.T
    if return_info:
        return W, iters, info
    return W, iters


def dimension_record(G, sl, w, updates, deltas):
    """The trace record of one latent dimension: max |G| of its (deflated) Gram matrix, its view updates, its
    convergence deltas and the deflation scalars s_i = w_i^T G_ii w_i of its final weights."""
    return {"gmax": float(np.abs(G).max()), "updates": updates, "deltas": list(deltas),
            "s": [float(w[i] @ G[sl[i], sl[i]] @ w[i]) for i in range(len(sl))]}


def ref_als_fit(views, kind, latent_dimensions=1, params=None, mu=1.0, max_iter=500, tol=1e-6, random_state=None,
                center=True, return_info=False):
    """Data-space restatement of the reference loop (cca_zoo/linear/_iterative.py:65-117 and the models'
    _update_weight / _fit_single, deflate of cca_zoo/_utils/_linalg.py:91-116), in the views' dtype."""
    views, _ = setup_fit(views, center)
    dims = [v.shape[1] for v in views]
    m, k, n = len(views), int(latent_dimensions), views[0].shape[0]
    params = als_params(kind, dims) if params is None else params
    init = als_init(dims, k, random_state)
    W = [np.zeros((p, k)) for p in dims]
    iters, info = [], []
    Xs = [v.copy() for v in views]

    def cross(w, i):
        t = np.asarray(sum(Xs[j] @ w[j] for j in range(m) if j != i))
        return Xs[i].T @ t, np.linalg.norm(t)

    for d in range(k):
        w = [v.copy() for v in init[d]]
        sweeps, deltas = _als_loop(kind, dims, w, params, mu, n, max_iter, tol, cross, lambda i: Xs[i].T @ Xs[i])
        iters.append(sweeps)
        info.append(deltas)
        for i in range(m):
            W[i][:, d] = w[i]
        for i in range(m):
            t = Xs[i] @ w[i]
            s = float(t @ t)
            if s > 1e-12:
                Xs[i] = Xs[i] - np.outer(t, t @ Xs[i]) / s
    if return_info:
        return W, iters, info
    return W, iters
