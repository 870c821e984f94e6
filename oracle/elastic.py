"""CPU restatement (numpy, float64) of the elastic-net ALS estimators of the reference
(cca_zoo/linear/_iterative.py): ElasticCCA and SCCA_IPLS.

TEST INFRASTRUCTURE ONLY -- the checker of the regression kinds of csrc/als.cu, in the two forms of oracle/sparse.py
(a module of its own, so that oracle/sparse.py, the checker of the other ALS kinds, stays as it is):

* ``ref_elastic_fit`` -- the reference's data-space loop, restated, each sklearn regression replaced by an exact solve;
* ``cov_elastic_fit`` -- the Gram-space form the CUDA kernel implements.

Each view update is the penalised regression of sklearn's Ridge (l1_ratio 0) / Lasso (1) / ElasticNet:

    min_w 1/2 w^T Q w - b^T w + lam ||w||_1,   Q = X_i^T X_i / n + rho I,   b = X_i^T y / n,   lam = alpha l1

with rho = alpha (1 - l1) for Lasso / ElasticNet and rho = alpha / n for Ridge (whose objective is not divided by n),

solved to a KKT residual <= 1e-12 max(1, ||b||_inf): the minimum-norm solution through an eigendecomposition when
lam = 0 (sklearn's Ridge/SVD answer; its Lasso at alpha = 0 instead keeps a path-dependent null-space component), cyclic
coordinate descent from the current weights otherwise.  Where the minimiser is unique the result does not depend on
the solver, so it is comparable with sklearn's random-order coordinate descent to that solver's tolerance.
"""
from __future__ import annotations

import numpy as np

from .restatement import block_slices, perview, setup_fit
from .sparse import als_init, dimension_record, update_record

ELASTIC_KINDS = ("elastic", "ipls")
KKT_TOL = 1e-12
RCOND = 1e-12
CD_SWEEPS = 1000      # the max_iter of sklearn's Lasso / ElasticNet, as in csrc/als.cu


def elastic_params(kind, m, alpha=None, l1_ratio=None):
    """[(alpha_i, l1_i)] with the reference's defaults: alpha 0, l1_ratio 0.5 (ElasticCCA) / 1 (SCCA_IPLS)."""
    al = perview(0.0 if alpha is None else alpha, 0.0, m)
    default_l1 = 0.5 if kind == "elastic" else 1.0
    l1 = perview(default_l1 if l1_ratio is None else l1_ratio, default_l1, m)
    return [(float(a), float(r)) for a, r in zip(al, l1)]


def kkt_residual(Q, b, lam, w):
    g = Q @ w - b
    r = np.where(w != 0.0, np.abs(g + lam * np.sign(w)), np.maximum(np.abs(g) - lam, 0.0))
    return float(r.max()) if r.size else 0.0


def solve_penalised(Gii, b, n, alpha, l1, w0, rcond=RCOND, report=None, rec=None):
    """argmin 1/2 w^T (Gii / n + rho I) w - b^T w + alpha l1 ||w||_1 (see the module docstring).  A coordinate
    descent still above the KKT bound after CD_SWEEPS sweeps appends False to ``report`` (a list).  ``rec`` (a dict)
    receives the eigenvalue cut with the smallest kept and the largest dropped mu_k (lam = 0), or the KKT residual
    of every sweep of the coordinate descent and its bound (lam > 0)."""
    p = b.size
    rho, lam = (alpha / n if l1 == 0.0 else alpha * (1.0 - l1)), alpha * l1  # Ridge's alpha is not divided by n
    Q = Gii / n + rho * np.eye(p)
    if lam == 0.0:
        ev, V = np.linalg.eigh(Gii)
        mk = ev / n + rho
        inv = np.where(mk > rcond * max(mk.max(), 0.0), 1.0 / np.where(mk > 0, mk, 1.0), 0.0)
        if rec is not None:
            cut = rcond * max(mk.max(), 0.0)
            rec.update(cut=float(cut), kept_min=float(mk[mk > cut].min(initial=np.inf)),
                       dropped_max=float(mk[mk <= cut].max(initial=-np.inf)))
        return V @ (inv * (V.T @ b))
    tol = KKT_TOL * max(1.0, float(np.abs(b).max(initial=0.0)))
    w = np.array(w0, dtype=np.float64)
    if rec is not None:
        rec.update(kkt_tol=tol, kkt=[])
    for sweep in range(CD_SWEEPS + 1):
        g = Q @ w - b
        if rec is not None:
            rec["kkt"].append(kkt_residual(Q, b, lam, w))
        if kkt_residual(Q, b, lam, w) <= tol:
            break
        if sweep == CD_SWEEPS:
            if report is not None:
                report.append(False)
            break
        for j in range(p):
            q = Q[j, j]
            nw = np.sign(w[j] * q - g[j]) * max(abs(w[j] * q - g[j]) - lam, 0.0) / q if q > 0.0 else 0.0
            dl = nw - w[j]
            if dl != 0.0:
                g += dl * Q[:, j]
                w[j] = nw
    return w


def _loop(kind, dims, w, params, n, max_iter, tol, cross, gram_ii, colmean, report, rcond=RCOND, trace=None):
    """One latent dimension.  ``cross(w, i)`` -> (X_i^T t, ||t||) with the model's target t (ElasticCCA: all views,
    SCCA_IPLS: the others); ``gram_ii(i)`` -> X_i^T X_i; ``colmean(i)`` -> column means of X_i.  Returns the deltas;
    a capped coordinate descent appends to ``report``.  ``trace`` (a list) receives one record per view update
    (oracle.sparse.update_record, what solve_penalised records and, for SCCA_IPLS, the std)."""
    m = len(dims)
    deltas = []
    for it in range(max_iter):
        w_prev = [wi.copy() for wi in w]
        for i in range(m):
            raw, tn = cross(w, i)
            rec = update_record(trace, it, i, raw, tn)
            if tn > 1e-12:
                raw = raw / tn
            Gii = gram_ii(i)
            wi = solve_penalised(Gii, raw / n, n, params[i][0], params[i][1], w[i], rcond=rcond, report=report, rec=rec)
            if kind == "ipls":
                sd = np.sqrt(max(float(wi @ Gii @ wi) / n - float(colmean(i) @ wi) ** 2, 0.0))
                if rec is not None:
                    rec["sd"] = float(sd)
                if sd > 1e-12:
                    wi = wi / sd
            w[i] = wi
        delta = max(np.linalg.norm(w[i] - w_prev[i]) for i in range(m))
        deltas.append(delta)
        if delta < tol:
            break
    return deltas


def cov_elastic_fit(G, dims, n, kind, latent_dimensions=1, params=None, colmeans=None, init=None, max_iter=500,
                    tol=1e-6, random_state=None, return_info=False, rcond=RCOND, trace=None):
    """ElasticCCA / SCCA_IPLS on the block Gram matrix G ((n - 1) C, centred or not following ``center``), the form
    csrc/als.cu iterates.  ``colmeans`` (D,): column means of the views, zeros (the default) when they are centred;
    deflated with the views.  Returns (weights per view (d_i x k), sweeps per dimension); as in ccab_als_fit, the sweep
    count of a dimension in which a coordinate descent stopped at CD_SWEEPS above the KKT bound is negated.  ``rcond``:
    the relative eigenvalue cut of the lam = 0 solves (the ``mu`` of ops.als_fit); ``trace`` (a list) receives one
    record per dimension (oracle.sparse.dimension_record)."""
    G = np.array(G, dtype=np.float64)
    dims = [int(p) for p in dims]
    m, k, D = len(dims), int(latent_dimensions), G.shape[0]
    sl = block_slices(dims)
    params = elastic_params(kind, m) if params is None else params
    init = als_init(dims, k, random_state) if init is None else init
    mu = np.zeros(D) if colmeans is None else np.array(colmeans, dtype=np.float64)
    W = [np.zeros((p, k)) for p in dims]
    iters, info = [], []

    def cross(w, i):
        js = [j for j in range(m) if kind == "elastic" or j != i]
        u = sum(G[:, sl[j]] @ w[j] for j in js)
        tn2 = sum(float(w[j] @ u[sl[j]]) for j in js)
        return u[sl[i]], np.sqrt(max(tn2, 0.0))

    for d in range(k):
        w = [v.copy() for v in init[d]]
        report = []
        updates = None if trace is None else []
        deltas = _loop(kind, dims, w, params, n, max_iter, tol, cross, lambda i: G[sl[i], sl[i]], lambda i: mu[sl[i]],
                       report, rcond, updates)
        iters.append(-len(deltas) if report else len(deltas))
        info.append(deltas)
        for i in range(m):
            W[i][:, d] = w[i]
        if trace is not None:
            trace.append(dimension_record(G, sl, w, updates, deltas))
        if d + 1 < k:
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
            for i in range(m):
                mu[sl[i]] = mu[sl[i]] - float(mu[sl[i]] @ w[i]) * F[sl[i], i]
    if return_info:
        return W, iters, info
    return W, iters


def ref_elastic_fit(views, kind, latent_dimensions=1, params=None, max_iter=500, tol=1e-6, random_state=None,
                    center=True, return_info=False):
    """Data-space restatement of the reference loop (cca_zoo/linear/_iterative.py:65-117, SCCA_IPLS :599-623,
    ElasticCCA :808-831, deflate of cca_zoo/_utils/_linalg.py:91-116) in float64, the regressions solved exactly
    (sweep counts negated as in cov_elastic_fit)."""
    views, _ = setup_fit(views, center)
    views = [np.asarray(v, dtype=np.float64) for v in views]
    dims = [v.shape[1] for v in views]
    m, k, n = len(views), int(latent_dimensions), views[0].shape[0]
    params = elastic_params(kind, m) if params is None else params
    init = als_init(dims, k, random_state)
    W = [np.zeros((p, k)) for p in dims]
    iters, info = [], []
    Xs = [v.copy() for v in views]

    def cross(w, i):
        t = np.asarray(sum(Xs[j] @ w[j] for j in range(m) if kind == "elastic" or j != i))
        return Xs[i].T @ t, np.linalg.norm(t)

    for d in range(k):
        w = [v.copy() for v in init[d]]
        report = []
        deltas = _loop(kind, dims, w, params, n, max_iter, tol, cross, lambda i: Xs[i].T @ Xs[i],
                       lambda i: Xs[i].mean(axis=0), report)
        iters.append(-len(deltas) if report else len(deltas))
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
