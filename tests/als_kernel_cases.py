"""TEST INFRASTRUCTURE ONLY: the case table of tests/test_als_kernel_gpu.py (the ALS kernel ``als_dimension`` of
csrc/als.cu, driven through ``ops.als_fit``) and the float64 reference half of every case.

Each case builds from its seed a block Gram matrix G, the initial weights (k x D) and the per-view parameters, and runs
the Gram-space restatement (``oracle.sparse.cov_als_fit`` / ``oracle.elastic.cov_elastic_fit``) with a trace of every
decision it takes.  n - 1 is a power of two, so the covariance G / (n - 1) handed to the device and the kernel's
rescaling by n - 1 give back G bit for bit.

Every ALS kind makes discrete decisions: the support of a soft threshold, the sides of the PMD bisection, the Span
selection, the ADMM projection, the eigenvalue cut of the regression kinds, the 1e-12 guards and the convergence test.
A decision within rounding of its boundary can go either way on the device and in numpy, and the weights then differ
by O(1).  So the cases are chosen to keep a margin at every decision, or to sit exactly on it by construction (zero
cross blocks, thresholds above every entry, integer data with exact ties); tests/test_als_kernel_cases_cpu.py proves
that from the trace before any GPU run.  G is L L^T + diag with cross blocks of rank 8, so no view runs out of
cross-view signal within the k <= 3 dimensions a case deflates: a view whose blocks had been deflated to rounding
residue would turn that residue into a unit vector.

The shapes are picked where the kernel branches: widths at the unroll edges of ``matvec`` (96/97, 127-129, 255-257)
and of ``cta_matvec`` (32/33, 64/65), widths of 1, eight views, and D past one warp per row of the whole grid (4224
warps for ``als_dimension<false>``, 2112 for ``<true>`` on the 132 SMs of an H100 SXM at one CTA per SM), both for
the full pass and for a Gauss-Seidel phase (the rows of view i plus those of the previous view).
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

from oracle import elastic as E
from oracle import sparse as S

SMS_H100 = 132
WARPS_PER_SM = {False: 32, True: 16}     # als_dimension<REG>: one CTA of 1024 / 512 threads per SM
FIRST_TOL = 1e-12                        # max_iter <= 1, relative to max |w|
LATER_TOL = 1e-10                        # more sweeps
REG_KINDS = ("elastic", "ipls")
KINDS = ("pls", "pmd", "parkhomenko", "span", "admm") + REG_KINDS
RCOND = 1e-9                             # eigenvalue cut of the lam = 0 regressions: rounding residue stays 1e3 below it


@dataclass(frozen=True)
class AlsCase:
    name: str
    kind: str
    dims: tuple
    k: int
    max_iter: int
    tol: float = 0.0
    params: tuple = ()                   # per view: PMD / Parkhomenko / ADMM tau, Span span, or (alpha, l1_ratio)
    mu: float | None = None              # ADMM penalty; the regression kinds get RCOND
    gen: str = "lowrank"                 # lowrank | zero_cross | data | span_tie | span_zero
    j: int = 10                          # n - 1 = 2^j
    seed: int = 0
    tags: tuple = ()                     # the branches the case is there to reach

    @property
    def D(self):
        return sum(self.dims)

    @property
    def n(self):
        return 2 ** self.j + 1

    @property
    def reg(self):
        return self.kind in REG_KINDS


def _default_params(kind, dims):
    m = len(dims)
    return {"pls": (0.0,) * m, "pmd": (0.3,) * m, "parkhomenko": (0.05,) * m, "admm": (0.1,) * m,
            "span": tuple(max(1, p // 4) for p in dims), "elastic": ((0.05, 0.5),) * m,
            "ipls": ((0.05, 0.5),) * m}[kind]


def _case(name, kind, dims, k, max_iter, **kw):
    kw.setdefault("params", _default_params(kind, dims))
    if kind == "admm":
        kw.setdefault("j", 0)   # its gradient step is G_ii w against ||G_ii||_F / n: n = 2 keeps ||z|| near 1
    return AlsCase(name, kind, tuple(dims), k, max_iter, **kw)


MIX = ((0.0, 0.0), (0.5, 0.0), (0.05, 1.0), (0.05, 0.5))        # alpha = 0, Ridge, Lasso, ElasticNet

CASES = []
for _kind in KINDS:
    CASES += [
        _case(f"{_kind}_m2_k1_it0", _kind, (13, 17), 1, 0),
        _case(f"{_kind}_m2_k3_it1", _kind, (33, 65), 3, 1, seed=1),
        _case(f"{_kind}_m3_k3_it2", _kind, (32, 97, 129), 3, 2, seed=2),
        _case(f"{_kind}_m3_k1_it20", _kind, (96, 128, 257), 1, 20, seed=3),
        _case(f"{_kind}_m3_k3_conv", _kind, (20, 30, 40), 3, 1000, tol=1e-5 if _kind == "admm" else 1e-7, seed=4),
    ]
CASES += [
    # eight views at the unroll edges (k = 1: the width-1 view is exhausted by one deflation)
    _case("pls_m8", "pls", (1, 32, 33, 65, 96, 127, 129, 257), 1, 3, seed=5),
    _case("pmd_m8", "pmd", (1, 32, 33, 65, 96, 127, 129, 257), 1, 3, seed=6),
    _case("span_m8_k3", "span", (4, 31, 33, 64, 95, 97, 129, 255), 3, 3, seed=7),
    _case("admm_m8", "admm", (1, 32, 33, 65, 96, 127, 129, 257), 1, 3, seed=8),
    _case("elastic_m8", "elastic", (1, 32, 33, 64, 65, 97, 128, 255), 1, 2, seed=9,
          params=((0.05, 0.5),) * 8),
    _case("ipls_m8", "ipls", (1, 32, 33, 64, 65, 97, 128, 255), 1, 2, seed=10, params=((0.5, 0.0),) * 8),
    # the grid-stride loops wrap: D and both Gauss-Seidel phases exceed the warps of the grid
    _case("pls_wrap", "pls", (2400, 2400), 2, 4, seed=11, tags=("wrap",)),
    _case("span_wrap", "span", (2400, 2400), 2, 4, params=(300, 500), seed=12, tags=("wrap",)),
    _case("ipls_wrap", "ipls", (2048, 100), 2, 2, params=((0.0, 0.0), (0.05, 0.5)), seed=13, tags=("wrap",)),
    # branches by construction
    _case("pls_zero_cross", "pls", (12, 20), 2, 2, gen="zero_cross", seed=14, tags=("tn0", "norm0", "s0")),
    _case("parkhomenko_zero_view", "parkhomenko", (24, 30, 36), 2, 3, params=(1e3, 0.05, 0.05), seed=15,
          tags=("norm0", "s0")),
    _case("pmd_both_sides", "pmd", (40, 50), 2, 4, params=(50.0, 0.1), seed=16, tags=("pmd_nobisect", "pmd_bisect")),
    _case("span_tie", "span", (12, 9), 1, 1, params=(4, 9), gen="span_tie", tags=("span_tie", "span_all")),
    _case("span_zero", "span", (12, 9), 1, 1, params=(10, 12), gen="span_zero", tags=("span_thr0", "span_all")),
    _case("admm_cross", "admm", (30, 40, 50), 2, 6, params=(0.02, 0.3, 0.02), mu=10.0, j=2, seed=17,
          tags=("zn_above", "zn_below")),
    _case("elastic_mix", "elastic", (24, 32, 33, 40), 3, 4, params=MIX, seed=18, tags=("eig_cut",)),
    _case("ipls_mix", "ipls", (24, 32, 33, 40), 3, 4, params=MIX, seed=19, tags=("eig_cut",)),
    _case("ipls_means_sd0", "ipls", (20, 30, 25), 2, 3, params=((50.0, 1.0), (0.05, 0.5), (0.0, 0.0)), gen="data",
          seed=20, tags=("sd0", "means")),
    # Lasso with a tiny alpha: the first dimension converges, the deflated (singular) G_00 of the second caps a descent
    _case("elastic_capped", "elastic", (6, 8), 2, 2, params=((1e-4, 1.0), (0.05, 0.5)), seed=21, tags=("capped",)),
]
CASES = {c.name: c for c in CASES}


# ----------------------------------------------------------------------------------------------------------- inputs
def _unit_rows(rng, dims, k):
    out = []
    for _ in range(k):
        ws = [rng.standard_normal(p) for p in dims]
        out.append(np.concatenate([w / np.linalg.norm(w) for w in ws]))
    return np.vstack(out)


@functools.lru_cache(maxsize=None)
def inputs(case: AlsCase):
    """(G, init (k x D), colmeans or None): the Gram matrix the kernel iterates on and the initial weights."""
    rng = np.random.default_rng(7000 + case.seed)
    D, dims = case.D, case.dims
    off = np.concatenate([[0], np.cumsum(dims)])
    colmeans = None
    if case.gen in ("span_tie", "span_zero"):
        # integer G = L L^T + 4 I with L integer.  Row 0 of view 1 in L is e_0 and init w_1 = e_0 of view 1, so the
        # first target of view 0 is exactly the integer column L_0[:, 0] (designed ties) and ||t||^2 = G_11[0, 0]
        L = rng.integers(-2, 3, (D, 4)).astype(np.float64)
        L[off[1]] = [1.0, 0.0, 0.0, 0.0]
        L[:dims[0], 0] = [9, -7, 5, 5, -5, 3, 2, -1, 0, 0, 0, 1]     # |x| sorted: 9 7 5 5 5 3 2 1 1 0 0 0
        G = L @ L.T + 4.0 * np.eye(D)
        init = np.zeros((1, D))
        init[0, :dims[0]] = rng.integers(-3, 4, dims[0])
        init[0, off[1]] = 1.0
        return G, init, None
    if case.gen == "data":
        # uncentred Gram matrix of n rows with non-zero column means: the std of SCCA_IPLS sees the means
        n, r = case.n, 8
        Z = rng.standard_normal((n, r))
        X = Z @ rng.standard_normal((r, D)) + rng.standard_normal((n, D)) + rng.uniform(-2, 2, D)
        G, colmeans = X.T @ X, X.mean(axis=0)
    else:
        # (n - 1) C for a covariance C = (L L^T + diag) / r of unit-order entries
        r = 8
        L = rng.standard_normal((D, r)) * rng.uniform(0.5, 2.0, r)
        G = L @ L.T
        G[np.diag_indices(D)] += rng.uniform(0.5, 1.5, D) * r
        G *= (case.n - 1) / r
        if case.gen == "zero_cross":
            G[:dims[0], dims[0]:] = 0.0
            G[dims[0]:, :dims[0]] = 0.0
    return G, _unit_rows(rng, dims, case.k), colmeans


def device_params(case: AlsCase):
    """``params`` of ops.als_fit: one value per view, or the (alpha, l1) pairs flattened and the column means."""
    if not case.reg:
        return [float(p) for p in case.params]
    flat = [float(x) for pair in case.params for x in pair]
    if case.kind == "ipls":
        cm = inputs(case)[2]
        flat += list(np.zeros(case.D) if cm is None else cm)
    return flat


def device_mu(case: AlsCase):
    return RCOND if case.reg else (1.0 if case.mu is None else case.mu)


# ----------------------------------------------------------------------------------------------------------- reference
@functools.lru_cache(maxsize=None)
def reference(case: AlsCase):
    """(W (D x k), sweeps per dimension, trace) of the float64 restatement, with the device's sign convention for a
    capped coordinate descent (negated sweeps)."""
    G, init, cm = inputs(case)
    init_l = [[row[s] for s in S.block_slices(case.dims)] for row in init]
    trace = []
    if case.reg:
        W, iters = E.cov_elastic_fit(G, case.dims, case.n, case.kind, case.k, params=list(case.params), colmeans=cm,
                                     init=init_l, max_iter=case.max_iter, tol=case.tol, rcond=RCOND, trace=trace)
    else:
        W, iters = S.cov_als_fit(G, case.dims, case.n, case.kind, case.k, params=list(case.params),
                                 mu=device_mu(case), init=init_l, max_iter=case.max_iter, tol=case.tol, trace=trace)
    return np.vstack(W), iters, trace


def tolerance(case: AlsCase):
    return FIRST_TOL if case.max_iter <= 1 else LATER_TOL
