"""TEST INFRASTRUCTURE ONLY: the case table of tests/test_ey_kernel_gpu.py (the EY step kernel ``ey_steps`` of
csrc/ey.cu, driven through ``ops.ey_fit``) and the float64 reference half of every case.

Each case builds its inputs from a seed (a unit-diagonal SPD covariance for the covariance route, raw views of a latent
model for the mini-batch route, orthonormal initial weights scaled down, a learning rate from a bound on the largest
eigenvalue) and runs tests/fake_ops_ey.EyFit, i.e. ``oracle.ey.cov_step`` / ``mb_step`` in float64 numpy, with the
same call schedule the device fit gets.  ``ref_block`` lays the reference state out as the device state block:
header (prev objective, steps, stop flag, last |prev - obj|, 4 unused) | W (k x D) | velocity (k x D).

The shapes are picked where the kernel branches: k = 1 and k = 32 (= kEyMaxK), up to 8 views of ragged widths (1, 31,
33, 127-129: dead lanes of a 32-feature tile and several 128-column rounds), D > 16 x 132 (the row-tile loop of the
covariance products wraps even at two CTAs per SM of an H100 SXM), batches of 2, 3, 127, 128, 129, 8192, 8193 and
~20000 rows (one slice, ragged last slices, slices longer than 128 rows) and column slices of wider tensors.  In every
mini-batch case the row strides ascend with the view index, so a kernel that applied view 0's stride to another view
would read wrong rows inside that view's buffer rather than past its end.

tests/test_ey_kernel_cases_cpu.py checks on the CPU that no case is vacuous: the reference stays finite, the weights
move, and the stop case's deltas keep their margins from ``tol``.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np
import torch

from tests import fake_ops_ey

HEADER = 8                 # ops.EY_HEADER
MOMENTUM = 0.9
SMS_H100 = 132             # SMs of an H100 SXM: the large-D cases are sized against it
FIRST_TOL = 1e-12          # after one step, relative to max |.|
LATER_TOL = 1e-10          # after a few tens of steps
MOVE = 1e-3                # a case must move W by more than this fraction of |W_0| (Frobenius)


@dataclass(frozen=True)
class CovCase:
    name: str
    dims: tuple
    k: int
    c: float
    steps: int = 24
    lr_scale: float = 0.05
    init_scale: float = 0.5
    seed: int = 0

    @property
    def D(self):
        return sum(self.dims)


@dataclass(frozen=True)
class MbCase:
    name: str
    dims: tuple
    k: int
    c: float
    bs: int
    dtype: str             # "f32" | "f64"
    strided: bool          # column slice of a wider tensor with an odd row stride
    steps: int = 20
    n: int = 3001
    lr_scale: float = 0.05
    init_scale: float = 0.5
    seed: int = 0

    @property
    def D(self):
        return sum(self.dims)


COV_CASES = [
    CovCase("k1_w1_1", (1, 1), 1, 0.0),
    CovCase("k1_w1_2_31", (1, 2, 31), 1, 0.3),
    CovCase("k32_w32_33", (32, 33), 32, 1.0),
    CovCase("k1_m8_ragged", (1, 2, 31, 32, 33, 127, 128, 129), 1, 0.3),
    CovCase("k32_m8", (32, 33, 40, 47, 64, 65, 100, 129), 32, 0.0),
    CovCase("k17_largeD", (2048, 1536, 700), 17, 0.3, steps=20),
    CovCase("k32_largeD", (2048, 1536, 700), 32, 1.0, steps=20),
    CovCase("k3_w4000_96", (4000, 96), 3, 0.0, steps=20),
]
COV = {c.name: c for c in COV_CASES}

# a covering list over dtype x layout x batch x k x m x c, not the full product; widths ascend within each case
MB_CASES = [
    MbCase("bs2_k1_m2", (1, 3), 1, 0.0, 2, "f64", False),
    MbCase("bs2_k5_m3", (5, 31, 33), 5, 1.0, 2, "f32", True),
    MbCase("bs3_k1_m2", (2, 31), 1, 1.0, 3, "f32", True),
    MbCase("bs3_k5_m4", (5, 31, 33, 257), 5, 0.0, 3, "f64", False),
    MbCase("bs127_k5_m3", (5, 31, 33), 5, 0.0, 127, "f64", True),
    MbCase("bs127_k32_m2", (32, 33), 32, 0.0, 127, "f64", True),
    MbCase("bs128_k5_m2", (31, 33), 5, 1.0, 128, "f32", False),
    MbCase("bs128_k32_m2", (32, 129), 32, 1.0, 128, "f64", False),
    MbCase("bs129_k1_m4", (1, 31, 33, 40), 1, 0.0, 129, "f32", True),
    MbCase("bs129_k5_m2", (5, 33), 5, 1.0, 129, "f64", False),
    MbCase("bs129_k32_m8", (32, 33, 34, 40, 47, 64, 129, 200), 32, 1.0, 129, "f32", True),
    MbCase("bs8192_k5_m3", (8, 31, 33), 5, 0.0, 8192, "f64", False),
    MbCase("bs8192_k1_m4", (1, 31, 33, 130), 1, 1.0, 8192, "f32", False),
    MbCase("bs8193_k1_m2", (1, 33), 1, 1.0, 8193, "f32", True),
    MbCase("bs8193_k1_m8", (1, 2, 5, 31, 32, 33, 64, 129), 1, 0.0, 8193, "f64", True),
    MbCase("bs8193_k5_m8", (5, 6, 7, 31, 33, 33, 64, 100), 5, 0.0, 8193, "f32", False),
    MbCase("bs20000_k32_m3", (32, 40, 300), 32, 0.0, 20000, "f32", False),
    MbCase("bs20000_k1_m2", (1, 31), 1, 1.0, 20000, "f64", True),
    MbCase("bs19999_k5_m4", (5, 33, 64, 129), 5, 0.0, 19999, "f64", False),
    MbCase("bs20001_k5_m2", (5, 33), 5, 1.0, 20001, "f32", True),
]
MB = {c.name: c for c in MB_CASES}

# chunking: the same fit as one call, as 5 + 7 steps and as 12 one-step calls
CHUNK_COV = CovCase("chunk_cov", (31, 33, 40), 5, 0.3, steps=12)
CHUNK_MB = {dt: MbCase(f"chunk_mb_{dt}", (1, 31, 33), 1, 0.3, 129, dt, True, steps=12) for dt in ("f32", "f64")}

# stop: tol is picked from the reference's deltas (stop_plan); the fit starts above the optimum's scale so that the
# deltas shrink as it settles
STOP_CASE = CovCase("stop", (5, 7, 9), 2, 0.3, steps=40, lr_scale=0.1, init_scale=1.5, seed=3)
# divergence: a learning rate far beyond the stable range on the unregularised loss
DIVERGE_CASE = CovCase("diverge", (31, 33), 3, 0.0, steps=200, lr_scale=40.0)


# ----------------------------------------------------------------------------------------------------------- inputs
def orthonormal_init(rng, dims, k, scale):
    return np.vstack([scale * np.linalg.qr(rng.standard_normal((p, k)))[0] for p in dims])


@functools.lru_cache(maxsize=None)
def cov_inputs(case: CovCase):
    """(C, init, lr): C = S (L L^T + I) S with S making the diagonal one, L (D x 4) Gaussian loadings shared by all
    views (the cross-view correlation); lr = lr_scale * m / (4 lambda_max bound)."""
    rng = np.random.default_rng(1000 + case.seed)
    D, m = case.D, len(case.dims)
    L = 0.5 * rng.standard_normal((D, 4))
    s = 1.0 / np.sqrt((L * L).sum(axis=1) + 1.0)
    SL = s[:, None] * L
    C = SL @ SL.T
    C[np.diag_indices(D)] += s * s
    C[np.diag_indices(D)] = 1.0
    lam = np.linalg.norm(SL, 2) ** 2 + float((s * s).max())
    init = orthonormal_init(rng, case.dims, case.k, case.init_scale)
    return C, init, case.lr_scale * m / (4.0 * lam)


@functools.lru_cache(maxsize=None)
def mb_inputs(case: MbCase):
    """(views, init, lr, idx): raw views (n x p, the case's dtype, contiguous) of a 4-factor latent model with non-zero
    column means; lr = lr_scale * m / (4 trace of the covariance); idx (steps x bs) int32 with row 0, row n - 1 and
    repeated rows in it."""
    rng = np.random.default_rng(2000 + case.seed)
    n, m = case.n, len(case.dims)
    Z = rng.standard_normal((n, 4))
    views, trace = [], 0.0
    for p in case.dims:
        X = Z @ (0.5 * rng.standard_normal((p, 4))).T + rng.standard_normal((n, p)) + 0.5 * rng.standard_normal(p)
        X = X.astype(np.float32 if case.dtype == "f32" else np.float64)
        trace += float(X.astype(np.float64).var(axis=0, ddof=1).sum())
        views.append(X)
    init = orthonormal_init(rng, case.dims, case.k, case.init_scale)
    idx = rng.integers(0, n, (case.steps, case.bs))
    idx[0::2, 0] = 0
    idx[1::2, -1] = n - 1
    if case.bs >= 4:
        idx[:, case.bs // 2] = idx[:, 1]
    return views, init, case.lr_scale * m / (4.0 * trace), idx.astype(np.int32)


def row_strides(case: MbCase):
    """Row stride of each view: its width (contiguous), or an odd stride a few columns wider (column slice).  Both
    ascend with the view index."""
    if not case.strided:
        return [p for p in case.dims]
    return [(p + 3 + 2 * i) | 1 for i, p in enumerate(case.dims)]


# ----------------------------------------------------------------------------------------------------------- reference
def ref_fit(case, tol=0.0):
    """tests/fake_ops_ey.EyFit on the case's inputs (float64 numpy)."""
    if isinstance(case, CovCase):
        C, init, lr = cov_inputs(case)
        return fake_ops_ey.EyFit(case.dims, init, case.c, lr, MOMENTUM, tol, cov=torch.from_numpy(C))
    views, init, lr, _ = mb_inputs(case)
    return fake_ops_ey.EyFit(case.dims, init, case.c, lr, MOMENTUM, tol, views=[torch.from_numpy(v) for v in views],
                             batch=case.bs)


def ref_block(st):
    """The reference state laid out as the device state block."""
    W = np.vstack(st["W"]).T.reshape(-1)
    V = np.vstack(st["vel"]).T.reshape(-1)
    hdr = np.zeros(HEADER)
    hdr[:4] = st["prev"], st["steps"], float(st["stop"]), st["deltas"][-1] if st["deltas"] else 0.0
    return np.concatenate([hdr, W, V])


def ref_run(case, calls, tol=0.0):
    """Reference state blocks after each call of ``calls`` (step counts), the index rows sliced to match."""
    fit = ref_fit(case, tol)
    idx = None if isinstance(case, CovCase) else torch.from_numpy(mb_inputs(case)[3])
    out, start = [], 0
    with np.errstate(all="ignore"):
        for n in calls:
            fit.run(n, None if idx is None else idx[start:start + n])
            out.append(ref_block(fit.st))
            start += n
    return out


@functools.lru_cache(maxsize=None)
def ref_schedule(case):
    """The compared schedule of a case: one step (FIRST_TOL), then the rest (LATER_TOL)."""
    return (1, case.steps - 1), ref_run(case, (1, case.steps - 1))


def split_block(block, k, D):
    return block[:HEADER], block[HEADER:HEADER + k * D], block[HEADER + k * D:]


@functools.lru_cache(maxsize=None)
def stop_plan(case=STOP_CASE, ratio=1.01):
    """(tol, s, calls): the first step s >= 6 whose delta lies below every earlier one by the factor ``ratio``, tol
    their geometric mean, and three calls of which the second holds step s (at its second position)."""
    fit = ref_fit(case)
    with np.errstate(all="ignore"):
        fit.run(case.steps)
    deltas = fit.st["deltas"]
    for s in range(6, case.steps - 6):
        lo, hi = deltas[s - 1], min(deltas[:s - 1])
        if np.isfinite(lo) and lo * ratio < hi:
            return float(np.sqrt(lo * hi)), s, (s - 2, 4, 4)
    raise AssertionError(f"no step of {case.name} can be a clean stop: deltas {deltas}")
