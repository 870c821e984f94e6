"""The reference half of tests/test_ey_kernel_gpu.py on the CPU: every case of tests/ey_kernel_cases.py must be worth
comparing (the float64 reference stays finite and the weights move), its shapes must reach the kernel branches the
table is there for, and the stop and divergence cases must behave as the GPU tests expect.  A badly chosen case fails
here rather than on the GPU."""
import numpy as np
import pytest

from tests import ey_kernel_cases as K

ALL = K.COV_CASES + K.MB_CASES + [K.CHUNK_COV, *K.CHUNK_MB.values()]


def _init(case):
    return (K.cov_inputs(case) if isinstance(case, K.CovCase) else K.mb_inputs(case))[1]


@pytest.mark.parametrize("case", ALL, ids=lambda c: c.name)
def test_ey_kernel_case_is_not_vacuous(case):
    calls, blocks = K.ref_schedule(case)
    init = _init(case)
    assert init.shape == (case.D, case.k) and 1 <= case.k <= min(case.dims) and case.k <= 32
    for b in blocks:
        assert np.isfinite(b[0]) and np.isfinite(b[K.HEADER:]).all()
    h, W, _ = K.split_block(blocks[-1], case.k, case.D)
    assert h[1] == case.steps and h[2] == 0.0
    W0 = init.T.reshape(-1)
    assert np.linalg.norm(W - W0) > K.MOVE * np.linalg.norm(W0), "the weights barely move"


def test_ey_kernel_cases_cover_the_branches():
    cov, mb = K.COV_CASES, K.MB_CASES
    assert {c.c for c in cov} == {0.0, 0.3, 1.0}
    assert {1, 32} <= {c.k for c in cov} and any(len(c.dims) == 8 and c.k == 32 for c in cov)
    assert any(len(c.dims) == 8 and c.k == 1 and {1, 31, 33, 127, 128, 129} <= set(c.dims) for c in cov)
    large = [c for c in cov if c.D > 16 * K.SMS_H100]
    assert {c.k for c in large} == {3, 17, 32}
    assert 8 * K.SMS_H100 < 2 * 32 ** 2               # k = 32 wraps the 2k^2 loops at one CTA per SM
    assert {2, 3, 127, 128, 129, 8192, 8193} <= {c.bs for c in mb} and max(c.bs for c in mb) > 8192 * 2
    assert {c.dtype for c in mb} == {"f32", "f64"} and {c.strided for c in mb} == {False, True}
    assert {c.k for c in mb} == {1, 5, 32} and {len(c.dims) for c in mb} == {2, 3, 4, 8}
    assert {c.c for c in mb} == {0.0, 1.0} and {1, 31, 33} <= {p for c in mb for p in c.dims}
    for c in mb:
        ld = K.row_strides(c)
        assert list(ld) == sorted(ld) and all(s >= p for s, p in zip(ld, c.dims))
        assert not c.strided or all(s % 2 == 1 and s >= p + 3 for s, p in zip(ld, c.dims))
        idx = K.mb_inputs(c)[3]
        assert idx.shape == (c.steps, c.bs) and idx.dtype == np.int32
        assert 0 in idx and c.n - 1 in idx and idx.min() >= 0 and idx.max() < c.n
        assert any(len(np.unique(r)) < c.bs for r in idx) or c.bs < 4
    # nslices = min(64, ceil(bs / 128)) slices of ceil(bs / nslices) rows: the last one is short unless nslices | bs
    ragged = {c.bs for c in mb if c.bs % min(64, -(-c.bs // 128)) != 0}
    assert {129, 8193, 19999, 20001} <= ragged


def test_ey_kernel_stop_case_margins():
    tol, s, calls = K.stop_plan()
    case = K.STOP_CASE
    assert calls[0] < s <= calls[0] + calls[1]
    fit = K.ref_fit(case)
    fit.run(s)
    deltas = fit.st["deltas"]
    for j, d in enumerate(deltas):
        assert abs(d - tol) > 1e-3 * tol, f"step {j + 1}: delta {d} is within 1e-3 of tol {tol}"
        assert (d < tol) == (j + 1 == s)
    blocks = K.ref_run(case, calls, tol)
    assert blocks[1][1] == s and blocks[1][2] == 1.0 and np.array_equal(blocks[1], blocks[2])


def test_ey_kernel_divergent_case_ends_in_nan():
    case = K.DIVERGE_CASE
    h, W, _ = K.split_block(K.ref_run(case, (case.steps,))[0], case.k, case.D)
    assert np.isnan(W).all() and h[1] == case.steps and h[2] == 0.0
    fit = K.ref_fit(case)
    with np.errstate(all="ignore"):
        fit.run(case.steps // 2)
    assert np.isnan(np.vstack(fit.st["W"])).all(), "the divergence comes too late to be robust"
