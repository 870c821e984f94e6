"""The CCAR3 kernels on the GPU: ccab_ccar3_admm iterate for iterate against the float64 restatement
oracle/ccar3.py:admm_inverse (iteration counts, stop flag, residuals, exact zero rows) at every shape it branches on,
and ccab_row_norm4_sum against float64 numpy."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import ops
from oracle import ccar3 as O

pytestmark = pytest.mark.gpu


def _problem(p, q, seed):
    rng = np.random.default_rng(seed)
    n = max(2 * p // 3, 2)
    X = rng.standard_normal((n, p)) / np.sqrt(p)
    Sx = X.T @ X / n
    M = np.linalg.inv(Sx + (1.0 + 1e-8) * np.eye(p))
    B0 = M @ (rng.standard_normal((p, q)) / np.sqrt(p * q))
    return M, B0


def _kappa(B0, which):
    """lambda / rho: 0, just under the median row norm of B0 (about half the rows zeroed, no row norm equal to it), or
    above every row norm."""
    nrm = np.linalg.norm(B0, axis=1)
    return {"zero": 0.0, "mid": 0.97 * float(np.median(nrm)), "all": 2.0 * float(nrm.max()) + 1.0}[which]


def _run(M, B0, kappa, tol, max_iter):
    dev = torch.device("cuda")
    Z, U, info = ops.ccar3_admm(torch.from_numpy(M).to(dev), torch.from_numpy(B0).to(dev), kappa, 1.0, tol, max_iter)
    return Z.cpu().numpy(), U.cpu().numpy(), info.cpu().numpy()


@pytest.mark.parametrize("max_iter", [1, 2, 7])
@pytest.mark.parametrize("which", ["zero", "mid", "all"])
@pytest.mark.parametrize("p,q", [(1, 1), (37, 3), (1000, 129), (4096, 3), (37, 512), (1000, 1)])
def test_admm_iterate_for_iterate(p, q, which, max_iter):
    M, B0 = _problem(p, q, p + q)
    kappa = _kappa(B0, which)
    Zr, Ur, it, pr, du, st = O.admm_inverse(M, B0, kappa, 1.0, 1e-300, max_iter)
    Z, U, info = _run(M, B0, kappa, 1e-300, max_iter)
    assert int(info[0]) == it == max_iter and info[3] == 0.0
    scale = max(float(np.abs(Zr).max()), float(np.abs(B0).max()))
    np.testing.assert_allclose(Z, Zr, rtol=0, atol=1e-12 * scale)
    np.testing.assert_allclose(U, Ur, rtol=0, atol=1e-12 * scale)
    np.testing.assert_allclose(info[1:3], [pr, du], rtol=1e-9, atol=1e-12 * scale)
    zero_r, zero = np.linalg.norm(Zr, axis=1) == 0, np.linalg.norm(Z, axis=1) == 0
    assert np.array_equal(zero, zero_r)
    if which == "all":
        assert zero.all()


@pytest.mark.parametrize("which", ["zero", "mid"])
@pytest.mark.parametrize("p,q", [(37, 3), (1000, 129), (300, 512)])
def test_admm_stops_where_the_restatement_stops(p, q, which):
    """tol is placed between the restatement's stop statistics of iterations 10 and 11 (geometric mean; the statistic
    falls monotonically here): the loop must stop exactly after iteration 11."""
    M, B0 = _problem(p, q, 3 * p + q)
    kappa = _kappa(B0, which)
    trace = []
    O.admm_inverse(M, B0, kappa, 1.0, 1e-300, 12, trace)
    stat = np.array([max(t["primal"], t["dual"]) for t in trace])
    j = 10
    assert np.all(np.diff(stat) < 0)
    tol = float(np.sqrt(stat[j - 1] * stat[j]))
    _, _, it, _, _, st = O.admm_inverse(M, B0, kappa, 1.0, tol, 5000)
    assert st and it == j + 1
    _, _, info = _run(M, B0, kappa, tol, 5000)
    assert int(info[0]) == it and info[3] == 1.0
    assert max(info[1], info[2]) < tol


def test_admm_reruns_are_bit_identical():
    M, B0 = _problem(2048, 256, 1)
    a = _run(M, B0, _kappa(B0, "mid"), 1e-8, 50)
    b = _run(M, B0, _kappa(B0, "mid"), 1e-8, 50)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_admm_rejects_out_of_range_shapes():
    dev = torch.device("cuda")
    with pytest.raises(ValueError, match="q <= 512"):
        ops.ccar3_admm(torch.eye(4, dtype=torch.float64, device=dev), torch.zeros((4, 513), dtype=torch.float64,
                                                                                   device=dev), 0.0, 1.0, 1e-4, 10)


@pytest.mark.parametrize("n", [1, 31, 1_000_000])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_row_norm4_sum(n, dtype):
    rng = np.random.default_rng(n)
    d = 7
    Y = (1e4 + rng.standard_normal((n, d))).astype(np.float32 if dtype == torch.float32 else np.float64)
    mean = Y.astype(np.float64).mean(axis=0)
    want = float(np.sum(np.sum((Y.astype(np.float64) - mean) ** 2, axis=1) ** 2))
    dev = torch.device("cuda")
    got = ops.row_norm4_sum(torch.from_numpy(Y).to(dev), torch.from_numpy(mean).to(dev)).item()
    assert abs(got - want) <= 1e-12 * max(abs(want), 1e-300)


def test_row_norm4_sum_strided_view():
    rng = np.random.default_rng(3)
    big = rng.standard_normal((500, 40))
    dev = torch.device("cuda")
    t = torch.from_numpy(big).to(dev)[::3, 5:38]          # row stride 120, column offset 5
    Y = big[::3, 5:38]
    mean = Y.mean(axis=0)
    want = float(np.sum(np.sum((Y - mean) ** 2, axis=1) ** 2))
    got = ops.row_norm4_sum(t, torch.from_numpy(mean).to(dev)).item()
    assert abs(got - want) <= 1e-12 * want
    a = ops.row_norm4_sum(t, torch.from_numpy(mean).to(dev)).item()
    assert a == got
