"""The TCCA kernels against float64 restatements: ``krprod_moment`` (``ops.tcca_moment``) against an einsum at every
shape it branches on (2 to 8 views, ragged widths around the 64-wide tile, n below one k step and not a multiple of
it, split and unsplit plans, more tiles than CTAs), and ``ccab_tcca_fit`` (``ops.tcca_fit``) state by state against
oracle/tcca.py: after the start and after 1, 2 and 100 iterations, the stop flag, k = 1 and 64, k > p_j."""
import numpy as np
import pytest
import torch

from cca_zoo_b200 import ops
from cca_zoo_b200.datasets import conftest_views
from oracle import tcca as O

pytestmark = pytest.mark.gpu


def _einsum_moment(Z):
    n = Z[0].shape[0]
    kr = Z[1]
    for z in Z[2:]:
        kr = np.einsum("sa,sb->sab", kr, z).reshape(n, -1)
    return np.einsum("sa,sb->ab", Z[0], kr) / n


MOMENT_SHAPES = [
    ((5, 4), 100), ((3, 4, 5), 100), ((2, 3, 2, 3), 50), ((2, 2, 3, 2, 2), 40), ((2, 2, 2, 2, 2, 2), 33),
    ((2, 1, 2, 2, 3, 1, 2), 20), ((2, 2, 1, 2, 2, 2, 1, 2), 17),
    ((1, 1), 10), ((63, 64), 37), ((64, 65), 16), ((65, 63, 2), 48), ((129, 1, 70), 100), ((1, 129, 1), 9),
    ((7, 5, 3), 1), ((7, 5, 3), 15), ((9, 4), 1001),
    ((6, 5), 200000),            # few tiles, many samples: split over n
    ((130, 130, 70), 300),       # 429 output tiles: more tiles than CTAs at once
]


@pytest.mark.parametrize("dims,n", MOMENT_SHAPES)
def test_krprod_moment_matches_einsum(dims, n):
    rng = np.random.default_rng(sum(dims) + n)
    Z = [rng.standard_normal((n, p)) for p in dims]
    want = _einsum_moment(Z)
    Zd = [torch.from_numpy(z).cuda() for z in Z]
    got = ops.tcca_moment(Zd).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * max(1.0, float(np.abs(want).max())) * np.sqrt(n))
    again = ops.tcca_moment(Zd).cpu().numpy()
    np.testing.assert_array_equal(got, again)


@pytest.mark.parametrize("nsplit", [1, 3, 7])
def test_krprod_moment_split_plans(nsplit):
    rng = np.random.default_rng(nsplit)
    Z = [rng.standard_normal((5000, p)) for p in (9, 7, 5)]
    want = _einsum_moment(Z)
    Zd = [torch.from_numpy(z).cuda() for z in Z]
    got = ops.tcca_moment(Zd, nsplit=nsplit).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-13 * np.sqrt(5000))
    np.testing.assert_array_equal(got, ops.tcca_moment(Zd, nsplit=nsplit).cpu().numpy())


def test_krprod_moment_strided_views_unmodified():
    rng = np.random.default_rng(5)
    big = torch.from_numpy(rng.standard_normal((300, 20))).cuda()
    Z = [big[:, :7], big[:, 7:12], big[:, 12:20]]
    before = big.clone()
    got = ops.tcca_moment(Z).cpu().numpy()
    np.testing.assert_allclose(got, _einsum_moment([z.cpu().numpy() for z in Z]), rtol=0, atol=1e-12)
    assert torch.equal(big, before)


# ----------------------------------------------------------------------------------------------------------------------
def _tensor(dims, seed):
    rng = np.random.default_rng(seed)
    n = 200
    z = rng.standard_normal((n, 2))
    views = [z @ rng.standard_normal((2, p)) + rng.standard_normal((n, p)) for p in dims]
    return O.tensor_of(views)[0]


def _compare(dev_state, st, dims, k, tol):
    d = ops.decode_tcca_state(dev_state.cpu().numpy(), dims, k)
    assert d["iters"] == st["iters"] and d["stop"] == st["stop"] and not d["singular"]
    for a, b in zip(d["F"], st["F"]):
        assert float(np.abs(a - b).max()) <= tol * max(1.0, float(np.abs(b).max()))
    np.testing.assert_allclose(d["rec"], st["rec"], rtol=tol, atol=0)
    return d


@pytest.mark.parametrize("dims,k,seed", [((10, 8, 6), 2, 0), ((10, 8, 6), 1, 1), ((5, 4, 6, 3), 3, 2),
                                         ((6, 3, 4), 5, 3), ((3, 2, 4, 2, 3), 2, 4)])
def test_tcca_fit_state_by_state(dims, k, seed):
    M = _tensor(dims, seed)
    rand = O.random_columns(M.shape, k, np.random.RandomState(seed))
    st = O.gram_start(M, k, rand)
    Md = torch.from_numpy(M).cuda()
    state = ops.tcca_fit(Md, dims, k, 0, rand=rand)
    _compare(state, st, dims, k, 1e-12)
    for steps in (1, 1, 98):
        for _ in range(steps):
            O.als_step(st, M)
        state = ops.tcca_fit(Md, dims, k, steps, state=state)
        _compare(state, st, dims, k, 1e-12 if st["iters"] <= 2 else 1e-9)


def test_tcca_fit_stop_flag_and_rerun_bits():
    M = _tensor((10, 8, 6), 0)
    st = O.gram_start(M, 2, [None] * 3)
    for _ in range(100):
        O.als_step(st, M)
        if st["stop"]:
            break
    assert st["stop"] and st["iters"] < 100
    Md = torch.from_numpy(M).cuda()
    a = ops.tcca_fit(Md, (10, 8, 6), 2, 100, rand=[None] * 3)
    d = _compare(a, st, (10, 8, 6), 2, 1e-9)
    assert d["stop"]
    more = ops.tcca_fit(Md, (10, 8, 6), 2, 5, state=a.clone())          # a stopped fit does nothing
    assert torch.equal(more, a)
    b = ops.tcca_fit(Md, (10, 8, 6), 2, 100, rand=[None] * 3)
    assert torch.equal(a, b)


def test_tcca_fit_k64():
    dims = (64, 65, 66)
    rng = np.random.default_rng(9)
    M = rng.standard_normal(dims) / 100.0
    st = O.gram_start(M, 64, [None, None, None])
    Md = torch.from_numpy(M).cuda()
    state = ops.tcca_fit(Md, dims, 64, 0)
    _compare(state, st, dims, 64, 1e-11)
    O.als_step(st, M)
    state = ops.tcca_fit(Md, dims, 64, 1, state=state)
    _compare(state, st, dims, 64, 1e-9)


def test_tcca_fit_three_views_fixture_k_gt_p():
    views = conftest_views("three_views")
    M = O.tensor_of(views)[0]
    rand = O.random_columns(M.shape, 8, np.random.RandomState(0))
    st = O.gram_start(M, 8, rand)
    Md = torch.from_numpy(M).cuda()
    state = ops.tcca_fit(Md, M.shape, 8, 0, rand=rand)
    _compare(state, st, M.shape, 8, 1e-12)
    for _ in range(2):
        O.als_step(st, M)
    state = ops.tcca_fit(Md, M.shape, 8, 2, state=state)
    _compare(state, st, M.shape, 8, 1e-11)
