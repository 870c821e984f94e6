"""The Khatri-Rao adjoint ``ccab_tcca_moment_adjoint`` (``ops.tcca_moment_adjoint``) against the float64 einsum of
oracle/tccaloss.py at every edge of its tiling: n below, at and past the 64-sample tile and not a multiple of the
16-wide reduction step; k_i and P_i = prod_{j != i} k_j on both sides of 64 and P_i = 1; 2 to 8 modes, so every mode
position (first, middle, last) is read through its own strides; the 2^25-entry limit accepted and exceeded; the
device scale; and bit-identical repeat calls (the kernel has no sample or reduction splits)."""
import ctypes as C

import numpy as np
import pytest
import torch

from cca_zoo_b200 import _lib, ops
from oracle import tccaloss as O

pytestmark = pytest.mark.gpu

SHAPES = [
    ((5, 4), 100), ((3, 4, 5), 37), ((2, 3, 2, 3), 64), ((2, 2, 3, 2, 2), 65), ((2, 2, 2, 2, 2, 2), 33),
    ((2, 1, 2, 2, 3, 1, 2), 20), ((2, 3, 2, 2, 1, 2, 3, 2), 129),
    ((1, 1), 10), ((70, 1), 50), ((1, 70), 17), ((63, 64), 37), ((64, 65), 16), ((65, 63, 2), 48),
    ((129, 1, 70), 100), ((1, 129, 1), 9), ((7, 5, 3), 1), ((7, 5, 3), 15), ((33, 2, 33), 200), ((9, 4), 1001),
]


def _check(dims, n, seed):
    rng = np.random.default_rng(seed)
    H = [rng.standard_normal((n, p)) for p in dims]
    M = rng.standard_normal(dims)
    want = O.adjoint(M, H)
    Hd = [torch.from_numpy(h).cuda() for h in H]
    Md = torch.from_numpy(M).cuda()
    got = [y.cpu().numpy() for y in ops.tcca_moment_adjoint(Md, Hd, scale=0.5)]
    for i, (g, w) in enumerate(zip(got, want)):
        # every entry is a dot product of length P_i: bound its rounding by P_i u times the sum of |terms|
        absw = O.adjoint(np.abs(M), [np.abs(h) for h in H])[i]
        err = np.abs(g - 0.5 * w)
        assert (err <= 0.5 * absw * (M.size // dims[i] + 2) * 2.3e-16).all(), f"mode {i}: {err.max():.3e}"
    return Md, Hd, got


@pytest.mark.parametrize("dims,n", SHAPES)
def test_adjoint_matches_einsum(dims, n):
    _check(dims, n, sum(dims) + n)


def test_repeat_calls_are_bit_identical_and_the_device_scale_applies():
    Md, Hd, got = _check((33, 2, 70), 300, 1)
    again = ops.tcca_moment_adjoint(Md, Hd, scale=0.5)
    assert all(torch.equal(a, torch.from_numpy(b).cuda()) for a, b in zip(again, got))
    f = torch.tensor([-3.0], dtype=torch.float64, device="cuda")
    scaled = ops.tcca_moment_adjoint(Md, Hd, scale=0.5, scale_dev=f)
    assert all(torch.equal(s, -3.0 * a) for s, a in zip(scaled, again))   # powers of two and 3: exact


def test_limit_of_2_25_entries_is_accepted():
    """Five views of width 32: M has exactly 2^25 entries.  <Y_i, H_i> = n ||M||^2 for every mode with M the
    contraction of the same H, and the full einsum for the last mode."""
    n, dims = 20, (32,) * 5
    rng = np.random.default_rng(7)
    H = [torch.from_numpy(rng.standard_normal((n, p))).cuda() for p in dims]
    M = ops.tcca_moment(H)
    Y = ops.tcca_moment_adjoint(M, H)
    sq = float((M * M).sum())
    for y, h in zip(Y, H):
        assert abs(float((y * h).sum()) - n * sq) <= 1e-12 * n * sq
    Mh = M.cpu().numpy().reshape(dims)
    want = np.einsum("abcde,za,zb,zc,zd->ze", Mh, *[h.cpu().numpy() for h in H[:4]], optimize=True)
    assert np.abs(Y[4].cpu().numpy() - want).max() <= 1e-12 * np.abs(want).max()


def test_more_than_2_25_entries_is_rejected_before_any_launch():
    lib = _lib.load()
    dims = [4097, 4096, 2]
    dummy = torch.zeros(1, dtype=torch.float64, device="cuda")
    ptrs = (C.c_void_p * 3)(*[dummy.data_ptr()] * 3)
    before = lib.ccab_launch_count()
    rc = lib.ccab_tcca_moment_adjoint(3, _lib.i64_array(dims), 4, C.c_void_p(dummy.data_ptr()), ptrs,
                                      _lib.i64_array(dims), 1.0, None, ptrs, _lib.i64_array(dims), None)
    assert rc != 0 and "2^25" in _lib.last_error()
    assert lib.ccab_launch_count() == before
