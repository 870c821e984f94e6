"""The tf32x3b moment kernel computes pair tiles: A blocks (2i, 2i + 1) against a B block j >= 2i.  A j = 2i tile loads
one block and computes only the diagonal block, a j = 2i + 1 tile uses the second A block as B, a j > 2i + 1 tile loads
B on its own; the j <= 2i + 1 tiles write block j's column sums, and an odd block count leaves a lone last block.

11 blocks in three ragged views (widths 300, 520, 257) give every tile kind at several i next to each other, pairs that
straddle a view boundary and a lone last block.  They are checked bit for bit on small integers (every value exact in
TF32 and bf16, every fp32 partial sum exact) and against the float64 emulation of the tf32x3b operand rounding on data
with large lo parts; n = 150001 runs 74 splits of the sample axis."""
import pytest
import torch

from tests.test_moments_fragments_gpu import _padded_reference
from tests.test_moments_x3b_gpu import (_emulated_x3b, _hi, _large_lo, _moments, _normalised, _padded,
                                        _real_columns)

pytestmark = pytest.mark.gpu

MANY_BLOCKS = [300, 520, 257]


@pytest.mark.parametrize("precision", ["tf32", "tf32x3", "tf32x3b"])
def test_integer_moments_of_eleven_blocks_are_exact(precision):
    from cca_zoo_b200 import ops

    n = 9001
    g = torch.Generator(device="cuda").manual_seed(n + len(MANY_BLOCKS))
    views = [torch.randint(-8, 9, (n, d), generator=g, device="cuda").float() for d in MANY_BLOCKS]
    mom = ops.moments(views, precision=precision)
    M_ref, s_ref = _padded_reference(views)
    Dp = M_ref.shape[0]
    assert Dp == 11 * 128 and mom.numel() == Dp * Dp + Dp
    M = mom[:Dp * Dp].view(Dp, Dp)
    bad = (M != M_ref).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} of {Dp * Dp} moment entries differ, first at {bad[0].tolist()}: "
                              f"{M[tuple(bad[0])].item()} vs {M_ref[tuple(bad[0])].item()}")
    assert torch.equal(mom[Dp * Dp:], s_ref), "column sums differ"


@pytest.mark.parametrize("dims,n", [(MANY_BLOCKS, 9001), ([129, 40], 150001)])
def test_pair_tiles_match_the_emulated_operand_rounding(dims, n):
    g = torch.Generator(device="cuda").manual_seed(n + 7 * len(dims))
    views = [_large_lo(n, d, g) for d in dims]
    M, s = _moments(views, "tf32x3b")
    X = _padded(views)
    E = _emulated_x3b(X)
    X64 = X.double()
    exact = X64.T @ X64
    err = _normalised(M, E, views)
    assert err.max().item() < 5e-5, f"tf32x3b differs from its emulation by {err.max().item():.2e}"
    c = _real_columns(views)
    hi = _hi(X).double()
    cross = (torch.diagonal(E) - (hi * hi).sum(dim=0))[c] / torch.diagonal(exact)[c]
    assert cross.min().item() > 2e-4, "the test data must have large lo parts"
    assert _normalised(M, exact, views).max().item() < 5e-5
    ref_s = X64.sum(dim=0)
    assert ((s - ref_s).abs() / X64.abs().sum(dim=0).clamp_min(1e-30)).max().item() < 1e-5, "column sums differ"
