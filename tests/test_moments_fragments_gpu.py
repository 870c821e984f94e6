"""The TF32 moment kernel loads each column block as four [32 samples x 32 columns] TMA boxes with 128-byte swizzle; the
MMA warps read their A fragments straight from those boxes into registers, and the transpose warps turn the B block
into K-major shared tiles.  With small-integer inputs every value is exact in TF32 (its lo part is zero) and every
partial sum is exact in fp32, so the moments must equal the float64 X^T X and column sums exactly: any element read
from the wrong (sample, column) position shows up as a difference, not as rounding."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BLK = 128

# (view widths, n): 32-column boxes partly or wholly past a view's width (1, 31, 33, 127, 129, 300), diagonal and
# off-diagonal tiles, n a multiple of neither 32 nor 2048, and from one split to dozens of splits of many slices
SHAPES = [
    ([1], 45),
    ([31, 1, 33], 2085),
    ([33, 300, 127], 7001),
    ([127, 129, 300, 33, 1], 20011),
    ([300, 129], 66003),
]


def _padded_reference(views):
    """float64 moments in the padded block layout: X_p^T X_p on the upper block triangle (zero below), column sums."""
    cols = []
    for v in views:
        d = v.shape[1]
        cols.append(torch.nn.functional.pad(v.double(), (0, -(-d // BLK) * BLK - d)))
    X = torch.cat(cols, dim=1)
    M = X.T @ X
    nb = X.shape[1] // BLK
    blk = torch.arange(nb, device=X.device).repeat_interleave(BLK)
    M[blk[:, None] > blk[None, :]] = 0.0
    return M, X.sum(dim=0)


@pytest.mark.parametrize("precision", ["tf32", "tf32x3", "tf32x3b"])
@pytest.mark.parametrize("dims,n", SHAPES)
def test_integer_moments_are_exact(precision, dims, n):
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(n + len(dims))
    views = [torch.randint(-8, 9, (n, d), generator=g, device="cuda").float() for d in dims]
    mom = ops.moments(views, precision=precision)
    M_ref, s_ref = _padded_reference(views)
    Dp = M_ref.shape[0]
    assert mom.numel() == Dp * Dp + Dp
    M = mom[:Dp * Dp].view(Dp, Dp)
    bad = (M != M_ref).nonzero()
    assert bad.numel() == 0, (f"{bad.shape[0]} of {Dp * Dp} moment entries differ, first at {bad[0].tolist()}: "
                              f"{M[tuple(bad[0])].item()} vs {M_ref[tuple(bad[0])].item()}")
    assert torch.equal(mom[Dp * Dp:], s_ref), "column sums differ"
