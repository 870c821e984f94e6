"""The tf32x3b moment kernel: hi*hi as a TF32 MMA per 8-sample k-step, and the two cross terms lo*hi + hi*lo as bf16
MMAs per 16-sample k-step, with the k index of a bf16 step permuted so that its A fragments come from the registers of
the TF32 ones.  hi = trunc_tf32(x), and the bf16 copies are rne_bf16(hi) and rne_bf16(x - hi).

The kernel is checked against a float64 emulation of exactly those operand roundings with float64 accumulation, on
data whose lo parts are large (the low 13 mantissa bits at 0.5 .. 1 of a TF32 ulp): there the cross terms carry about
1e-3 of each diagonal entry, so a permutation that differs between the A and B operands, a dropped cross term or the
bf16 hi / lo tiles used the wrong way round show up far above the fp32 accumulation error."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BLK = 128

# (view widths, n): ragged widths (1, 33, 127, 129, 300), diagonal and off-diagonal tiles, n a multiple of neither 32
# nor 16, and one split, a few splits and dozens of splits of the sample axis
SHAPES = [
    ([1], 45),
    ([33, 1], 3001),
    ([127, 129], 5000),
    ([300, 33], 20011),
    ([129, 127, 1], 70001),
]


def _large_lo(n, d, g):
    """float32 N(0, 1) values with the 13 bits below the TF32 mantissa set to 0x1000 .. 0x1FFF: lo = x - trunc_tf32(x)
    is 0.5 .. 1 TF32 ulp of x, with the sign of x."""
    x = torch.randn(n, d, generator=g, device="cuda")
    low = torch.randint(0x1000, 0x2000, (n, d), generator=g, device="cuda", dtype=torch.int32)
    return ((x.view(torch.int32) & ~0x1FFF) | low).view(torch.float32)


def _padded(views):
    cols = []
    for v in views:
        d = v.shape[1]
        cols.append(torch.nn.functional.pad(v, (0, -(-d // BLK) * BLK - d)))
    return torch.cat(cols, dim=1)


def _real_columns(views):
    idx, off = [], 0
    for v in views:
        d = v.shape[1]
        idx.extend(range(off, off + d))
        off += -(-d // BLK) * BLK
    return torch.tensor(idx, device="cuda")


def _upper_blocks(Dp):
    blk = torch.arange(Dp // BLK, device="cuda").repeat_interleave(BLK)
    return blk[:, None] <= blk[None, :]


def _hi(X):
    return (X.view(torch.int32) & ~0x1FFF).view(torch.float32)   # trunc_tf32


def _emulated_x3b(X):
    """float64 X^T X of the operands tf32x3b feeds the tensor cores: hi*hi + bf16(hi)*bf16(lo) + bf16(lo)*bf16(hi)."""
    hi = _hi(X)
    lo = X - hi   # exact in float32
    bhi, blo = hi.bfloat16().double(), lo.bfloat16().double()   # round to nearest even
    hi = hi.double()
    return hi.T @ hi + bhi.T @ blo + blo.T @ bhi


def _moments(views, precision):
    from cca_zoo_b200 import ops

    mom = ops.moments(views, precision=precision)
    Dp = sum(-(-v.shape[1] // BLK) * BLK for v in views)
    return mom[:Dp * Dp].view(Dp, Dp), mom[Dp * Dp:]


def _normalised(M, ref, views):
    """|M - ref| / sqrt(ref_ii ref_jj) over the real columns of the upper block triangle."""
    Dp = M.shape[0]
    err = (M - ref).abs()
    err[~_upper_blocks(Dp)] = 0.0
    c = _real_columns(views)
    d = torch.diagonal(ref)[c]
    return err[c][:, c] / torch.sqrt(d[:, None] * d[None, :])


@pytest.mark.parametrize("dims,n", SHAPES)
def test_x3b_matches_the_emulated_operand_rounding(dims, n):
    g = torch.Generator(device="cuda").manual_seed(n + 7 * len(dims))
    views = [_large_lo(n, d, g) for d in dims]
    M, s = _moments(views, "tf32x3b")
    X = _padded(views)
    E = _emulated_x3b(X)
    X64 = X.double()
    exact = X64.T @ X64
    err = _normalised(M, E, views)
    # the operand roundings of the emulation are those of the kernel: what is left is the fp32 accumulation (its
    # round-toward-zero drift over one 2048-sample run stays near 1e-5 of a diagonal entry)
    assert err.max().item() < 5e-5, f"tf32x3b differs from its emulation by {err.max().item():.2e}"
    # the cross terms are large on this data: dropping them, or pairing the wrong samples, moves the diagonal ~1e-3
    c = _real_columns(views)
    hi = _hi(X).double()
    cross = (torch.diagonal(E) - (hi * hi).sum(dim=0))[c] / torch.diagonal(exact)[c]
    assert cross.min().item() > 2e-4, "the test data must have large lo parts"
    assert _normalised(M, exact, views).max().item() < 5e-5
    ref_s = X64.sum(dim=0)
    assert ((s - ref_s).abs() / X64.abs().sum(dim=0).clamp_min(1e-30)).max().item() < 1e-5, "column sums differ"


def test_x3b_diagonal_is_unbiased():
    """hi * lo >= 0 under truncation, so a diagonal without its cross terms would sit about 2^-11 low on every entry."""
    g = torch.Generator(device="cuda").manual_seed(11)
    views = [torch.randn(40000, d, generator=g, device="cuda") for d in (300, 129)]
    M, _ = _moments(views, "tf32x3b")
    X = _padded(views).double()
    c = _real_columns(views)
    ref = (X * X).sum(dim=0)[c]
    rel = (torch.diagonal(M)[c] - ref) / ref
    # without the cross terms the mean would be about -7e-4 on this data
    assert abs(rel.mean().item()) < 5e-5, f"mean relative error of the diagonal {rel.mean().item():.2e}"
    assert rel.abs().max().item() < 1e-4


def test_x3b_and_x3_are_different_kernels_of_fp32_grade():
    g = torch.Generator(device="cuda").manual_seed(3)
    views = [torch.randn(9000, d, generator=g, device="cuda") + 0.5 for d in (129, 300)]
    Mb, sb = _moments(views, "tf32x3b")
    M3, s3 = _moments(views, "tf32x3")
    assert not torch.equal(Mb, M3), "tf32x3b must run its own kernel, not the 3xTF32 one"
    X = _padded(views).double()
    exact = X.T @ X
    for M in (Mb, M3):
        assert _normalised(M, exact, views).max().item() < 5e-5
    ref_s = X.sum(dim=0)
    for s in (sb, s3):
        assert ((s - ref_s).abs() / X.abs().sum(dim=0).clamp_min(1e-30)).max().item() < 1e-5
