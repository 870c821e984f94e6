"""The bfloat16 / float16 moment routes of ``ops.moments``: the 16-bit wgmma pair-tile kernel (every tensor precision)
and the SIMT kernel instantiated for 16-bit views ("exact").

The product of two bf16 or two fp16 values is exact in fp32, so on views of small integers every fp32 accumulator run
is exact whatever its order or rounding: each |x_i x_j| <= 225 and a run spans at most 2048 samples, so every run sum
stays below 2048 * 225 < 2^24.  There the moment buffer must equal the float64 moments bit for bit, at every tile edge
the kernel has (rows around a 16-sample k step, a 32-sample slice, a 2048-sample run and a pass; widths around a 64-
column box and a 128-column block; odd pair-tile counts and diagonal tiles) and for strided and unaligned views."""
import ctypes as C

import pytest
import torch

from cca_zoo_b200 import _lib, ops

pytestmark = pytest.mark.gpu

BLK = 128
HALF = [torch.bfloat16, torch.float16]
PRECISIONS = ["tf32", "tf32x3", "tf32x3b", "exact"]
# rows one pass of the 16-bit kernel takes for a padded width of at most 2896: 256 splits of 2048-sample runs
PASS_ROWS = 256 * 2048


def _ints(n, d, dtype, g):
    return torch.randint(-15, 16, (n, d), generator=g, device="cuda").to(dtype)


def _padded(views):
    return torch.cat([torch.nn.functional.pad(v.double(), (0, -(-v.shape[1] // BLK) * BLK - v.shape[1]))
                      for v in views], dim=1)


def _split(mom, Dp):
    return mom[:Dp * Dp].reshape(Dp, Dp), mom[Dp * Dp:]


def _assert_bit_exact(views, precision):
    X = _padded(views)
    Dp = X.shape[1]
    M, s = _split(ops.moments(views, precision=precision), Dp)
    ref = X.T @ X
    upper = torch.ones(Dp, Dp, dtype=torch.bool, device="cuda").triu()
    assert torch.equal(M[upper], ref[upper]), \
        f"{precision}: max |diff| {(M - ref)[upper].abs().max().item()} over the upper triangle"
    assert torch.equal(s, X.sum(dim=0)), f"{precision}: column sums differ"


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n", [1, 15, 16, 17, 63, 64, 65, 2047, 2048, 2049, 4097])
def test_integer_views_bit_exact_by_rows(dtype, precision, n):
    g = torch.Generator(device="cuda").manual_seed(n)
    _assert_bit_exact([_ints(n, 65, dtype, g), _ints(n, 129, dtype, g)], precision)


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("d", [1, 7, 8, 9, 63, 64, 65, 127, 128, 129, 257])
def test_integer_views_bit_exact_by_width(dtype, precision, d):
    g = torch.Generator(device="cuda").manual_seed(d)
    _assert_bit_exact([_ints(3001, d, dtype, g)], precision)


# (view widths): 1, 2, 3 and 8 views; 1, 2, 3 and 5 padded blocks (odd pair-tile counts, a lone last block) and 8
VIEW_SETS = [[100], [129], [257], [129, 257], [128, 1, 129], [1, 7, 8, 9, 63, 64, 65, 127]]


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dims", VIEW_SETS)
def test_integer_views_bit_exact_by_views_and_blocks(dtype, precision, dims):
    g = torch.Generator(device="cuda").manual_seed(len(dims) * 1000 + sum(dims))
    _assert_bit_exact([_ints(5003, d, dtype, g) for d in dims], precision)


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", ["tf32x3b", "exact"])
def test_integer_views_bit_exact_past_one_pass(dtype, precision):
    g = torch.Generator(device="cuda").manual_seed(11)
    n = PASS_ROWS + 4097
    _assert_bit_exact([_ints(n, 100, dtype, g), _ints(n, 30, dtype, g)], precision)


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_strided_and_unaligned_views(dtype, precision):
    g = torch.Generator(device="cuda").manual_seed(5)
    wide = _ints(4099, 48, dtype, g)
    strided = wide[:, 8:25]                    # 16-byte aligned, row pitch 48 elements: read in place
    unaligned = wide[:, 3:20]                  # base 6 bytes past the allocation: ops._row_major copies it
    assert strided.data_ptr() % 16 == 0 and unaligned.data_ptr() % 16 != 0
    _assert_bit_exact([strided, unaligned], precision)


@pytest.mark.parametrize("dtype", HALF)
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dims,n", [([300, 33], 20011), ([129, 127, 1], 70001)])
def test_random_views_within_the_run_bound(dtype, precision, dims, n):
    """Bound: the products are exact, and a 2048-sample fp32 run takes at most 256 accumulator updates of the tensor
    core (one per 8-sample half of a k16 step, a conservative count), each truncating by at most 2^-23 of the running
    sum, whose magnitude is at most sum |x_i x_j| <= sqrt(M_ii M_jj).  The float64 sum of the runs adds nothing at
    this scale.  So |M - M_64| / sqrt(M_ii M_jj) <= 256 * 2^-23 = 3.05e-5, tighter than the 5e-5 of the tf32x3b tests.
    The SIMT route's 2048 round-to-nearest FMAs per run have unbiased errors of 2^-24, far inside it on this data."""
    g = torch.Generator(device="cuda").manual_seed(n)
    views = [torch.randn(n, d, generator=g, device="cuda").to(dtype) for d in dims]
    X = _padded(views)
    Dp = X.shape[1]
    M, s = _split(ops.moments(views, precision=precision), Dp)
    ref = X.T @ X
    real, off = [], 0
    for d in dims:
        real.extend(range(off, off + d))
        off += -(-d // BLK) * BLK
    real = torch.tensor(real, device="cuda")
    upper = torch.ones(Dp, Dp, dtype=torch.bool, device="cuda").triu()
    err = ((M - ref).abs() * upper)[real][:, real]
    dg = torch.diagonal(ref)[real]
    bound = 256 * 2.0 ** -23
    assert (err / torch.sqrt(dg[:, None] * dg[None, :])).max().item() <= bound
    # column sums: fp32 sums of at most 2048 exactly representable values per run, the same bound against sum |x|
    assert ((s - X.sum(dim=0)).abs()[real] <= bound * X.abs().sum(dim=0)[real] + 1e-30).all()


@pytest.mark.parametrize("dtype,code", [(torch.bfloat16, _lib.BF16), (torch.float16, _lib.F16)])
def test_pitch_not_a_multiple_of_8_is_an_argument_error(dtype, code):
    """The TMA route needs a 16-byte row pitch: 8 elements of a 16-bit view.  A pitch of 12 (a multiple of 4, which
    float32 would accept) is refused with the argument error before anything is launched."""
    lib = _lib.load()
    n, d, ld = 256, 10, 12
    buf = torch.zeros(n, ld, dtype=dtype, device="cuda")
    dims, lds = _lib.i64_array([d]), _lib.i64_array([ld])
    ptrs = (C.c_void_p * 1)(buf.data_ptr())
    out = torch.empty(lib.ccab_moments_size(1, dims), dtype=torch.float64, device="cuda")
    wsb = lib.ccab_moments_workspace_bytes(code, _lib.PREC_TF32X3B, 1, dims, n)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = lib.ccab_launch_count()
    rc = lib.ccab_moments(code, _lib.PREC_TF32X3B, 1, ptrs, dims, lds, n, C.c_void_p(out.data_ptr()),
                          C.c_void_p(ws.data_ptr()), wsb, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == -1
    assert "lds % 8" in _lib.last_error()
    assert lib.ccab_launch_count() == before


def test_other_entry_points_reject_16_bit_codes():
    lib = _lib.load()
    dims = _lib.i64_array([4, 4])
    x0 = (C.c_void_p * 2)(0, 0)
    mom = torch.zeros(lib.ccab_moments_size(2, dims), dtype=torch.float64, device="cuda")
    for code in (_lib.BF16, _lib.F16):
        rc = lib.ccab_moments_unshift(code, 2, dims, C.c_void_p(mom.data_ptr()), x0, 10.0, None)
        assert rc == -1 and "bad dtype" in _lib.last_error()
