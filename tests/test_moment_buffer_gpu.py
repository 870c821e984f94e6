"""The moment buffer ``[M (Dp x Dp) | s (Dp)]`` of ccab_moments, bit for bit, from every kernel that writes or
transforms it: the exact kernels (float64 DMMA, float32 SIMT), their split reduction, the shifted accumulation (pilot,
shift, unshift), the exchange message (pack / unpack) and the covariance kernel, plus what the consumers of the buffer
read.

Inputs are small integers (``randint(-8, 9)``, plus integer offsets where a test needs them), so every product is exact
in float64, and exact in TF32 with every fp32 partial sum exact while a run stays below 2^24.  The reference is a plain
float64 X^T X of the padded views on the device, exact in any summation order, so most assertions are ``torch.equal``.

The layout the reference helpers spell out (include/ccab200.h, ccab_moments): each view is padded to a multiple of 128
columns; M[r, c] with r <= c holds the moment of padded columns r and c, M is zero below the 128-block diagonal, and
the strictly lower part of a diagonal 128-block is unspecified (no consumer reads it; test E holds them to that).
"""
import numpy as np
import pytest
import torch

from oracle import restatement as R

pytestmark = pytest.mark.gpu

BLK = 128
f32, f64 = torch.float32, torch.float64


# --------------------------------------------------------------------------------------------------
# reference layout
# --------------------------------------------------------------------------------------------------
def padded(views):
    """The views side by side in float64, each padded with zero columns to a multiple of 128."""
    cols = []
    for v in views:
        d = v.shape[1]
        cols.append(torch.nn.functional.pad(v.double(), (0, -(-d // BLK) * BLK - d)))
    return torch.cat(cols, dim=1)


def reference(views):
    """(M, s): M = X_p^T X_p (full, symmetric) and s = 1^T X_p of the padded views X_p."""
    X = padded(views)
    return X.T @ X, X.sum(dim=0)


def split(mom, Dp):
    """(M as a Dp x Dp view, s) of a moment buffer."""
    assert mom.numel() == Dp * Dp + Dp
    return mom[:Dp * Dp].view(Dp, Dp), mom[Dp * Dp:]


def masks(Dp, device="cuda"):
    """(r <= c, below the 128-block diagonal, strictly lower part of a diagonal 128-block)."""
    r = torch.arange(Dp, device=device)[:, None]
    c = torch.arange(Dp, device=device)[None, :]
    return r <= c, r // BLK > c // BLK, (r > c) & (r // BLK == c // BLK)


def packed_reference(mom, Dp, n_local):
    """The exchange message: the upper 128-blocks row-major over bi <= bj (each block row-major), s, n_local, 0."""
    M, s = split(mom, Dp)
    nb = Dp // BLK
    blocks = [M[bi * BLK:(bi + 1) * BLK, bj * BLK:(bj + 1) * BLK].reshape(-1)
              for bi in range(nb) for bj in range(bi, nb)]
    return torch.cat(blocks + [s, torch.tensor([float(n_local), 0.0], dtype=f64, device=mom.device)])


def check_buffer(mom, views, what=""):
    """The buffer's contract against the reference: exact for r <= c, zero below the block diagonal, exact s."""
    M_ref, s_ref = reference(views)
    Dp = M_ref.shape[0]
    assert mom.numel() == Dp * Dp + Dp, what
    M, s = split(mom, Dp)
    up, below, _ = masks(Dp)
    bad = ((M != M_ref) & up).nonzero()
    assert bad.numel() == 0, (f"{what}: {bad.shape[0]} moment entries with r <= c differ, first at {bad[0].tolist()}: "
                              f"{M[tuple(bad[0])].item()} vs {M_ref[tuple(bad[0])].item()}")
    assert not M[below].any(), f"{what}: nonzero entries below the block diagonal"
    assert torch.equal(s, s_ref), f"{what}: column sums differ at {(s != s_ref).nonzero()[:4].flatten().tolist()}"


def int_views(dims, n, dtype, seed, offsets=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    views = [torch.randint(-8, 9, (n, d), generator=g, device="cuda").to(dtype) for d in dims]
    if offsets is not None:
        views = [v + o.to(dtype) for v, o in zip(views, offsets)]
    return views


def int_offsets(dims, seed, lo=900, hi=1100):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randint(lo, hi, (d,), generator=g, device="cuda").double() for d in dims]


# --------------------------------------------------------------------------------------------------
# A. exact kernels: float64 DMMA and float32 SIMT ("exact")
# --------------------------------------------------------------------------------------------------
# (widths, n) and the split plan of plan_simt on an H100 (132 SMs) each one reaches
EXACT_SHAPES = [
    ([1], 1),                                          # a single row
    ([64], 15),                                        # less than one 16-row chunk; the second 64-half is empty
    ([63, 65, 1], 17),                                 # one full chunk plus one row
    ([127, 128, 129], 777),                            # S = 7, short last split
    ([1], 70001),                                      # S capped at 64, short last split
    ([300, 33, 64, 1, 65, 127, 128, 2], 4099),         # 8 views (the limit), Dp = 1280: S = 1
    ([512, 512], 3001),                                # S = 1, past one 2048-row accumulator run
]


@pytest.mark.parametrize("dtype", [f64, f32], ids=["dmma-f64", "simt-f32"])
@pytest.mark.parametrize("dims,n", EXACT_SHAPES, ids=[f"{'-'.join(map(str, d))}-n{n}" for d, n in EXACT_SHAPES])
def test_exact_kernels_are_exact_on_integers(dtype, dims, n):
    from cca_zoo_b200 import ops

    views = int_views(dims, n, dtype, seed=n + 31 * len(dims))
    check_buffer(ops.moments(views, precision="exact"), views, f"{dims} n={n} {dtype}")


@pytest.mark.parametrize("dtype", [f64, f32])
def test_exact_kernels_read_column_slices_in_place(dtype):
    """A view that is a column slice of a wider tensor: ld > d and a base pointer off the 16-byte grid."""
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(4)
    wide = torch.randint(-8, 9, (1001, 203), generator=g, device="cuda").to(dtype)
    views = [wide[:, 3:140], wide[:, 141:142], wide[:, 150:201]]
    assert views[0].data_ptr() % 16 != 0 and views[0].stride(0) == 203
    check_buffer(ops.moments(views, precision="exact"), views, f"column slices {dtype}")


@pytest.mark.parametrize("dtype", [f64, f32])
def test_exact_kernels_are_deterministic(dtype):
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(9)
    views = [torch.randn(5000, d, generator=g, device="cuda", dtype=dtype) for d in (200, 70)]
    assert torch.equal(ops.moments(views, precision="exact"), ops.moments(views, precision="exact"))


def test_layouts_the_kernels_cannot_hold_are_refused_with_a_message():
    from cca_zoo_b200 import _lib, ops

    nine = [torch.zeros(4, 2, device="cuda") for _ in range(9)]
    with pytest.raises(ValueError, match="between 1 and 8 views"):
        ops.moments(nine, precision="exact")
    lib = _lib.load()
    assert lib.ccab_moments_size(9, _lib.i64_array([2] * 9)) < 0 and "n_views" in _lib.last_error()
    wide = [torch.zeros(2, 8192, device="cuda"), torch.zeros(2, 8193, device="cuda")]     # Dp = 8192 + 8320
    with pytest.raises(ValueError, match="padded width 16512 exceeds 16384"):
        ops.moments(wide, precision="exact")


# --------------------------------------------------------------------------------------------------
# B. shifted accumulation, exactly
# --------------------------------------------------------------------------------------------------
SHIFT_CASES = [("tf32", f32), ("tf32x3", f32), ("tf32x3b", f32), ("exact", f32), ("exact", f64)]


@pytest.mark.parametrize("precision,dtype", SHIFT_CASES, ids=[f"{p}-{str(d)[6:]}" for p, d in SHIFT_CASES])
def test_shifted_accumulation_rebuilds_the_raw_moments_exactly(precision, dtype):
    """Integer views with integer column offsets of about 1000 and an integer x0: the shifted values are small integers,
    the unshift adds integers below 2^53, so the rebuilt buffer is the raw X^T X exactly."""
    from cca_zoo_b200 import ops

    dims, n = [129, 300, 5], 5000                     # Dp-crossing widths, n past one 2048-sample run
    off = int_offsets(dims, seed=1)
    views = int_views(dims, n, dtype, seed=2, offsets=off)
    x0 = [(o + 1).to(dtype) for o in off]             # not the mean: the shifted columns keep a nonzero mean
    mom, used = ops.moments_safe(views, precision=precision, x0=x0)
    assert used is x0
    check_buffer(mom, views, f"shifted {precision} {dtype}")


@pytest.mark.parametrize("dtype", [f64, f32])
def test_unshift_leaves_unshifted_views_untouched(dtype):
    """x0 = None for a view: its block and column sums are not touched; the cross blocks are still exact."""
    from cca_zoo_b200 import ops

    dims, n = [130, 64, 200], 3000
    off = int_offsets(dims, seed=3)
    views = int_views(dims, n, dtype, seed=4, offsets=[off[0] * 0, off[1], off[2] * 0])
    x0 = [None, off[1].to(dtype), None]
    shifted = [views[0], ops.shift_rows(views[1], x0[1]), views[2]]
    mom = ops.moments(shifted, precision="exact")
    before = mom.clone()
    ops.moments_unshift_(mom, dims, x0, n)
    check_buffer(mom, views, f"partial unshift {dtype}")
    Dp = 256 + 128 + 256
    M, s = split(mom, Dp)
    Mb, sb = split(before, Dp)
    for lo, hi in ((0, 256), (384, 640)):              # the unshifted views' diagonal blocks, lower parts included
        assert torch.equal(M[lo:hi, lo:hi], Mb[lo:hi, lo:hi]) and torch.equal(s[lo:hi], sb[lo:hi])
    assert torch.equal(M[0:256, 384:640], Mb[0:256, 384:640])     # and the block between them


@pytest.mark.parametrize("precision,dtype", [("tf32x3b", f32), ("exact", f32), ("exact", f64)])
def test_shards_shifted_by_different_x0_sum_to_the_raw_moments(precision, dtype):
    """The multi-GPU contract on one GPU: whatever x0 each shard chose, the rebuilt buffers add up to the raw moments
    of the whole input, exactly."""
    from cca_zoo_b200 import ops

    dims, n, cut = [129, 40], 4500, 2600
    off = int_offsets(dims, seed=5)
    views = int_views(dims, n, dtype, seed=6, offsets=off)
    xa = [(o - 3).to(dtype) for o in off]
    xb = [(o + 5).to(dtype) for o in off]
    a, _ = ops.moments_safe([v[:cut] for v in views], precision=precision, x0=xa)
    b, _ = ops.moments_safe([v[cut:] for v in views], precision=precision, x0=xb)
    check_buffer(a + b, views, f"two shards {precision} {dtype}")


# --------------------------------------------------------------------------------------------------
# C. pilot and shift kernels against float64
# --------------------------------------------------------------------------------------------------
def pilot_reference(X):
    """(x0, ratio) over the leading min(n, 4096) rows: mean, mean^2 / population variance (1e30 for a constant nonzero
    column, 0 for an all-zero one, capped at 1e30).  Summed in extended precision, so that the reference mean itself
    is far inside one float64 ulp."""
    A = X[:4096].astype(np.longdouble)
    mean = A.mean(axis=0)
    var = ((A - mean) ** 2).mean(axis=0)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(var > 0, mean * mean / np.where(var > 0, var, 1.0), np.where(mean != 0, 1e30, 0.0))
    return mean, float(np.minimum(r, 1e30).max())


def within_one_ulp(x0, mean, dtype):
    return bool((np.abs(x0.astype(np.longdouble) - mean) <= np.spacing(np.abs(mean).astype(dtype))).all())


def pilot_views(n, d, dtype, seed):
    """Columns with means of either sign between 20 and 1000 std (so that one ulp of x0 is far above the float64
    rounding of the mean); rows 4096+ wildly different, so that a kernel reading past the pilot rows fails."""
    rng = np.random.default_rng(seed)
    mu = rng.uniform(20.0, 1000.0, d) * rng.choice([-1.0, 1.0], d)
    X = rng.standard_normal((n, d)) * rng.uniform(0.5, 2.0, d) + mu
    X[4096:] = X[4096:] * 50.0 - 7e4
    return X.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("d", [1, 33, 300])
@pytest.mark.parametrize("n", [1, 31, 4096, 9000])
def test_column_pilot_matches_float64(n, d, dtype):
    from cca_zoo_b200 import ops

    X = pilot_views(n, d, dtype, seed=n + d)
    (x0,), ratio = ops.column_pilot([torch.from_numpy(X).cuda()])
    mean, r_ref = pilot_reference(X)
    x0 = x0.cpu().numpy()
    assert x0.dtype == dtype
    assert within_one_ulp(x0, mean, dtype), float(np.abs(x0 - mean).max())
    assert abs(ratio - r_ref) <= 1e-6 * r_ref, (ratio, r_ref)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_column_pilot_strided_constant_zero_columns_and_the_maximum_over_views(dtype):
    from cca_zoo_b200 import ops

    X = pilot_views(5000, 40, dtype, seed=3)
    wide = torch.from_numpy(X).cuda()
    sl = wide[:, 5:38]                                  # ld = 40 > d = 33, base off the 16-byte grid
    (x0,), ratio = ops.column_pilot([sl])
    mean, r_ref = pilot_reference(X[:, 5:38])
    assert within_one_ulp(x0.cpu().numpy(), mean, dtype)
    assert abs(ratio - r_ref) <= 1e-6 * r_ref
    const = torch.full((100, 3), 2.5, dtype=wide.dtype, device="cuda")
    (c0,), rc = ops.column_pilot([const])
    assert rc == float(np.float32(1e30)) and bool((c0 == 2.5).all())          # the shift is taken
    (z0,), rz = ops.column_pilot([torch.zeros_like(const)])
    assert rz == 0.0 and not z0.any()
    # the ratio is the maximum over every column of every view
    rng = np.random.default_rng(7)
    mild = [(rng.standard_normal((3000, d)) + m).astype(dtype) for d, m in ((20, 0.5), (7, 3.0), (50, 1.5))]
    _, r_all = ops.column_pilot([torch.from_numpy(v).cuda() for v in mild])
    r_ref = max(pilot_reference(v)[1] for v in mild)
    assert abs(r_all - r_ref) <= 1e-6 * r_ref


@pytest.mark.parametrize("dtype,limit", [(f32, 16.0), (f64, 1e8)])
def test_shift_decision_at_the_ratio_threshold(dtype, limit):
    """moments_safe shifts exactly when the pilot's mean^2 / var exceeds SHIFT_RATIO: a column alternating mu +- 1 has
    mean mu and variance 1, so mu = sqrt(limit) (1 +- 1%) lands on either side."""
    from cca_zoo_b200 import ops

    assert ops.SHIFT_RATIO[dtype] == limit
    for factor, shifts in ((1.01, True), (0.99, False)):
        mu = np.sqrt(limit) * factor
        col = torch.tensor([mu + 1.0, mu - 1.0], dtype=f64).repeat(3000)[:, None].to(dtype).cuda()
        other = torch.randn(6000, 5, dtype=dtype, device="cuda")
        _, x0 = ops.moments_safe([other, col], precision="tf32x3b")
        assert (x0 is not None) == shifts, (dtype, factor)


@pytest.mark.parametrize("dtype", [f32, f64])
def test_shift_rows_is_bitwise_the_subtraction(dtype):
    from cca_zoo_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    wide = torch.randn(777, 70, generator=g, device="cuda", dtype=dtype) * 300 + 1000
    for v in (wide[:, 3:36], wide[:, :1], wide.T[:33, :50], wide):      # strided, one column, transposed, contiguous
        x0 = torch.randn(v.shape[1], generator=g, device="cuda", dtype=dtype) * 300 + 1000
        out = ops.shift_rows(v, x0)
        assert out.shape == v.shape and out.stride(1) == 1
        assert (out.stride(0) * out.element_size()) % 16 == 0 and out.data_ptr() % 16 == 0
        assert torch.equal(out, v - x0)


# --------------------------------------------------------------------------------------------------
# D. exchange message
# --------------------------------------------------------------------------------------------------
def _buffers(dims, n, seed):
    """Moment buffers of three producers: K1 (tf32x3b), the DMMA kernel, and a shifted float32 pass after the unshift."""
    from cca_zoo_b200 import ops

    views = int_views(dims, n, f32, seed=seed)
    k1 = ops.moments(views, precision="tf32x3b")
    dmma = ops.moments([v.double() for v in views], precision="exact")
    off = int_offsets(dims, seed=seed + 1)
    shifted, _ = ops.moments_safe([v + o.float() for v, o in zip(views, off)], precision="exact",
                                  x0=[o.float() for o in off])
    return {"k1": k1, "dmma": dmma, "unshifted": shifted}


PACK_DIMS = [[300, 129], [300, 33, 64, 1, 65, 127, 128, 2]]


@pytest.mark.parametrize("dims", PACK_DIMS, ids=["2views", "8views"])
def test_pack_follows_the_header_layout_and_unpack_inverts_the_sum(dims):
    from cca_zoo_b200 import _lib, ops

    Dp = int(_lib.load().ccab_moments_padded_dim(len(dims), _lib.i64_array(dims)))
    a = _buffers(dims, 1500, seed=20)
    b = _buffers(dims, 700, seed=40)
    for name in a:
        pa = ops.moments_pack(a[name], dims, 1500)
        assert torch.equal(pa, packed_reference(a[name], Dp, 1500)), name
        pb = ops.moments_pack(b[name], dims, 700)
        mom, n_dev = ops.moments_unpack(pa + pb, dims)
        assert torch.equal(mom, a[name] + b[name]), name          # the all-reduce, run as a plain sum
        assert n_dev.item() == 2200.0 and (pa + pb)[-1].item() == 0.0, name


# --------------------------------------------------------------------------------------------------
# E. what the consumers read: entries with r > c never are
# --------------------------------------------------------------------------------------------------
def poisoned(mom, Dp):
    """A copy with NaN in the strictly lower part of every diagonal 128-block."""
    out = mom.clone()
    M, _ = split(out, Dp)
    M[masks(Dp)[2]] = float("nan")
    return out


@pytest.mark.parametrize("dtype", [f64, f32])
def test_covariance_never_reads_the_lower_part_of_a_diagonal_block(dtype):
    from cca_zoo_b200 import ops

    dims, n = [300, 129, 1], 2000
    views = int_views(dims, n, f64, seed=50)
    clean = ops.moments(views, precision="exact")
    bad = poisoned(clean, 384 + 256 + 128)
    for center in (True, False):
        Cc, mc = ops.covariance(clean, dims, n, center=center, dtype=dtype)
        Cb, mb = ops.covariance(bad, dims, n, center=center, dtype=dtype)
        assert torch.isfinite(Cc).all() and torch.equal(Cb, Cc) and torch.equal(mb, mc), center
    # through the exchange message: pack -> unpack keeps the diagonal blocks whole, NaN included
    mom, _ = ops.moments_unpack(ops.moments_pack(bad, dims, n), dims)
    assert torch.equal(ops.covariance(mom, dims, n, dtype=dtype)[0], ops.covariance(clean, dims, n, dtype=dtype)[0])


def _fit_outputs(block, offsets, dims, k, dtype):
    from cca_zoo_b200 import ops

    hdr, mean, sig, ws = ops.decode_fit_block(block.cpu(), offsets, dims, k, dtype)
    return [hdr[:6].copy(), mean.copy(), sig.copy()] + [w.copy() for w in ws]


@pytest.mark.parametrize("dtype", [f64, f32])
def test_rcca_fit_never_reads_the_lower_part_of_a_diagonal_block(dtype):
    """The ridge-perview case of test_fit_routes_gpu.py (300 x 260, k = 8, p = 24, 6 iterations)."""
    from cca_zoo_b200 import ops
    from tests.test_fit_routes_gpu import rcca_problem

    dims, k, p = [300, 260], 8, 24
    views, _, _ = rcca_problem(*dims, k, p, seed=dims[0] + 7 * dims[1] + k)
    n = views[0].shape[0]
    clean = ops.moments([torch.from_numpy(v).cuda() for v in views], "exact")
    bad = poisoned(clean, 384 + 384)
    outs = [_fit_outputs(*ops.rcca_fit(m, dims, n, None, True, [0.0, 0.0], k, p, 6, dtype), dims, k, dtype)
            for m in (clean, bad)]
    assert int(outs[1][0][0]) == 0, f"status {int(outs[1][0][0])}"
    assert all(np.array_equal(x, y) for x, y in zip(*outs))


def test_mcca_fit_never_reads_the_lower_part_of_a_diagonal_block():
    """The 3views-w1-w65 case of test_fit_routes_gpu.py (widths 65, 1, 100, k = 4, p = 36, 32 iterations)."""
    from cca_zoo_b200 import ops
    from tests.test_fit_routes_gpu import mcca_problem

    dims, k, p, c = [65, 1, 100], 4, 36, [0.0, 0.0, 0.1]
    views = mcca_problem(dims, k, seed=len(dims) * 13 + k)
    n = views[0].shape[0]
    clean = ops.moments([torch.from_numpy(v).cuda() for v in views], "exact")
    bad = poisoned(clean, 3 * 128)
    outs = [_fit_outputs(*ops.mcca_fit(m, dims, n, None, True, c, 1e-6, k, p, 32, f64), dims, k, f64)
            for m in (clean, bad)]
    assert int(outs[1][0][0]) == 0, f"status {int(outs[1][0][0])}"
    assert all(np.array_equal(x, y) for x, y in zip(*outs))


# --------------------------------------------------------------------------------------------------
# F. covariance kernel
# --------------------------------------------------------------------------------------------------
def test_covariance_is_the_float64_formula_bit_for_bit():
    """From exact integer moments: C = (M - s s^T / n) / (n - 1) in float64 in the kernel's order (quotient subtracted,
    then divided: nothing to contract into an FMA), cast once for float32; exactly symmetric; mean = s / n."""
    from cca_zoo_b200 import ops

    dims, n = [127, 128, 129, 1], 999
    views = int_views(dims, n, f64, seed=60, offsets=int_offsets(dims, seed=61, lo=-3, hi=4))
    mom = ops.moments(views, precision="exact")
    X = torch.cat(views, dim=1)
    M, s = X.T @ X, X.sum(dim=0)
    # divisors as device tensors: torch turns division by a host scalar into a product with its reciprocal
    n_dev = torch.tensor(float(n), dtype=f64, device="cuda")
    for center in (True, False):
        ref = ((M - torch.outer(s, s) / n_dev) if center else M) / (n_dev - 1.0)
        ref_mean = s / n_dev if center else torch.zeros_like(s)
        for dtype in (f64, f32):
            Cm, mean = ops.covariance(mom, dims, n, center=center, dtype=dtype)
            assert torch.equal(Cm, ref.to(dtype)), (center, dtype, (Cm.double() - ref).abs().max().item())
            assert torch.equal(Cm, Cm.T) and torch.equal(mean, ref_mean.to(dtype)), (center, dtype)


# --------------------------------------------------------------------------------------------------
# G. consumers of the shifted accumulation
# --------------------------------------------------------------------------------------------------
def offset_views(dims, n, seed):
    """float32 views of a latent model with column means of about 1000 std."""
    from cca_zoo_b200.datasets import joint_data

    views = joint_data(n_views=len(dims), n_samples=n, n_features=dims, latent_dimensions=3, signal_to_noise=1.0,
                       random_state=seed)
    return [(v + 1000.0 * v.std(axis=0) * np.linspace(-1.0, 1.0, v.shape[1])).astype(np.float32) for v in views]


def correlations_f64(views, weights):
    """Pairwise correlations of the variates in float64 from the float32 inputs: centre, project, correlate."""
    Z = []
    for v, w in zip(views, weights):
        X = v.astype(np.float64)
        Z.append((X - X.mean(axis=0)) @ w.astype(np.float64))
    Z = np.stack(Z)
    Z = Z / np.linalg.norm(Z, axis=1, keepdims=True)
    return np.einsum("isd,jsd->ijd", Z, Z)


def test_device_score_of_badly_centred_views_matches_float64():
    from cca_zoo_b200.linear import MCCA, rCCA

    for est, dims in ((rCCA(latent_dimensions=3, c=0.1), [40, 30]), (MCCA(latent_dimensions=3, c=0.1), [40, 30, 20])):
        views = offset_views(dims, 6000, seed=len(dims))
        est.fit(views)
        ref = correlations_f64(views, est.weights_)
        dev = [torch.from_numpy(v).cuda() for v in views]
        got = est.pairwise_correlations(dev)
        err = float(np.abs(got - ref).max())
        print(f"{type(est).__name__}: device pairwise correlations off by {err:.2e}")
        assert err < 1e-4, f"{type(est).__name__}: pairwise correlations off by {err:.2e}"
        m = len(dims)
        ref_score = (ref.sum(axis=(0, 1)) - sum(ref[i, i] for i in range(m))) / (m * (m - 1))
        assert np.abs(est.score(dev) - ref_score).max() < 1e-4


def test_streamed_and_partial_fits_of_badly_centred_views_match_the_reference():
    """Each chooses its own x0: the streamed fit from its first chunk, partial_fit per batch."""
    from cca_zoo_b200.linear import rCCA

    views = offset_views([40, 30], 6000, seed=2)
    w_ref, _ = R.ref_rcca_fit([v.astype(np.float64) for v in views], 3, 0.1)
    st = rCCA(latent_dimensions=3, c=0.1)
    st._stream_threshold_bytes = 1 << 20
    st._stream_chunk_rows = 1000
    st.fit(views)
    assert st._stream_x0 is not None, "the streamed fit must take the shifted accumulation"
    inc = rCCA(latent_dimensions=3, c=0.1)
    for lo, hi, last in ((0, 2000, False), (2000, 2001, False), (2001, 6000, True)):
        inc.partial_fit([v[lo:hi] for v in views], solve=last)
    for name, est in (("streamed", st), ("partial_fit", inc)):
        err = R.max_rel_err_per_vector([w.astype(np.float64) for w in est.weights_], w_ref)
        assert err < 1e-3, f"{name}: weights off by {err:.2e}"


# --------------------------------------------------------------------------------------------------
# H. float32 "exact" over one long split
# --------------------------------------------------------------------------------------------------
def test_float32_exact_keeps_its_accuracy_over_one_long_split():
    """Dp = 1024 gives plan_simt one split: 2^20 rows go through one CTA per tile.  The fp32 accumulator run is bounded
    (folded into float64 every 2048 rows), so the covariance keeps the 2e-5 bar of short inputs."""
    from cca_zoo_b200 import ops

    n, dims = 1 << 20, [512, 512]
    g = torch.Generator(device="cuda").manual_seed(12)
    views = [torch.randn(n, d, generator=g, device="cuda") for d in dims]
    mom = ops.moments(views, precision="exact")
    Cm, _ = ops.covariance(mom, dims, n, center=True, dtype=f64)
    M = torch.zeros(1024, 1024, dtype=f64, device="cuda")
    s = torch.zeros(1024, dtype=f64, device="cuda")
    for r0 in range(0, n, 1 << 16):                  # float64 reference over row chunks: no 8 GB copy
        X = torch.cat([v[r0:r0 + (1 << 16)] for v in views], dim=1).double()
        M += X.T @ X
        s += X.sum(dim=0)
        del X
    ref = (M - torch.outer(s, s) / n) / (n - 1)
    scale = torch.sqrt(torch.outer(ref.diagonal(), ref.diagonal()))
    err = float(((Cm - ref).abs() / scale).max())
    print(f"float32 exact, n = 2^20, one split: max normalised covariance error {err:.2e}")
    assert err < 2e-5, f"max normalised covariance error {err:.2e}"
