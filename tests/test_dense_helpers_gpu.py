"""The dense helpers of csrc/dense.cu that every estimator and deep loss calls: ``ops.scale``, ``ops.whiten_rows``,
``ops.center_columns_`` and ``ops.frobenius_norm``, each against a CPU reference in float64 (long double for float64
kernels).

Bitwise checks are made only where the kernel's arithmetic has a single admissible result:

* ``scale`` multiplies and never adds, so no product can be contracted into an FMA and the emulation
  ``A * ((1 * pow(r)) * pow(c))`` in the tensor's dtype (IEEE ``1/x`` and ``1/sqrt(x)``) is exact;
* ``center_columns_`` on integer data: every column sum is exact in double in any order, so the mean and the
  subtraction are single roundings;
* ``frobenius_norm`` of ``2^k A`` in float64: the kernel scales by a power of two chosen from max |a|, so the sum it
  forms does not depend on k.

Everything else is held to a bound derived in the test's docstring, and the observed ratio is printed.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = {torch.float32: 2.0 ** -24, torch.float64: 2.0 ** -53}     # unit roundoff
NP = {torch.float32: np.float32, torch.float64: np.float64}
DTYPES = [torch.float32, torch.float64]


def _launches():
    from cca_zoo_b200 import _lib

    torch.cuda.synchronize()
    return int(_lib.load().ccab_launch_count())


def _view(parent, lo, n):
    return parent[:, lo:lo + n]


def _outside_unchanged(parent, before, lo, hi):
    return torch.equal(parent[:, :lo], before[:, :lo]) and torch.equal(parent[:, hi:], before[:, hi:])


# --------------------------------------------------------------------------------------------------
# ops.scale
# --------------------------------------------------------------------------------------------------
def _pow(v, p):
    if p == 1:
        return v
    one = v.dtype.type(1)
    return one / v if p == -1 else one / np.sqrt(v)


def _scale_emulation(A, r, rp, c, cp):
    """out = A * ((1 * pow(r)) * pow(c)) in A's dtype, rounding after every operation as the kernel does."""
    t = A.dtype.type
    f = np.ones(A.shape, dtype=A.dtype)
    if r is not None:
        f = f * _pow(r, rp)[:, None]
    if c is not None:
        f = f * _pow(c, cp)[None, :]
    out = A * f
    assert out.dtype == t
    return out


def _positive(g, size, dtype):
    """Positive factors spread over about 2^+-8, so 1/x and 1/sqrt(x) round in every way."""
    return torch.exp(3.0 * torch.randn(size, generator=g, dtype=torch.float64)).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("which", ["rows", "cols", "both"])
@pytest.mark.parametrize("rp,cp", [(1, 1), (-1, -1), (-0.5, -0.5), (-1, -0.5), (-0.5, 1)])
def test_scale_matches_its_exact_emulation(dtype, which, rp, cp):
    """Power codes on rows, columns and both; A a strided view (lda = n + 5) and ``out`` another (ldb = n + 9); the
    columns around ``out`` stay untouched."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(100 * DTYPES.index(dtype) + 10 * ["rows", "cols", "both"].index(which)
                                      + int(4 * rp) + int(2 * cp))
    m, n = 203, 150
    A = torch.randn(m, n, generator=g, dtype=torch.float64).to(dtype)
    r = _positive(g, m, dtype) if which in ("rows", "both") else None
    c = _positive(g, n, dtype) if which in ("cols", "both") else None
    pa = torch.randn(m, n + 5, generator=g, dtype=torch.float64).to(dtype).cuda()
    pa[:, 2:2 + n] = A.cuda()
    pb = torch.randn(m, n + 9, generator=g, dtype=torch.float64).to(dtype).cuda()
    pb0 = pb.clone()
    out = _view(pb, 4, n)
    l0 = _launches()
    ops.scale(_view(pa, 2, n), rows=None if r is None else r.cuda(), rows_pow=rp,
              cols=None if c is None else c.cuda(), cols_pow=cp, out=out)
    assert _launches() - l0 == 1
    want = _scale_emulation(A.numpy(), None if r is None else r.numpy(), rp, None if c is None else c.numpy(), cp)
    assert np.array_equal(out.cpu().numpy(), want)
    assert _outside_unchanged(pb, pb0, 4, 4 + n), "scale wrote outside its output view"


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_in_place(dtype):
    """``out`` aliased to A, as the kernel methods scale their Gram matrices: each element is read before it is
    written by the same thread."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(11)
    A = torch.randn(300, 257, generator=g, dtype=torch.float64).to(dtype)
    r, c = _positive(g, 300, dtype), _positive(g, 257, dtype)
    Ad = A.cuda()
    ops.scale(Ad, rows=r.cuda(), rows_pow=-0.5, cols=c.cuda(), cols_pow=-0.5, out=Ad)
    assert np.array_equal(Ad.cpu().numpy(), _scale_emulation(A.numpy(), r.numpy(), -0.5, c.numpy(), -0.5))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,n", [(0, 7), (7, 0), (0, 0)])
def test_scale_empty(dtype, m, n):
    """An empty matrix launches nothing and is not an error, whether or not its tensors have storage."""
    from cca_zoo_b200 import ops

    A = torch.empty(m, n, dtype=dtype, device="cuda")
    r = torch.ones(m, dtype=dtype, device="cuda")
    l0 = _launches()
    out = ops.scale(A, rows=r, rows_pow=-1)
    assert tuple(out.shape) == (m, n) and _launches() == l0
    parent = torch.ones(4, 9, dtype=dtype, device="cuda")   # zero-size views of allocated storage
    ops.scale(parent[:m, :n], rows=r, rows_pow=-1, out=parent[2:2 + m, 1:1 + n])
    assert torch.equal(parent, torch.ones_like(parent))


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale_past_65535_rows(dtype):
    """70000 rows: more than gridDim.y can hold.  Every row, including the last, is scaled, in one launch."""
    from cca_zoo_b200 import ops

    g = torch.Generator().manual_seed(70000)
    m, n = 70000, 130
    A = torch.randn(m, n, generator=g, dtype=torch.float64).to(dtype)
    r, c = _positive(g, m, dtype), _positive(g, n, dtype)
    l0 = _launches()
    out = ops.scale(A.cuda(), rows=r.cuda(), rows_pow=-1, cols=c.cuda(), cols_pow=-0.5)
    assert _launches() - l0 == 1
    assert np.array_equal(out.cpu().numpy(), _scale_emulation(A.numpy(), r.numpy(), -1, c.numpy(), -0.5))


# --------------------------------------------------------------------------------------------------
# ops.whiten_rows
# --------------------------------------------------------------------------------------------------
def _g_ref(lam, c, fl, scale, rank_tol, max_rank, lam_floor):
    """g_j = 1 / sqrt(((1 - c) max(lam_j, lam_floor) + c + fl) scale) for the kept rows, in float64; kept means
    lam_j > rank_tol * max(lam_0, 0) (strictly) and j < max_rank."""
    lam = lam.astype(np.float64)
    l0 = max(lam[0], 0.0)
    keep = (lam > rank_tol * l0) & (np.arange(lam.size) < max_rank)
    with np.errstate(divide="ignore", invalid="ignore"):
        g = 1.0 / np.sqrt(((1.0 - c) * np.maximum(lam, lam_floor) + c + fl) * scale)
    return np.where(keep, g, 0.0), keep


def _check_whiten(dtype, lam, c=0.1, floor_add=0.0, floor_dev=None, scale=1.0, rank_tol=0.0, max_rank=None,
                  lam_floor=-1e300, seed=0):
    """g is computed in double, where the compiler may contract ``(1 - c) * lam + c`` into an FMA, so it is held to
    the float64 formula within a bound, not bitwise.  With u = 2^-53 and every term of
    s = ((1 - c) max(lam, lam_floor) + c + floor) non-negative for the kept rows, the two evaluation orders differ by
    the dropped rounding of the product (<= u s) and by the two additions rounding different values (<= 2u s each
    way): 5u s; the product with ``scale`` adds 2u, sqrt halves the 7u and adds 2u, the reciprocal 2u more, so
    |g - g_ref| <= 7.5u g_ref, taken as 8u.  Wt = (T)(g * Vt) with g in double: exactly g_out * Vt in float64, one
    float32 rounding of g * Vt in float32."""
    from cca_zoo_b200 import ops

    g_ = torch.Generator().manual_seed(seed)
    d = lam.size
    Vt = torch.randn(d, d, generator=g_, dtype=torch.float64).to(dtype)
    lam_t = torch.from_numpy(lam.astype(NP[dtype]))
    fd = None if floor_dev is None else torch.tensor([floor_dev], dtype=dtype, device="cuda")
    Wt, g, rank = ops.whiten_rows(lam_t.cuda(), Vt.cuda(), c, floor_add=floor_add, floor_dev=fd, scale=scale,
                                  rank_tol=rank_tol, max_rank=max_rank, lam_floor=lam_floor)
    fl = floor_add + (0.0 if floor_dev is None else float(np.asarray(floor_dev, dtype=NP[dtype])))
    g_ref, keep = _g_ref(lam_t.numpy(), c, fl, scale, rank_tol, d if max_rank is None else max_rank, lam_floor)
    g_dev = g.cpu().numpy().astype(np.float64)
    assert int(rank.item()) == int(keep.sum())
    assert np.all(g_dev[~keep] == 0.0) and np.all(Wt.cpu().numpy()[~keep] == 0.0)
    if dtype == torch.float64:
        rel = np.abs(g_dev - g_ref)[keep] / g_ref[keep]
        print(f"whiten_rows float64: max |g - g_ref| / g_ref = {rel.max(initial=0) / U[dtype]:.2f} u (bound 8)")
        assert np.all(rel <= 8 * U[dtype])
        assert torch.equal(Wt.cpu(), g.cpu()[:, None] * Vt), "Wt must be g_out * Vt exactly in float64"
    else:
        rel = np.abs(g_dev - g_ref)[keep] / g_ref[keep]
        bound = U[dtype] + 8 * U[torch.float64]     # g_out = (float)g: one rounding of a value within 8u64 of g_ref
        print(f"whiten_rows float32: max |g - g_ref| / g_ref = {rel.max(initial=0) / bound:.3f} of the bound")
        assert np.all(rel <= bound)
        exact = g_ref[:, None] * Vt.double().numpy()
        err = np.abs(Wt.double().cpu().numpy() - exact)
        bound = (U[dtype] + 9 * U[torch.float64]) * np.abs(exact)
        print(f"whiten_rows float32: Wt error / bound = {float((err / np.where(bound > 0, bound, 1)).max()):.3f}")
        assert np.all(err <= bound)
    return keep


@pytest.mark.parametrize("dtype", DTYPES)
def test_whiten_rows_formula_and_rank_at_the_strict_threshold(dtype):
    """lam_3 equals rank_tol * lam_0 exactly (all powers of two times 3): the comparison is strict, so row 3 goes."""
    rank_tol = 2.0 ** -10
    lam = np.array([3.0, 1.5, 3.0 * 2.0 ** -9, 3.0 * 2.0 ** -10, 0.7, 3.0 * 2.0 ** -11, 2.0, -0.5, 1e-3 * 3, 5.0,
                    0.33, 0.0] + list(np.linspace(0.01, 2.0, 53)))
    keep = _check_whiten(dtype, lam, c=0.3, scale=0.125, rank_tol=rank_tol, seed=1)
    assert keep[2] and not keep[3] and not keep[5] and not keep[7] and not keep[11]


@pytest.mark.parametrize("dtype", DTYPES)
def test_whiten_rows_negative_leading_eigenvalue(dtype):
    """lam_0 < 0: the threshold is max(lam_0, 0) = 0, so exactly the positive rows are kept (row 0 is not)."""
    lam = np.array([-0.25, 1.0, 0.0, 2.0 ** -30, -1.0, 0.5] * 6)
    keep = _check_whiten(dtype, lam, c=0.0, rank_tol=0.5, lam_floor=0.0, seed=2)
    assert list(keep[:6]) == [False, True, False, True, False, True]


@pytest.mark.parametrize("dtype", DTYPES)
def test_whiten_rows_max_rank_floors(dtype):
    """max_rank below the kept count, the device floor added to the host floor, and lam_floor lifting the small
    eigenvalues (and the negative ones, which then stay finite)."""
    g = np.random.default_rng(3)
    lam = np.sort(g.uniform(-0.1, 4.0, 97))[::-1].copy()
    keep = _check_whiten(dtype, lam, c=0.05, rank_tol=0.0, max_rank=40, seed=3)
    assert keep.sum() == 40
    _check_whiten(dtype, lam, c=0.05, floor_add=0.25, floor_dev=0.125, scale=3.0, lam_floor=1e-2, seed=4)
    keep = _check_whiten(dtype, lam, c=0.2, floor_dev=1e-3, lam_floor=0.5, rank_tol=-np.inf, seed=5)
    assert keep.all()


# --------------------------------------------------------------------------------------------------
# ops.center_columns_
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m", [1, 31, 32, 33, 1000, 100003])
def test_center_columns(dtype, m):
    """Each n in {1, 31, 32, 33, 100} as a view of a wider parent (lda = n + 7; columns 0-2 and past the view must
    stay as they were).

    Integer data: every column sum is exact in double whatever the order, so the result is exactly
    ``a - T(sum / m)``.  Random data: with S the double sum (error <= (m - 1) u64 sum|a|), mu = T(S / m) and the
    subtraction rounding once in T, |out - (a - mean)| <= u_T |mean| + u_T |a - mean| + m u64 mean|a| to first
    order (the last term covers the sum and the division); the factor 1 + 4 u_T covers the second-order terms."""
    from cca_zoo_b200 import ops

    t = NP[dtype]
    g = np.random.default_rng(m)
    worst = 0.0
    for n in (1, 31, 32, 33, 100):
        for kind in ("integer", "random"):
            if kind == "integer":
                A = g.integers(-1000, 1001, size=(m, n)).astype(t)
            else:
                A = (g.standard_normal((m, n)) * 10.0 ** g.uniform(-3, 3, size=n) + g.uniform(-5, 5, size=n)).astype(t)
            parent = torch.from_numpy(g.standard_normal((m, n + 7)).astype(t)).cuda()
            parent[:, 3:3 + n] = torch.from_numpy(A).cuda()
            before = parent.clone()
            ops.center_columns_(_view(parent, 3, n))
            got = _view(parent, 3, n).cpu().numpy()
            assert _outside_unchanged(parent, before, 3, 3 + n), "center_columns_ wrote outside its view"
            if kind == "integer":
                mu = (A.astype(np.float64).sum(axis=0) / m).astype(t)
                assert np.array_equal(got, A - mu), f"n={n}: integer columns must centre exactly"
            else:
                Al = A.astype(np.longdouble)
                mean = Al.sum(axis=0) / m
                exact = Al - mean
                bound = (U[dtype] * (np.abs(mean) + np.abs(exact)) + m * U[torch.float64] * np.abs(Al).mean(axis=0)) \
                    * (1 + 4 * U[dtype])
                err = np.abs(got.astype(np.longdouble) - exact)
                worst = max(worst, float((err / bound).max()))
                assert np.all(err <= bound), f"n={n}: error / bound = {float((err / bound).max()):.3f}"
    print(f"center_columns_ {dtype} m={m}: max error / bound = {worst:.3f}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_center_columns_empty(dtype):
    from cca_zoo_b200 import ops

    for m, n in ((0, 5), (5, 0)):
        l0 = _launches()
        ops.center_columns_(torch.empty(m, n, dtype=dtype, device="cuda"))
        assert _launches() == l0


# --------------------------------------------------------------------------------------------------
# ops.frobenius_norm
# --------------------------------------------------------------------------------------------------
def _frob_ref(A):
    return np.sqrt((A.astype(np.longdouble) ** 2).sum())


def _frob_bound(dtype, mn):
    """Relative bound: the m n squares (exact for float32 input, one rounding each for float64) summed in double
    lose at most (m n - 1) u64, sqrt halves that and adds u64 / 2, so (m n + 1) u64 covers it with room; a float32
    result rounds once more (u32)."""
    return (mn + 1) * U[torch.float64] + (U[dtype] if dtype == torch.float32 else 0.0)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("m,n", [(1, 1), (37, 1), (1, 1500), (1000, 33), (511, 257)])
def test_frobenius_norm_strided(dtype, m, n):
    """A strided view (lda = n + 3) of entries spread over 2^+-20, against long double."""
    from cca_zoo_b200 import ops

    g = np.random.default_rng(m * n)
    A = (g.standard_normal((m, n)) * 2.0 ** g.uniform(-20, 20, size=(m, n))).astype(NP[dtype])
    parent = torch.zeros(m, n + 3, dtype=dtype, device="cuda")
    parent[:, 1:1 + n] = torch.from_numpy(A).cuda()
    l0 = _launches()
    got = float(ops.frobenius_norm(_view(parent, 1, n)).item())
    assert _launches() - l0 == 1
    ref = _frob_ref(A)
    ratio = float(abs(np.longdouble(got) - ref) / ref) / _frob_bound(dtype, m * n)
    print(f"frobenius_norm {dtype} {m}x{n}: relative error / bound = {ratio:.3f}")
    assert ratio <= 1.0


@pytest.mark.parametrize("dtype", DTYPES)
def test_frobenius_norm_special_values(dtype):
    """Zero and empty matrices give 0; an inf entry gives inf and a NaN entry NaN."""
    from cca_zoo_b200 import ops

    assert float(ops.frobenius_norm(torch.zeros(40, 70, dtype=dtype, device="cuda")).item()) == 0.0
    assert float(ops.frobenius_norm(torch.empty(0, 7, dtype=dtype, device="cuda")).item()) == 0.0
    A = torch.ones(30, 30, dtype=dtype, device="cuda")
    A[7, 3] = float("inf")
    assert float(ops.frobenius_norm(A).item()) == float("inf")
    A[7, 3] = float("nan")
    assert np.isnan(float(ops.frobenius_norm(A).item()))


def test_frobenius_norm_float64_is_exactly_scale_equivariant():
    """frob(2^k A) = 2^k frob(A) bit for bit for k in [-600, 600]: the kernel sums (a 2^-e)^2 with max |a 2^-e| in
    [0.5, 1), which is the same sum for every k.  Without that scaling the squares overflow to inf past about 2^511
    and vanish below about 2^-537.  At k = 0 the result is checked against long double."""
    from cca_zoo_b200 import ops

    g = np.random.default_rng(600)
    A = g.standard_normal((300, 41)) * 2.0 ** g.uniform(-8, 8, size=(300, 41))
    parent = torch.zeros(300, 45, dtype=torch.float64, device="cuda")
    parent[:, 2:43] = torch.from_numpy(A).cuda()
    f0 = float(ops.frobenius_norm(_view(parent, 2, 41)).item())
    ratio = float(abs(np.longdouble(f0) - _frob_ref(A)) / _frob_ref(A)) / _frob_bound(torch.float64, A.size)
    print(f"frobenius_norm float64 at unit scale: relative error / bound = {ratio:.3f}")
    assert ratio <= 1.0
    for k in range(-600, 601, 25):
        parent[:, 2:43] = torch.from_numpy(np.ldexp(A, k)).cuda()
        fk = float(ops.frobenius_norm(_view(parent, 2, 41)).item())
        assert fk == np.ldexp(f0, k), f"k={k}: frob(2^k A) = {fk!r}, 2^k frob(A) = {np.ldexp(f0, k)!r}"


def test_frobenius_norm_float32_over_its_range():
    """float32 input scaled by 2^k, k in [-120, 100]: the entries reach into the float32 subnormals at the low end and
    the norm stays below the float32 overflow at the high end; the bound holds at every scale."""
    from cca_zoo_b200 import ops

    g = np.random.default_rng(120)
    base = g.standard_normal((200, 63)) * 2.0 ** g.uniform(-3, 3, size=(200, 63))
    worst = 0.0
    for k in range(-120, 101, 20):
        A = np.ldexp(base, k).astype(np.float32)
        got = float(ops.frobenius_norm(torch.from_numpy(A).cuda()).item())
        ref = _frob_ref(A)
        ratio = float(abs(np.longdouble(got) - ref) / ref) / _frob_bound(torch.float32, A.size)
        worst = max(worst, ratio)
        assert ratio <= 1.0, f"k={k}: relative error / bound = {ratio:.3f}"
    print(f"frobenius_norm float32 over 2^-120 ... 2^100: max relative error / bound = {worst:.3f}")
