"""Device-side building blocks: torch CUDA tensors in, torch CUDA tensors out, arithmetic in libccab200.

torch is used for device memory (the caching allocator owns every buffer, including workspaces) and
for the current stream -- nothing else.  Every function fails loudly when called without CUDA.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib

_DT = {torch.float32: _lib.F32, torch.float64: _lib.F64}


def _require_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"{name} must be a CUDA tensor: cca_zoo_b200 runs on sm_90a only and has no CPU fallback"
        )


def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _ws(nbytes: int, device) -> torch.Tensor:
    return torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)


def _row_major(t: torch.Tensor, tma: bool) -> torch.Tensor:
    """2-D tensor with unit column stride (and, for TMA, 16-byte aligned rows)."""
    if t.dim() != 2:
        raise ValueError("expected a 2-D tensor")
    ok = t.stride(1) == 1 and t.stride(0) >= t.shape[1]
    if ok and tma:
        ok = t.data_ptr() % 16 == 0 and (t.stride(0) * t.element_size()) % 16 == 0
    if ok:
        return t
    if tma and (t.shape[1] * t.element_size()) % 16 != 0:
        per = 16 // t.element_size()
        ld = (t.shape[1] + per - 1) // per * per
        buf = torch.zeros((t.shape[0], ld), dtype=t.dtype, device=t.device)
        buf[:, : t.shape[1]] = t
        return buf[:, : t.shape[1]]
    return t.contiguous()


# --------------------------------------------------------------------------------------------------
# K1 / K2
# --------------------------------------------------------------------------------------------------
def moments(views, precision: str = "tf32x3b") -> torch.Tensor:
    """Block moments of the row shard held in ``views`` (list of (n, d_i) CUDA tensors, same dtype).

    Returns the additive double buffer ``[Dp*Dp + Dp]`` (see ccab_moments in include/ccab200.h).
    precision: "tf32" | "tf32x3" | "tf32x3b" (3xTF32 with bf16 cross terms) | "exact" (float64 views always use "exact").
    """
    lib = _lib.load()
    if not (1 <= len(views) <= _lib.MAX_VIEWS):
        raise ValueError(f"between 1 and {_lib.MAX_VIEWS} views are supported, got {len(views)}")
    dt = views[0].dtype
    for v in views:
        _require_cuda(v, "view")
        if v.dtype != dt or v.dtype not in _DT:
            raise ValueError("views must share one dtype (float32 or float64)")
        if v.shape[0] != views[0].shape[0]:
            raise ValueError("All views must have the same number of samples.")
        if v.device != views[0].device:
            raise ValueError(f"views live on different devices: {v.device} vs {views[0].device}")
    prec = {"tf32": _lib.PREC_TF32, "tf32x3": _lib.PREC_TF32X3, "exact": _lib.PREC_EXACT,
            "tf32x3b": _lib.PREC_TF32X3B}[precision]
    if dt == torch.float64:
        prec = _lib.PREC_EXACT
    vs = [_row_major(v, tma=prec != _lib.PREC_EXACT) for v in views]
    n = vs[0].shape[0]
    dims = _lib.i64_array([v.shape[1] for v in vs])
    lds = _lib.i64_array([v.stride(0) for v in vs])
    ptrs = (C.c_void_p * len(vs))(*[v.data_ptr() for v in vs])
    dev = vs[0].device
    size = lib.ccab_moments_size(len(vs), dims)
    if size < 0:
        raise ValueError(_lib.last_error())
    out = torch.empty(size, dtype=torch.float64, device=dev)
    wsb = lib.ccab_moments_workspace_bytes(_DT[dt], prec, len(vs), dims, n)
    ws = _ws(wsb, dev)
    with torch.cuda.device(dev):
        rc = lib.ccab_moments(_DT[dt], prec, len(vs), ptrs, dims, lds, n, _ptr(out), _ptr(ws), ws.numel(), _stream(out))
    _lib.check(rc, "ccab_moments")
    return out


def moments_pack(mom: torch.Tensor, dims, n_local) -> torch.Tensor:
    """The exchange-step message (ccab_moments_pack): upper block triangle | column sums | n | reserved."""
    lib = _lib.load()
    _require_cuda(mom, "moments")
    d = _lib.i64_array(dims)
    size = lib.ccab_moments_packed_size(len(dims), d)
    if size < 0:
        raise ValueError(_lib.last_error())
    packed = torch.empty(size, dtype=torch.float64, device=mom.device)
    with torch.cuda.device(mom.device):
        rc = lib.ccab_moments_pack(len(dims), d, _ptr(mom), float(n_local), _ptr(packed), _stream(mom))
    _lib.check(rc, "ccab_moments_pack")
    return packed


def moments_unpack(packed: torch.Tensor, dims, out=None):
    """(moments buffer, n_total as a 1-element device tensor) from an all-reduced message."""
    lib = _lib.load()
    _require_cuda(packed, "packed")
    d = _lib.i64_array(dims)
    size = lib.ccab_moments_size(len(dims), d)
    mom = out if out is not None else torch.empty(size, dtype=torch.float64, device=packed.device)
    with torch.cuda.device(packed.device):
        rc = lib.ccab_moments_unpack(len(dims), d, _ptr(packed), _ptr(mom), _stream(packed))
    _lib.check(rc, "ccab_moments_unpack")
    return mom, packed[-2:-1]


def moments_exchange_nvls(mom: torch.Tensor, dims, n_local, sym: torch.Tensor, multicast_ptr: int, pads_dev_ptr: int,
                          rank: int, world: int, pad_slots: int, epoch: int):
    """Fused exchange step (ccab_moments_exchange_nvls): pack, in-switch all-reduce on the multicast address, unpack --
    one kernel, in place on ``mom``.  Returns the summed sample count as a 1-element device tensor."""
    lib = _lib.load()
    _require_cuda(mom, "moments")
    d = _lib.i64_array(dims)
    n_dev = torch.empty(1, dtype=torch.float64, device=mom.device)
    with torch.cuda.device(mom.device):
        rc = lib.ccab_moments_exchange_nvls(len(dims), d, _ptr(mom), float(n_local), _ptr(sym), C.c_void_p(multicast_ptr),
                                            C.c_void_p(pads_dev_ptr), int(rank), int(world), int(pad_slots),
                                            sym.numel(), int(epoch) & 0xFFFFFFFF, _ptr(n_dev), _stream(mom))
    _lib.check(rc, "ccab_moments_exchange_nvls")
    return n_dev


#: a column whose pilot mean^2 / variance exceeds this is accumulated shifted (relative covariance error of the float32
#: moment kernels ~ 1e-6 * ratio; float64 kernels have 9 more digits and never need it below 1e8)
SHIFT_RATIO = {torch.float32: 16.0, torch.float64: 1e8}
PILOT_ROWS = 4096


def column_pilot(views):
    """Per view x0 (pilot column means of the leading rows, device tensors in the views' dtype) and the largest
    mean^2 / variance over all columns (ONE host read-back: it decides whether an extra pass is worth taking)."""
    lib = _lib.load()
    ratio = torch.zeros(1, dtype=torch.float32, device=views[0].device)
    x0 = []
    for v in views:
        _require_cuda(v, "view")
        vv = v if v.stride(1) == 1 else v.contiguous()
        o = torch.empty(v.shape[1], dtype=v.dtype, device=v.device)
        with torch.cuda.device(v.device):
            rc = lib.ccab_column_pilot(_DT[v.dtype], _ptr(vv), min(int(v.shape[0]), PILOT_ROWS), int(v.shape[1]),
                                       vv.stride(0), _ptr(o), _ptr(ratio), _stream(v))
        _lib.check(rc, "ccab_column_pilot")
        x0.append(o)
    return x0, float(ratio.item())


def shift_rows(v, x0):
    """v - x0 (row-major copy with a TMA-friendly leading dimension)."""
    lib = _lib.load()
    vv = v if v.stride(1) == 1 else v.contiguous()
    per = 16 // v.element_size()
    ld = (v.shape[1] + per - 1) // per * per
    out = torch.empty((v.shape[0], ld), dtype=v.dtype, device=v.device)
    with torch.cuda.device(v.device):
        rc = lib.ccab_shift_rows(_DT[v.dtype], _ptr(vv), int(v.shape[0]), int(v.shape[1]), vv.stride(0), _ptr(x0),
                                 _ptr(out), ld, _stream(v))
    _lib.check(rc, "ccab_shift_rows")
    return out[:, : v.shape[1]]


def moments_unshift_(mom, dims, x0, n_rows):
    """In place: moments of the shifted views -> raw moments (float64 algebra)."""
    lib = _lib.load()
    ptrs = (C.c_void_p * len(x0))(*[0 if t is None else t.data_ptr() for t in x0])
    dt = next(t.dtype for t in x0 if t is not None)
    with torch.cuda.device(mom.device):
        rc = lib.ccab_moments_unshift(_DT[dt], len(dims), _lib.i64_array(dims), _ptr(mom), ptrs, float(n_rows),
                                      _stream(mom))
    _lib.check(rc, "ccab_moments_unshift")
    return mom


def moments_safe(views, precision: str = "tf32x3b", x0=None):
    """``moments`` with the shifted accumulation when it matters: a pilot over the leading rows decides (one tiny
    kernel per view and one scalar read-back); badly centred views are accumulated as X - x0 and the raw moments are
    rebuilt in float64.  ``x0`` given = shift by it unconditionally (streamed fits keep one x0 for all chunks).
    Returns (moments, x0 or None)."""
    if x0 is None:
        cand, ratio = column_pilot(views)
        if not ratio > SHIFT_RATIO[views[0].dtype]:
            return moments(views, precision=precision), None
        x0 = cand
    shifted = [shift_rows(v, o) for v, o in zip(views, x0)]
    mom = moments(shifted, precision=precision)
    return moments_unshift_(mom, [int(v.shape[1]) for v in views], x0, views[0].shape[0]), x0


def covariance(mom: torch.Tensor, dims, n_total: float, center: bool = True, dtype=torch.float64):
    """(C [D,D], mean [D]) from an (all-reduced) moments buffer."""
    lib = _lib.load()
    _require_cuda(mom, "moments")
    D = int(sum(dims))
    expect = lib.ccab_moments_size(len(dims), _lib.i64_array(dims))
    if expect < 0:
        raise ValueError(_lib.last_error())
    if mom.dtype != torch.float64 or mom.numel() != expect or not mom.is_contiguous():
        raise ValueError(f"moments buffer must be a contiguous float64 tensor of {expect} elements for widths "
                         f"{list(dims)}, got {mom.dtype} x {mom.numel()}")
    if not n_total >= 2:
        raise ValueError(f"at least 2 samples are needed for a covariance, got n = {n_total}")
    Cm = torch.empty((D, D), dtype=dtype, device=mom.device)
    mean = torch.empty(D, dtype=dtype, device=mom.device)
    with torch.cuda.device(mom.device):
        rc = lib.ccab_covariance(_DT[dtype], len(dims), _lib.i64_array(dims), _ptr(mom), float(n_total),
                                 1 if center else 0, _ptr(Cm), D, _ptr(mean), _stream(mom))
    _lib.check(rc, "ccab_covariance")
    return Cm, mean


# --------------------------------------------------------------------------------------------------
# K3 / K4
# --------------------------------------------------------------------------------------------------
def _jacobi_converged(what, sweeps, offdiag, caller_checks):
    """The library reports a solve that ran out of sweeps as a negative sweep count: no silent use of unconverged
    eigen / singular vectors.  Callers that ask for the diagnostics (return_info=True) decide themselves."""
    if sweeps < 0 and not caller_checks:
        if not (offdiag == offdiag) or offdiag > 0.5:      # NaN or no progress at all: the vectors are meaningless
            raise RuntimeError(f"{what}: the Jacobi iteration did not converge in {-sweeps} sweeps "
                               f"(normalised off-diagonal {offdiag:.3e}); the matrix may contain NaN / inf or be "
                               f"pathologically scaled")
        import warnings

        warnings.warn(f"{what}: the Jacobi iteration stopped after {-sweeps} sweeps with a normalised off-diagonal of "
                      f"{offdiag:.3e} (tolerance not reached: nearly rank-deficient input); the trailing eigen / "
                      f"singular vectors may be inaccurate", RuntimeWarning, stacklevel=3)


def syevj(A: torch.Tensor, shift: float = 0.0, return_info: bool = False):
    """Symmetric eigendecomposition.  A: (n,n) or (batch,n,n).  Returns (evals desc, evecs_t) where
    evecs_t[..., j, :] is the j-th eigenvector."""
    lib = _lib.load()
    _require_cuda(A, "A")
    squeeze = A.dim() == 2
    Ab = (A.unsqueeze(0) if squeeze else A).contiguous()
    batch, n, n2 = Ab.shape
    if n != n2:
        raise ValueError("square matrices expected")
    dt = _DT[Ab.dtype]
    evals = torch.empty((batch, n), dtype=Ab.dtype, device=Ab.device)
    evt = torch.empty((batch, n, n), dtype=Ab.dtype, device=Ab.device)
    ws = _ws(lib.ccab_syevj_workspace_bytes(dt, n, batch), Ab.device)
    info = C.c_int(0)
    off = C.c_float(0)
    with torch.cuda.device(Ab.device):
        rc = lib.ccab_syevj(dt, n, batch, _ptr(Ab), n, n * n, float(shift), _ptr(evals), _ptr(evt), n,
                            C.byref(info), C.byref(off), _ptr(ws), ws.numel(), _stream(Ab))
    _lib.check(rc, "ccab_syevj")
    _jacobi_converged("ccab_syevj", info.value, off.value, return_info)
    if squeeze:
        evals, evt = evals[0], evt[0]
    if return_info:
        return evals, evt, {"sweeps": abs(info.value), "offdiag": off.value, "converged": info.value > 0}
    return evals, evt


def syevj_small(A: torch.Tensor):
    """Single-launch eigensolver for small symmetric matrices (n <= 128 float32 / 104 float64), (n,n) or (batch,n,n).
    Returns (evals desc, evecs_t rows, info int32[batch] on the device: sweeps, negative = not converged)."""
    lib = _lib.load()
    _require_cuda(A, "A")
    squeeze = A.dim() == 2
    Ab = (A.unsqueeze(0) if squeeze else A).contiguous()
    batch, n, _ = Ab.shape
    evals = torch.empty((batch, n), dtype=Ab.dtype, device=Ab.device)
    evt = torch.empty((batch, n, n), dtype=Ab.dtype, device=Ab.device)
    info = torch.empty(batch, dtype=torch.int32, device=Ab.device)
    with torch.cuda.device(Ab.device):
        rc = lib.ccab_syevj_small(_DT[Ab.dtype], n, batch, _ptr(Ab), n, n * n, _ptr(evals), _ptr(evt), n, _ptr(info),
                                  _stream(Ab))
    _lib.check(rc, "ccab_syevj_small")
    if squeeze:
        return evals[0], evt[0], info
    return evals, evt, info


def gesvj(Gt: torch.Tensor, return_info: bool = False):
    """SVD of G (m x n) given as its transpose ``Gt`` (n x m, row-major: row j = column j of G).

    Returns (sigma [n] desc, right_t [n,n] rows = right singular vectors of G,
             left_t [n,m] rows = left singular vectors of G)."""
    lib = _lib.load()
    _require_cuda(Gt, "Gt")
    Gt = Gt.contiguous()
    n, m = Gt.shape
    dt = _DT[Gt.dtype]
    sigma = torch.empty(n, dtype=Gt.dtype, device=Gt.device)
    right = torch.empty((n, n), dtype=Gt.dtype, device=Gt.device)
    left = torch.zeros((n, m), dtype=Gt.dtype, device=Gt.device)
    ws = _ws(lib.ccab_gesvj_workspace_bytes(dt, m, n), Gt.device)
    info = C.c_int(0)
    off = C.c_float(0)
    with torch.cuda.device(Gt.device):
        rc = lib.ccab_gesvj(dt, m, n, _ptr(Gt), m, _ptr(sigma), _ptr(right), n, _ptr(left), m, C.byref(info),
                            C.byref(off), _ptr(ws), ws.numel(), _stream(Gt))
    _lib.check(rc, "ccab_gesvj")
    _jacobi_converged("ccab_gesvj", info.value, off.value, return_info)
    if return_info:
        return sigma, right, left, {"sweeps": abs(info.value), "offdiag": off.value, "converged": info.value > 0}
    return sigma, right, left


# --------------------------------------------------------------------------------------------------
# dense glue
# --------------------------------------------------------------------------------------------------
def gemm(A, B, transa=False, transb=False, alpha=1.0, beta=0.0, out=None):
    """out = alpha * op(A) @ op(B) + beta * out  (row-major views with unit inner stride)."""
    lib = _lib.load()
    _require_cuda(A, "A")
    _require_cuda(B, "B")
    A = _row_major(A, False)
    B = _row_major(B, False)
    m, k = (A.shape[1], A.shape[0]) if transa else A.shape
    k2, n = (B.shape[1], B.shape[0]) if transb else B.shape
    if k != k2:
        raise ValueError(f"gemm inner dimensions differ: {k} vs {k2}")
    if A.dtype != B.dtype or A.device != B.device:
        raise ValueError(f"gemm operands differ in dtype/device: {A.dtype}@{A.device} vs {B.dtype}@{B.device}")
    if out is None:
        out = torch.empty((m, n), dtype=A.dtype, device=A.device)
        beta = 0.0
    elif (out.dim() != 2 or tuple(out.shape) != (m, n) or out.stride(1) != 1 or out.stride(0) < n
          or out.dtype != A.dtype or out.device != A.device):
        raise ValueError(f"gemm `out` must be a row-major ({m}, {n}) {A.dtype} tensor on {A.device}, got "
                         f"{tuple(out.shape)} strides {out.stride()} {out.dtype} on {out.device}")
    with torch.cuda.device(A.device):
        rc = lib.ccab_gemm(_DT[A.dtype], int(transa), int(transb), m, n, k, float(alpha), _ptr(A), A.stride(0),
                           _ptr(B), B.stride(0), float(beta), _ptr(out), out.stride(0), _stream(A))
    _lib.check(rc, "ccab_gemm")
    return out


def _tc_ok(t: torch.Tensor) -> bool:
    return (t.dtype == torch.float32 and t.dim() in (2, 3) and t.stride(-1) == 1 and t.data_ptr() % 16 == 0
            and t.stride(-2) % 4 == 0 and t.stride(-2) >= t.shape[-1] and (t.dim() == 2 or t.stride(0) % 4 == 0))


def gemm_tc(A, B, transa=False, transb=False, alpha=1.0, beta=0.0, out=None, out_t=None, want_c=True,
            lower_only=False):
    """Tensor-core GEMM (ccab_gemm_tc): float32, 2-D or batched 3-D operands (row-major, unit inner stride).

    out = alpha * op(A) @ op(B) + beta * out; ``out_t`` (optional) receives the transpose as well.  Returns
    ``out`` (or ``out_t`` when ``want_c`` is False).  Raises ValueError when the operands do not meet the TMA
    alignment rules (16-byte aligned, leading dimensions % 4 == 0): callers use ``gemm`` then."""
    lib = _lib.load()
    _require_cuda(A, "A")
    _require_cuda(B, "B")
    if not (_tc_ok(A) and _tc_ok(B)) or A.dim() != B.dim():
        raise ValueError("gemm_tc: float32 row-major operands, 16-byte aligned, leading dimensions % 4 == 0")
    batched = A.dim() == 3
    batch = A.shape[0] if batched else 1
    if batched and B.shape[0] != batch:
        raise ValueError("gemm_tc: batch sizes differ")
    m, k = (A.shape[-1], A.shape[-2]) if transa else (A.shape[-2], A.shape[-1])
    k2, n = (B.shape[-1], B.shape[-2]) if transb else (B.shape[-2], B.shape[-1])
    if k != k2:
        raise ValueError(f"gemm inner dimensions differ: {k} vs {k2}")
    shape = (batch, m, n) if batched else (m, n)
    shape_t = (batch, n, m) if batched else (n, m)
    if out is None and want_c:
        out = torch.empty(shape, dtype=A.dtype, device=A.device)
        beta = 0.0
    for t, shp, nm in ((out, shape, "out"), (out_t, shape_t, "out_t")):
        if t is not None and (tuple(t.shape) != shp or t.stride(-1) != 1 or t.dtype != A.dtype or t.device != A.device):
            raise ValueError(f"gemm_tc `{nm}` must be a row-major {shp} float32 tensor on {A.device}")
    if out is None and out_t is None:
        raise ValueError("gemm_tc: no output requested")
    sa = A.stride(0) if batched else 0
    sb = B.stride(0) if batched else 0
    with torch.cuda.device(A.device):
        rc = lib.ccab_gemm_tc(int(transa), int(transb), m, n, k, float(alpha), _ptr(A), A.stride(-2), sa, _ptr(B),
                              B.stride(-2), sb, float(beta), _ptr(out), 0 if out is None else out.stride(-2),
                              (out.stride(0) if (batched and out is not None) else 0), _ptr(out_t),
                              0 if out_t is None else out_t.stride(-2),
                              (out_t.stride(0) if (batched and out_t is not None) else 0), batch, int(lower_only),
                              _stream(A))
    _lib.check(rc, "ccab_gemm_tc")
    return out if want_c else out_t


def gemm_batched(A, B, transa=False, transb=False, alpha=1.0):
    """Batched product of (batch, m, k) x (batch, k, n) stacks: tensor cores for TMA-addressable float32 operands,
    a loop over ``gemm`` otherwise."""
    if _tc_ok(A) and _tc_ok(B):
        return gemm_tc(A, B, transa=transa, transb=transb, alpha=alpha)
    return torch.stack([gemm(A[i], B[i], transa=transa, transb=transb, alpha=alpha) for i in range(A.shape[0])])


def whiten_rows(lam, Vt, c, floor_add=0.0, floor_dev=None, scale=1.0, rank_tol=0.0, max_rank=None,
                lam_floor=-1e300):
    """(Wt, g, rank_dev) -- see ccab_whiten_rows."""
    lib = _lib.load()
    _require_cuda(Vt, "Vt")
    d = Vt.shape[0]
    Wt = torch.empty_like(Vt)
    g = torch.empty(d, dtype=Vt.dtype, device=Vt.device)
    rank = torch.zeros(1, dtype=torch.int32, device=Vt.device)
    with torch.cuda.device(Vt.device):
        rc = lib.ccab_whiten_rows(_DT[Vt.dtype], d, _ptr(lam), _ptr(Vt), Vt.stride(0), float(c), float(floor_add),
                                  _ptr(floor_dev), float(scale), float(rank_tol),
                                  int(d if max_rank is None else max_rank), float(lam_floor), _ptr(Wt), Wt.stride(0),
                                  _ptr(g),
                                  _ptr(rank), _stream(Vt))
    _lib.check(rc, "ccab_whiten_rows")
    return Wt, g, rank


def ccaloss_small(Cm, d1, d2, eps):
    """Fused loss stage for widths <= 64: returns (loss[1], G11, P, G22, min_pivot[1]) device tensors."""
    lib = _lib.load()
    _require_cuda(Cm, "C")
    dev, dt = Cm.device, Cm.dtype
    loss = torch.empty(1, dtype=dt, device=dev)
    minp = torch.empty(1, dtype=dt, device=dev)
    G11 = torch.empty((d1, d1), dtype=dt, device=dev)
    P = torch.empty((d1, d2), dtype=dt, device=dev)
    G22 = torch.empty((d2, d2), dtype=dt, device=dev)
    with torch.cuda.device(dev):
        rc = lib.ccab_ccaloss_small(_DT[dt], d1, d2, _ptr(Cm), Cm.stride(0), float(eps), _ptr(loss), _ptr(G11), _ptr(P),
                                    _ptr(G22), _ptr(minp), _stream(Cm))
    _lib.check(rc, "ccab_ccaloss_small")
    return loss, G11, P, G22, minp


def ccaloss_fwd(z1, z2, eps, precision="exact"):
    """Device-side deep-CCA objective (ccab_ccaloss_fwd): returns (loss[1], saved, flags int32[3]) -- all on the device,
    nothing read back.  z1 / z2: row-major CUDA tensors of one dtype."""
    lib = _lib.load()
    _require_cuda(z1, "z1")
    _require_cuda(z2, "z2")
    n, d1, d2 = z1.shape[0], z1.shape[1], z2.shape[1]
    dt = _DT[z1.dtype]
    prec = {"tf32": _lib.PREC_TF32, "tf32x3": _lib.PREC_TF32X3, "exact": _lib.PREC_EXACT,
            "tf32x3b": _lib.PREC_TF32X3B}[precision]
    if z1.dtype == torch.float64:
        prec = _lib.PREC_EXACT
    loss = torch.empty(1, dtype=z1.dtype, device=z1.device)
    saved = torch.empty(d1 * d1 + d1 * d2 + d2 * d2 + d1 + d2, dtype=z1.dtype, device=z1.device)
    flags = torch.empty(3, dtype=torch.int32, device=z1.device)
    ws = _ws(lib.ccab_ccaloss_workspace_bytes(dt, prec, d1, d2, n), z1.device)
    with torch.cuda.device(z1.device):
        rc = lib.ccab_ccaloss_fwd(dt, prec, _ptr(z1), z1.stride(0), _ptr(z2), z2.stride(0), n, d1, d2, float(eps),
                                  _ptr(loss), _ptr(saved), _ptr(flags), _ptr(ws), ws.numel(), _stream(z1))
    _lib.check(rc, "ccab_ccaloss_fwd")
    return loss, saved, flags


def ccaloss_bwd(z1, z2, saved, grad_out):
    """Analytic backward of the deep-CCA objective (ccab_ccaloss_bwd): (dL/dz1, dL/dz2), already scaled by grad_out."""
    lib = _lib.load()
    n, d1, d2 = z1.shape[0], z1.shape[1], z2.shape[1]
    g1 = torch.empty((n, d1), dtype=z1.dtype, device=z1.device)
    g2 = torch.empty((n, d2), dtype=z1.dtype, device=z1.device)
    with torch.cuda.device(z1.device):
        rc = lib.ccab_ccaloss_bwd(_DT[z1.dtype], _ptr(z1), z1.stride(0), _ptr(z2), z2.stride(0), n, d1, d2, _ptr(saved),
                                  _ptr(grad_out), _ptr(g1), d1, _ptr(g2), d2, _stream(z1))
    _lib.check(rc, "ccab_ccaloss_bwd")
    return g1, g2


def potrf_inv_(A, pivot_tol=0.0):
    """In place lower Cholesky of A (n x n or batch x n x n, row-major) AND the explicit inverse of the factor.

    Returns (Linv, info): Linv like A (zeros above the diagonal), info int32[batch] on the device (0 = ok)."""
    lib = _lib.load()
    _require_cuda(A, "A")
    squeeze = A.dim() == 2
    Ab = A.unsqueeze(0) if squeeze else A
    if Ab.dim() != 3 or Ab.shape[1] != Ab.shape[2] or Ab.stride(2) != 1 or Ab.dtype not in _DT:
        raise ValueError("square row-major float32/float64 matrices expected")
    batch, n, _ = Ab.shape
    Linv = torch.empty((batch, n, n), dtype=A.dtype, device=A.device)
    info = torch.empty(batch, dtype=torch.int32, device=A.device)
    dt = _DT[A.dtype]
    ws = _ws(lib.ccab_potrf_inv_workspace_bytes(dt, n, batch), A.device)
    with torch.cuda.device(A.device):
        rc = lib.ccab_potrf_inv(dt, n, batch, _ptr(Ab), Ab.stride(1), Ab.stride(0) if batch > 1 else 0, _ptr(Linv), n,
                                n * n, float(pivot_tol), _ptr(info), _ptr(ws), ws.numel(), _stream(A))
    _lib.check(rc, "ccab_potrf_inv")
    return (Linv[0] if squeeze else Linv), info


# status bits of the device-side fit (csrc/fit.cuh)
FIT_NOT_POSITIVE_DEFINITE, FIT_NOT_CONVERGED, FIT_NON_FINITE, FIT_TOO_FEW_SAMPLES = 1, 2, 4, 8
FIT_HEADER_DOUBLES = 32


def rcca_fit_workspace_bytes(dims, k: int, p: int, dtype) -> int:
    """Workspace of ``rcca_fit`` in bytes; 0 when the fit refuses this (dims, k, p) in ``dtype``."""
    return int(_lib.load().ccab_rcca_fit_workspace_bytes(_DT[dtype], _lib.i64_array(dims), int(k), int(p)))


def mcca_fit_workspace_bytes(dims, k: int, p: int, dtype) -> int:
    """Workspace of ``mcca_fit`` in bytes; 0 when the fit refuses this (dims, k, p) in ``dtype``."""
    return int(_lib.load().ccab_mcca_fit_workspace_bytes(_DT[dtype], len(dims), _lib.i64_array(dims), int(k), int(p)))


def rcca_fit(mom: torch.Tensor, dims, n_host, n_dev, center: bool, c, k: int, p: int, iters: int, dtype):
    """Device-side rCCA fit (ccab_rcca_fit): moments -> result block, asynchronous, nothing read back.

    Returns (block, offsets): ``block`` is a uint8 CUDA tensor, ``offsets`` = byte offsets of
    (mean float64[D], sigma[k], W1[d1 x k], W2[d2 x k], total).  ``decode_fit_block`` turns a host copy into arrays."""
    lib = _lib.load()
    _require_cuda(mom, "moments")
    dt = _DT[dtype]
    d = _lib.i64_array(dims)
    offs = (C.c_int64 * 5)()
    _lib.check(lib.ccab_rcca_fit_result_layout(dt, d, int(k), int(p), offs), "ccab_rcca_fit_result_layout")
    offsets = [int(x) for x in offs]
    block = torch.empty(offsets[4] + 256, dtype=torch.uint8, device=mom.device)
    shift = (-block.data_ptr()) % 256
    block = block[shift:shift + offsets[4]]
    wsb = lib.ccab_rcca_fit_workspace_bytes(dt, d, int(k), int(p))
    ws = _ws(wsb, mom.device)
    cc = (C.c_double * 2)(float(c[0]), float(c[1]))
    with torch.cuda.device(mom.device):
        rc = lib.ccab_rcca_fit(dt, d, _ptr(mom), _ptr(n_dev), float(n_host if n_host is not None else 0.0),
                               1 if center else 0, cc, int(k), int(p), int(iters), _ptr(block), block.numel(), _ptr(ws),
                               ws.numel(), _stream(mom))
    _lib.check(rc, "ccab_rcca_fit")
    return block, offsets


def mcca_fit(mom: torch.Tensor, dims, n_host, n_dev, center: bool, c, eps: float, k: int, p: int, iters: int, dtype):
    """Device-side MCCA fit (ccab_mcca_fit); same conventions as ``rcca_fit``; offsets = (mean, eigenvalues,
    W_1 .. W_m, total)."""
    lib = _lib.load()
    _require_cuda(mom, "moments")
    dt = _DT[dtype]
    m = len(dims)
    d = _lib.i64_array(dims)
    offs = (C.c_int64 * (m + 3))()
    _lib.check(lib.ccab_mcca_fit_result_layout(dt, m, d, int(k), int(p), offs), "ccab_mcca_fit_result_layout")
    offsets = [int(x) for x in offs]
    block = torch.empty(offsets[-1] + 256, dtype=torch.uint8, device=mom.device)
    shift = (-block.data_ptr()) % 256
    block = block[shift:shift + offsets[-1]]
    ws = _ws(lib.ccab_mcca_fit_workspace_bytes(dt, m, d, int(k), int(p)), mom.device)
    cc = (C.c_double * m)(*[float(x) for x in c])
    with torch.cuda.device(mom.device):
        rc = lib.ccab_mcca_fit(dt, m, d, _ptr(mom), _ptr(n_dev), float(n_host if n_host is not None else 0.0),
                               1 if center else 0, cc, float(eps), int(k), int(p), int(iters), _ptr(block),
                               block.numel(), _ptr(ws), ws.numel(), _stream(mom))
    _lib.check(rc, "ccab_mcca_fit")
    return block, offsets


def decode_fit_block(host: torch.Tensor, offsets, dims, k: int, dtype):
    """(header float64[32], mean float64[D], sigma[k], [W_i (d_i x k)]) as numpy views of a HOST copy of the block."""
    import numpy as np

    buf = host.numpy()
    np_dt = np.float32 if dtype == torch.float32 else np.float64
    D = int(sum(dims))
    hdr = buf[:8 * FIT_HEADER_DOUBLES].view(np.float64)
    mean = buf[offsets[0]:offsets[0] + 8 * D].view(np.float64)
    sig = buf[offsets[1]:offsets[1] + np_dt().itemsize * k].view(np_dt)
    ws = []
    for i, d in enumerate(dims):
        o = offsets[2 + i]
        ws.append(buf[o:o + np_dt().itemsize * d * k].view(np_dt).reshape(d, k))
    return hdr, mean, sig, ws


def column_means(mom: torch.Tensor, dims, n_total: float):
    """Column means of the views (float64 numpy, hstack order) from the column sums that follow the padded Dp x Dp
    moment matrix in a moments buffer (each view padded to a multiple of 128 columns, see ccab_moments_size)."""
    import numpy as np

    pads = [(int(p) + 127) // 128 * 128 for p in dims]
    Dp = sum(pads)
    sums = mom[Dp * Dp:Dp * Dp + Dp].to(torch.float64).cpu().numpy()
    off = np.concatenate([[0], np.cumsum(pads)]).astype(int)
    return np.concatenate([sums[off[i]:off[i] + int(p)] for i, p in enumerate(dims)]) / float(n_total)


ALS_KINDS = {"pls": 0, "pmd": 1, "parkhomenko": 2, "span": 3, "admm": 4, "elastic": 5, "ipls": 6}


ALS_RCOND_F64 = 1e-12   # relative eigenvalue cut of the alpha l1 = 0 regressions on an exact (float64) Gram matrix


def als_fit(cov, dims, n_total, kind: str, params, init, max_iter: int, tol: float, mu: float | None = None):
    """Sparse / ALS fit on the block covariance (ccab_als_fit): ``cov`` is the float64 D x D covariance on the device,
    the iteration runs on the Gram matrix (n_total - 1) cov.  ``init`` (k x D float64, host or device) holds the
    initial weights of every dimension.  ``params``: one value per view, or for "elastic" / "ipls" the pairs
    (alpha_i, l1_ratio_i) flattened, followed for "ipls" by the D column means of the views (zeros when centred).
    ``mu``: the ADMM penalty (default 1), or for "elastic" / "ipls" the relative eigenvalue cut of the alpha l1 = 0
    solves (default ALS_RCOND_F64).  Returns (W (D x k float64 numpy), sweeps per dimension) after ONE copy to the
    host; a dimension in which a coordinate descent stopped at its sweep limit above the KKT bound is reported by a
    ConvergenceWarning, as sklearn's solvers do."""
    import numpy as np

    lib = _lib.load()
    _require_cuda(cov, "cov")
    if cov.dtype != torch.float64:
        raise ValueError("als_fit iterates in float64")
    cov = cov.contiguous()
    D, k = int(sum(dims)), int(init.shape[0])
    d = _lib.i64_array(dims)
    init = torch.as_tensor(init, dtype=torch.float64).to(cov.device).contiguous()
    out = torch.empty(D * k + (k + 1) // 2, dtype=torch.float64, device=cov.device)   # W | int32 sweeps[k]
    regression = kind in ("elastic", "ipls")
    if mu is None:
        mu = ALS_RCOND_F64 if regression else 1.0
    ws_bytes = (lib.ccab_als_regression_workspace_bytes if regression else lib.ccab_als_fit_workspace_bytes)(len(dims), d)
    ws = _ws(ws_bytes, cov.device)
    if regression:
        want = 2 * len(dims) + (D if kind == "ipls" else 0)
        if len(params) != want:
            raise ValueError(f"als_fit({kind!r}) takes {want} params, got {len(params)}")
    pp = (C.c_double * max(len(params), len(dims)))(*[float(x) for x in params])
    with torch.cuda.device(cov.device):
        rc = lib.ccab_als_fit(ALS_KINDS[kind], len(dims), d, _ptr(cov), float(n_total - 1), float(n_total), pp,
                              float(mu), _ptr(init), k, int(max_iter), float(tol), _ptr(out),
                              C.c_void_p(out.data_ptr() + 8 * D * k), _ptr(ws), ws.numel(), _stream(cov))
    _lib.check(rc, "ccab_als_fit")
    host = out.cpu().numpy()
    iters = host[D * k:].view(np.int32)[:k].astype(int).tolist()
    capped = [d for d, it in enumerate(iters) if it < 0]
    if capped:
        import warnings

        from sklearn.exceptions import ConvergenceWarning

        warnings.warn(f"als_fit({kind!r}): a coordinate descent of latent dimension(s) {capped} stopped at its sweep "
                      "limit above the KKT bound (1e-12 max(1, ||b||_inf)); consider a larger alpha",
                      ConvergenceWarning, stacklevel=2)
    return host[:D * k].reshape(D, k).copy(), [abs(it) for it in iters]


EY_HEADER = 8      # doubles in front of W and the velocity in the state block of ccab_ey_fit
EY_MAX_K = 32


class EyFit:
    """One Eckart-Young gradient fit on the device (ccab_ey_fit): the state block (header | W (k x D) | velocity) and
    the workspace of a route, kept across the chunked calls of one fit.

    ``cov`` (float64 D x D CUDA tensor) selects the covariance route; otherwise ``views`` (CUDA tensors of one dtype,
    unit column stride) and ``batch`` the mini-batch route.  ``init`` is the D x k float64 host array of initial
    weights.  ``run(n_steps, idx=None)`` enqueues one call; ``stopped()`` reads the stop flag back (one small copy);
    ``result()`` copies the state block to the host once and returns (W (D x k float64 numpy), steps taken)."""

    def __init__(self, dims, init, c, learning_rate, momentum, tol, cov=None, views=None, batch=0):
        import numpy as np

        self.lib = _lib.load()
        self.dims = [int(d) for d in dims]
        self.D, self.k = int(sum(self.dims)), int(init.shape[1])
        self.hyper = (float(c), float(learning_rate), float(momentum), float(tol))
        self.cov, self.batch = cov, int(batch) if cov is None else 0
        ref = cov if cov is not None else views[0]
        _require_cuda(ref, "cov" if cov is not None else "view")
        self.device = ref.device
        self._d = _lib.i64_array(self.dims)
        if cov is not None:
            if cov.dtype != torch.float64 or tuple(cov.shape) != (self.D, self.D):
                raise ValueError("the covariance route takes the float64 D x D covariance")
            self.cov = cov.contiguous()
            self._views, self._ld, self.dtype = None, None, _lib.F64
        else:
            for v in views:
                _require_cuda(v, "view")
                if v.dtype != views[0].dtype or v.dtype not in _DT or v.stride(1) != 1 or v.device != self.device:
                    raise ValueError("the mini-batch route takes CUDA views of one dtype with unit column stride")
            self.views = views
            self._views = (C.c_void_p * len(views))(*[v.data_ptr() for v in views])
            self._ld = _lib.i64_array([v.stride(0) for v in views])
            self.dtype = _DT[views[0].dtype]
        nbytes = self.lib.ccab_ey_fit_workspace_bytes(len(self.dims), self._d, self.k, self.batch)
        if nbytes == 0:
            raise ValueError(f"ccab_ey_fit does not support widths {self.dims} with k = {self.k} (1 <= k <= "
                             f"{EY_MAX_K}, 2 to {_lib.MAX_VIEWS} views) and batch = {self.batch}")
        self.ws = _ws(nbytes, self.device)
        host = np.zeros(EY_HEADER + 2 * self.D * self.k)
        host[0] = np.inf
        host[EY_HEADER:EY_HEADER + self.D * self.k] = np.asarray(init, dtype=np.float64).T.reshape(-1)
        self.state = torch.from_numpy(host).to(self.device)
        self._flag = torch.empty(1, dtype=torch.float64, pin_memory=True)

    def run(self, n_steps: int, idx=None):
        c, lr, mom, tol = self.hyper
        with torch.cuda.device(self.device):
            rc = self.lib.ccab_ey_fit(len(self.dims), self._d, self.k, c, lr, mom, tol, int(n_steps),
                                      _ptr(self.cov), self.dtype, self._views, self._ld, self.batch, _ptr(idx),
                                      _ptr(self.state), _ptr(self.ws), self.ws.numel(),
                                      C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        _lib.check(rc, "ccab_ey_fit")

    def stopped(self) -> bool:
        self._flag.copy_(self.state[2:3])
        return bool(self._flag[0] != 0.0)

    def result(self):
        host = self.state.cpu().numpy()
        W = host[EY_HEADER:EY_HEADER + self.D * self.k].reshape(self.k, self.D).T.copy()
        return W, int(host[1])


def ey_fit(dims, init, c, learning_rate, momentum, tol, cov=None, views=None, batch=0) -> EyFit:
    """The device state of one Eckart-Young gradient fit (see ``EyFit``)."""
    return EyFit(dims, init, c, learning_rate, momentum, tol, cov=cov, views=views, batch=batch)


GFA_MAX_K = 64
GFA_HEADER = 16    # doubles of counters in front of the state block of ccab_gfa_fit
_GFA_SLOTS = 8     # per-view arrays of the state block have this many slots (_lib.MAX_VIEWS)
GFA_ARD_ALPHA_0 = GFA_ARD_BETA_0 = GFA_TAU_ALPHA_0 = GFA_TAU_BETA_0 = 1e-14   # CCAGFA::getDefaultOpts() priors
GFA_INIT_TAU = 1e3


def gfa_layout(K: int, D: int) -> dict:
    """Offsets (doubles) of the arrays in the state block of ccab_gfa_fit (include/ccab200.h), and its ``total``."""
    V, o, at = _GFA_SLOTS, {}, GFA_HEADER
    for name, size in (("y_const", V), ("a_ard", V), ("a_tau", V), ("tau", V), ("b_tau", V), ("alpha", V * K),
                       ("b_ard", V * K), ("cov_w", V * K * K), ("ww", V * K * K), ("cov_z", K * K), ("zz", K * K),
                       ("index", K), ("W", K * D), ("B0", K * D), ("B1", K * D), ("GB0", K * D), ("GB1", K * D)):
        o[name] = at
        at += size
    o["total"] = at
    return o


class GfaFit:
    """One GFA fit on the device (ccab_gfa_fit): the state block and the workspace, kept across chunked calls.

    ``G`` is the float64 D x D Gram matrix (CUDA), ``XtZ0`` the D x k float64 product X^T z0 (CUDA).  The host writes
    the initial state once: tau = 1e3, alpha_m = k d_m / max(datavar_m - 1e-3, 1e-8) from the (always centred) data
    variance of each view, zz = z0^T z0 + n I, and the constants y_const_m = tr G_mm.  ``run(n)`` enqueues one call of
    up to n iterations; ``stopped()`` reads the stop flag back (one small copy); ``result()`` copies the state block to
    the host once and returns it decoded (dictionary of numpy arrays at the active width k)."""

    def __init__(self, dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=True):
        import numpy as np

        self.lib = _lib.load()
        self.dims = [int(d) for d in dims]
        m, D = len(self.dims), int(sum(self.dims))
        self.D, self.k = D, int(XtZ0.shape[1])
        _require_cuda(G, "G")
        _require_cuda(XtZ0, "XtZ0")
        if G.dtype != torch.float64 or tuple(G.shape) != (D, D):
            raise ValueError(f"G must be the float64 {D} x {D} Gram matrix")
        if XtZ0.dtype != torch.float64 or tuple(XtZ0.shape) != (D, self.k):
            raise ValueError(f"XtZ0 must be a float64 {D} x k matrix")
        self.device = G.device
        self._d = _lib.i64_array(self.dims)
        nbytes = self.lib.ccab_gfa_fit_workspace_bytes(m, self._d, self.k)
        if nbytes == 0:
            raise ValueError(f"ccab_gfa_fit does not support widths {self.dims} with k = {self.k} (1 <= k <= "
                             f"{GFA_MAX_K}, 1 to {_lib.MAX_VIEWS} views)")
        self.G = G.contiguous()
        self.XtZ0 = XtZ0.T.contiguous()                   # k x D: column x of X^T z0 is row x
        self.n, self.tol, self.drop_k = float(n_samples), float(tol), bool(drop_k)
        self.ws = _ws(nbytes, self.device)
        K, o = self.k, gfa_layout(self.k, D)
        self.o = o
        h = np.zeros(o["total"])
        h[1] = K
        d = np.asarray(self.dims, dtype=np.float64)
        h[o["y_const"]:o["y_const"] + m] = y_const
        h[o["a_ard"]:o["a_ard"] + m] = GFA_ARD_ALPHA_0 + d / 2.0
        h[o["a_tau"]:o["a_tau"] + m] = GFA_TAU_ALPHA_0 + self.n * d / 2.0
        h[o["tau"]:o["tau"] + m] = GFA_INIT_TAU
        h[o["b_tau"]:o["b_tau"] + m] = GFA_TAU_BETA_0
        alpha = h[o["alpha"]:o["alpha"] + _GFA_SLOTS * K].reshape(_GFA_SLOTS, K)
        for i in range(m):
            alpha[i] = K * self.dims[i] / max(float(datavar[i]) - 1.0 / GFA_INIT_TAU, 1e-8)
        h[o["b_ard"]:o["b_ard"] + _GFA_SLOTS * K] = GFA_ARD_BETA_0
        h[o["cov_z"]:o["cov_z"] + K * K] = np.eye(K).reshape(-1)
        h[o["zz"]:o["zz"] + K * K] = (np.asarray(z0tz0, dtype=np.float64) + self.n * np.eye(K)).reshape(-1)
        h[o["index"]:o["index"] + K] = np.arange(K)
        self.state = torch.from_numpy(h).to(self.device)
        self._flag = torch.empty(1, dtype=torch.float64, pin_memory=True)

    def run(self, n_steps: int):
        with torch.cuda.device(self.device):
            rc = self.lib.ccab_gfa_fit(len(self.dims), self._d, self.k, _ptr(self.G), self.n, _ptr(self.XtZ0), self.tol,
                                       int(self.drop_k), int(n_steps), _ptr(self.state), _ptr(self.ws), self.ws.numel(),
                                       C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        _lib.check(rc, "ccab_gfa_fit")

    def stopped(self) -> bool:
        self._flag.copy_(self.state[3:4])
        return bool(self._flag[0] != 0.0)

    def result(self) -> dict:
        return decode_gfa_state(self.state.cpu().numpy(), self.dims, self.k)


def decode_gfa_state(h, dims, K: int) -> dict:
    """The state block of ccab_gfa_fit (host float64 array) as numpy arrays at the active width k: counters, tau,
    b_tau, alpha / b_ard (m x k), cov_w / ww (m x k x k), cov_z, zz, index, and W, B, GB, B_prev, GB_prev (D x k)."""
    import numpy as np

    m, D = len(dims), int(sum(dims))
    o = gfa_layout(K, D)
    k = int(h[1])
    cur = int(h[4])

    def kk(at, count=None):
        blk = h[at:at + (count or 1) * K * K].reshape(count or 1, K, K)[:, :k, :k].copy()
        return blk if count else blk[0]

    def kd(at):
        return h[at:at + K * D].reshape(K, D)[:k].T.copy()

    B, GB = (o["B0"], o["B1"]), (o["GB0"], o["GB1"])
    return dict(iters=int(h[0]), k=k, stable=int(h[2]), stop=bool(h[3]), rel=float(h[5]), prunes=int(h[6]),
                tau=h[o["tau"]:o["tau"] + m].copy(), b_tau=h[o["b_tau"]:o["b_tau"] + m].copy(),
                alpha=h[o["alpha"]:o["alpha"] + m * K].reshape(m, K)[:, :k].copy(),
                b_ard=h[o["b_ard"]:o["b_ard"] + m * K].reshape(m, K)[:, :k].copy(),
                cov_w=kk(o["cov_w"], m), ww=kk(o["ww"], m), cov_z=kk(o["cov_z"]), zz=kk(o["zz"]),
                index=h[o["index"]:o["index"] + k].astype(np.int64), W=kd(o["W"]), B=kd(B[cur]), GB=kd(GB[cur]),
                B_prev=kd(B[cur ^ 1]), GB_prev=kd(GB[cur ^ 1]))


def gfa_fit(dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=True) -> GfaFit:
    """The device state of one GFA fit (see ``GfaFit``)."""
    return GfaFit(dims, G, n_samples, XtZ0, z0tz0, datavar, y_const, tol, drop_k=drop_k)


TCCA_MAX_K = 64
TCCA_MAX_VIEWS = 8
TCCA_MAX_ENTRIES = 1 << 25     # prod of the view widths: M in float64 is 256 MB
TCCA_MAX_ITER = 100            # tensorly's n_iter_max
TCCA_HEADER = 8                # doubles in front of the rec history in the state block of ccab_tcca_fit


def tcca_moment(Z, nsplit: int = 0):
    """M = Z_1^T KR(Z_2, ..., Z_m) / n (p_1 x prod_{i>1} p_i float64, CUDA): the mode-0 unfolding of the cross-moment
    tensor of the float64 (n, p_i) CUDA tensors ``Z`` (ccab_tcca_moment).  ``nsplit`` > 0 forces that many sample
    splits; 0 lets the library choose from the shape."""
    lib = _lib.load()
    for i, z in enumerate(Z):
        _require_cuda(z, f"Z[{i}]")
    Z = [_row_major(z, False) for z in Z]
    if any(z.dtype != torch.float64 for z in Z):
        raise ValueError("tcca_moment takes float64 views")
    n = int(Z[0].shape[0])
    if any(int(z.shape[0]) != n for z in Z):
        raise ValueError("tcca_moment: the views differ in their number of rows")
    dims = [int(z.shape[1]) for z in Z]
    d = _lib.i64_array(dims)
    P = 1
    for p in dims[1:]:
        P *= p
    M = torch.empty((dims[0], P), dtype=torch.float64, device=Z[0].device)
    ws = _ws(lib.ccab_tcca_moment_workspace_bytes(len(dims), d, n, int(nsplit)), M.device)
    ptrs = (C.c_void_p * len(Z))(*[z.data_ptr() for z in Z])
    with torch.cuda.device(M.device):
        rc = lib.ccab_tcca_moment(len(dims), d, n, ptrs, _lib.i64_array([z.stride(0) for z in Z]), 1.0 / max(n, 1),
                                  int(nsplit), _ptr(M), _ptr(ws), ws.numel(), _stream(M))
    _lib.check(rc, "ccab_tcca_moment")
    return M


def tcca_layout(dims, k: int) -> dict:
    """Offsets (doubles) of the state block of ccab_tcca_fit: ``rec``, ``F`` (one per mode), ``G`` and ``total``."""
    at = TCCA_HEADER + TCCA_MAX_ITER
    F = []
    for p in dims:
        F.append(at)
        at += int(p) * k
    return {"rec": TCCA_HEADER, "F": F, "G": at, "total": at + len(dims) * k * k}


def tcca_fit(M, dims, k: int, n_iter: int, rand=None, state=None):
    """CP-ALS on the tensor M (float64 CUDA, prod(dims) entries in C order) with ccab_tcca_fit; returns the device
    state block.  Without ``state`` the fit starts: the leading eigenvectors of every unfolding Gram M_(j) M_(j)^T
    (one DMMA GEMM and one ``syevj`` per mode) and the host-drawn random columns ``rand`` (a list, one p_j x (k - p_j)
    array or None per mode) seed it.  With ``state`` the fit continues from it.  Up to ``n_iter`` iterations either
    way, nothing read back."""
    import numpy as np

    lib = _lib.load()
    _require_cuda(M, "M")
    dims = [int(p) for p in dims]
    m, d = len(dims), _lib.i64_array(dims)
    total = lib.ccab_tcca_state_size(m, d, int(k))
    if total < 0:
        raise ValueError(f"ccab_tcca_fit: {_lib.last_error()}")
    if M.dtype != torch.float64 or M.numel() != int(np.prod(dims)):
        raise ValueError(f"M must be a float64 tensor of {int(np.prod(dims))} entries")
    M = M.contiguous()
    dev = M.device
    ws = _ws(lib.ccab_tcca_fit_workspace_bytes(m, d, int(k)), dev)
    keep = []
    evecs, lam0, rnd = None, None, None
    if state is None:
        state = torch.empty(total, dtype=torch.float64, device=dev)
        T = M.reshape(dims)
        vecs = []
        for j in range(m):
            A = T.movedim(j, 0).reshape(dims[j], -1)
            lam, evt = syevj(gemm(A, A, transb=True))
            vecs.append(evt.contiguous())
            if j == 0:
                lam0 = lam
        keep += vecs
        evecs = (C.c_void_p * m)(*[v.data_ptr() for v in vecs])
        blocks = [np.asarray(r, dtype=np.float64).reshape(-1) for r in (rand or []) if r is not None]
        if blocks:
            rnd = torch.from_numpy(np.concatenate(blocks)).to(dev)
    elif state.dtype != torch.float64 or state.numel() != total or not state.is_cuda:
        raise ValueError(f"state must be a float64 CUDA tensor of {total} elements")
    with torch.cuda.device(dev):
        rc = lib.ccab_tcca_fit(m, d, int(k), _ptr(M), evecs, _ptr(lam0), _ptr(rnd), int(evecs is not None),
                               int(n_iter), _ptr(state), _ptr(ws), ws.numel(), _stream(M))
    _lib.check(rc, "ccab_tcca_fit")
    return state


def decode_tcca_state(h, dims, k: int) -> dict:
    """The state block of ccab_tcca_fit (host float64 array): iters, stop, singular, norm, rec (one per iteration
    done), F (p_j x k per mode) and G (their Grams)."""
    o = tcca_layout(dims, k)
    it = int(h[0])
    return dict(iters=it, stop=bool(h[1]), singular=bool(h[2]), norm=float(h[3]),
                rec=h[o["rec"]:o["rec"] + it].copy(),
                F=[h[f:f + int(p) * k].reshape(int(p), k).copy() for f, p in zip(o["F"], dims)],
                G=h[o["G"]:o["total"]].reshape(len(dims), k, k).copy())


def column_sums(view):
    """Column sums of an (n, d) CUDA tensor as one GEMM with a row of ones (float64 result)."""
    ones = torch.ones((1, view.shape[0]), dtype=view.dtype, device=view.device)
    return gemm(ones, view)[0].to(torch.float64)


_POW = {None: 0, 1: 0, -1: 1, -0.5: 2}


def scale(A, rows=None, rows_pow=1, cols=None, cols_pow=1, out=None):
    """out[i,j] = A[i,j] * rows[i]**rows_pow * cols[j]**cols_pow (pow in {1, -1, -0.5})."""
    lib = _lib.load()
    _require_cuda(A, "A")
    A = _row_major(A, False)
    if out is None:
        out = torch.empty_like(A)
    with torch.cuda.device(A.device):
        rc = lib.ccab_scale(_DT[A.dtype], A.shape[0], A.shape[1], _ptr(A), A.stride(0), _ptr(rows), _POW[rows_pow],
                            _ptr(cols), _POW[cols_pow], _ptr(out), out.stride(0), _stream(A))
    _lib.check(rc, "ccab_scale")
    return out


def center_columns_(A):
    """In place: subtract the column means."""
    lib = _lib.load()
    _require_cuda(A, "A")
    if A.stride(1) != 1:
        raise ValueError("row-major tensor expected")
    with torch.cuda.device(A.device):
        rc = lib.ccab_center_columns(_DT[A.dtype], A.shape[0], A.shape[1], _ptr(A), A.stride(0), _stream(A))
    _lib.check(rc, "ccab_center_columns")
    return A


def frobenius_norm(A):
    lib = _lib.load()
    _require_cuda(A, "A")
    A = _row_major(A, False)
    out = torch.empty(1, dtype=A.dtype, device=A.device)
    with torch.cuda.device(A.device):
        rc = lib.ccab_frobenius_norm(_DT[A.dtype], A.shape[0], A.shape[1], _ptr(A), A.stride(0), _ptr(out), _stream(A))
    _lib.check(rc, "ccab_frobenius_norm")
    return out


def pairwise_kernel(X, Y=None, metric: str = "linear", gamma: float = 1.0, degree: float = 1.0, coef0: float = 1.0):
    """K = k(X, Y) (float64, n_x x n_y, CUDA) for a metric name of sklearn's PAIRWISE_KERNEL_FUNCTIONS
    (ccab_pairwise_kernel).  X, Y: 2-D float32 / float64 CUDA tensors with unit column stride (any leading dimension)
    and one dtype; Y None means X (then, as in sklearn, the rbf distance is exactly 0 on the diagonal).  ``gamma`` is
    the resolved value (the caller applies sklearn's default 1 / n_features).  chi2 / additive_chi2 raise sklearn's
    ValueError on negative input, which costs one scalar read-back."""
    lib = _lib.load()
    if metric not in _lib.KERNEL_METRICS:
        raise ValueError(f"unknown kernel {metric!r}: supported are {sorted(_lib.KERNEL_METRICS)}")
    _require_cuda(X, "X")
    X = _row_major(X, False)
    Y = X if Y is None else _row_major(Y, False)
    _require_cuda(Y, "Y")
    if X.dtype != Y.dtype or X.dtype not in _DT or X.device != Y.device:
        raise ValueError(f"pairwise_kernel: X and Y must share one float dtype and device, got {X.dtype}@{X.device} "
                         f"and {Y.dtype}@{Y.device}")
    if X.shape[1] != Y.shape[1]:
        raise ValueError(f"Incompatible dimension for X and Y matrices: X.shape[1] == {X.shape[1]} while "
                         f"Y.shape[1] == {Y.shape[1]}")
    if metric in ("chi2", "additive_chi2"):
        neg = bool(((X < 0).any() | (Y < 0).any()).item())
        if neg:
            raise ValueError("X contains negative values." if bool((X < 0).any().item())
                             else "Y contains negative values.")
    met = _lib.KERNEL_METRICS[metric]
    nx, ny, d = int(X.shape[0]), int(Y.shape[0]), int(X.shape[1])
    K = torch.empty((nx, ny), dtype=torch.float64, device=X.device)
    ws = _ws(lib.ccab_pairwise_kernel_workspace_bytes(met, nx, ny), X.device)
    with torch.cuda.device(X.device):
        rc = lib.ccab_pairwise_kernel(met, _DT[X.dtype], _ptr(X), nx, X.stride(0), _ptr(Y), ny, Y.stride(0), d,
                                      float(gamma), float(degree), float(coef0), _ptr(K), ny, _ptr(ws), ws.numel(),
                                      _stream(X))
    _lib.check(rc, "ccab_pairwise_kernel")
    return K


KCCA_MAX_VIEWS = 8
KCCA_MAX_SAMPLES = 8192
KCCA_MAX_ORDER = 16384     # m * n: the whitened matrix T is at most 16384^2 float64 = 2 GB
