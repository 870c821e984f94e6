"""TEST INFRASTRUCTURE ONLY: a torch-CPU stand-in for ``cca_zoo_b200.ops`` (same functions, same contracts, LAPACK /
torch arithmetic instead of the CUDA kernels) so that the HOST-SIDE logic -- solver routes and their fall-backs,
the covariance-space algebra of PartialCCA / GRCCA, the sharded fit with its all-reduce -- can be exercised by the
``-m "not gpu"`` suite.  Nothing in the package imports this module; ``install(monkeypatch)`` swaps it in for one
test.  The product keeps failing loudly without a CUDA device (tests/test_abi_cpu.py checks that).

Contracts mirrored (see cca_zoo_b200/ops.py and include/ccab200.h): the padded moment buffer ``[Dp*Dp + Dp]`` with
every view padded to 128-column blocks, eigenvalues descending with eigenvectors as ROWS, ``gesvj`` taking the
transposed matrix, in-place ``potrf_inv_`` / ``center_columns_`` and the Cholesky status flags (1-based index of the
first pivot <= pivot_tol).
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch

BLK = 128


def _layout(dims):
    pads = [(int(d) + BLK - 1) // BLK * BLK for d in dims]
    poff = np.concatenate([[0], np.cumsum(pads)]).astype(int)
    return poff, int(poff[-1])


def moments(views, precision="tf32x3"):
    if not (1 <= len(views) <= 8):
        raise ValueError(f"between 1 and 8 views are supported, got {len(views)}")
    dims = [int(v.shape[1]) for v in views]
    poff, Dp = _layout(dims)
    X = torch.zeros((views[0].shape[0], Dp), dtype=torch.float64)
    for v, o in zip(views, poff):
        X[:, o:o + v.shape[1]] = v.to(torch.float64)
    return torch.cat([(X.T @ X).reshape(-1), X.sum(dim=0)])


SHIFT_RATIO = {torch.float32: 16.0, torch.float64: 1e8}


def column_pilot(views):
    return [v[:4096].mean(dim=0) for v in views], 0.0


def moments_safe(views, precision="tf32x3b", x0=None):
    return moments(views, precision), None          # float64 LAPACK arithmetic: no cancellation to guard against


def covariance(mom, dims, n_total, center=True, dtype=torch.float64):
    poff, Dp = _layout(dims)
    if mom.numel() != Dp * Dp + Dp:
        raise ValueError("moments buffer has the wrong size")
    if not n_total >= 2:
        raise ValueError("at least 2 samples are needed for a covariance")
    M = mom[:Dp * Dp].reshape(Dp, Dp)
    s = mom[Dp * Dp:]
    keep = np.concatenate([np.arange(o, o + d) for o, d in zip(poff, dims)])
    M, s = M[keep][:, keep], s[keep]
    if center:
        M = M - torch.outer(s, s) / n_total
    mean = s / n_total if center else torch.zeros_like(s)
    return (M / (n_total - 1)).to(dtype).contiguous(), mean.to(dtype)


def syevj(A, shift=0.0, return_info=False):
    squeeze = A.dim() == 2
    Ab = A.unsqueeze(0) if squeeze else A
    w, V = torch.linalg.eigh(0.5 * (Ab + Ab.transpose(-1, -2)).to(torch.float64))
    w, V = w.flip(-1), V.flip(-1)
    evals, evt = w.to(A.dtype), V.transpose(-1, -2).contiguous().to(A.dtype)
    if squeeze:
        evals, evt = evals[0], evt[0]
    if return_info:
        return evals, evt, {"sweeps": 0, "offdiag": 0.0}
    return evals, evt


def gesvj(Gt, return_info=False):
    G = Gt.T.to(torch.float64)                      # m x n
    m, n = G.shape
    U, S, Vh = torch.linalg.svd(G, full_matrices=False)
    r = S.shape[0]
    sigma = torch.zeros(n, dtype=torch.float64)
    right = torch.zeros((n, n), dtype=torch.float64)
    left = torch.zeros((n, m), dtype=torch.float64)
    sigma[:r], right[:r], left[:r] = S, Vh, U.T
    out = (sigma.to(Gt.dtype), right.to(Gt.dtype), left.to(Gt.dtype))
    return out + ({"sweeps": 0, "offdiag": 0.0},) if return_info else out


def gemm(A, B, transa=False, transb=False, alpha=1.0, beta=0.0, out=None):
    a = A.T if transa else A
    b = B.T if transb else B
    if a.shape[1] != b.shape[0]:
        raise ValueError(f"gemm inner dimensions differ: {a.shape[1]} vs {b.shape[0]}")
    res = alpha * (a @ b)
    if out is None:
        return res.contiguous()
    if tuple(out.shape) != tuple(res.shape) or out.stride(1) != 1:
        raise ValueError("gemm `out` has the wrong layout")
    out.copy_(res + beta * out if beta != 0.0 else res)
    return out


def whiten_rows(lam, Vt, c, floor_add=0.0, floor_dev=None, scale=1.0, rank_tol=0.0, max_rank=None, lam_floor=-1e300):
    d = Vt.shape[0]
    lam64 = lam.to(torch.float64)
    l0 = max(float(lam64[0]), 0.0)
    fl = floor_add + (float(floor_dev[0]) if floor_dev is not None else 0.0)
    keep = (lam64 > rank_tol * l0) & (torch.arange(d) < (d if max_rank is None else max_rank))
    g = torch.where(keep, 1.0 / torch.sqrt(((1.0 - c) * lam64.clamp_min(lam_floor) + c + fl) * scale),
                    torch.zeros_like(lam64))
    Wt = (g[:, None] * Vt.to(torch.float64)).to(Vt.dtype)
    return Wt, g.to(Vt.dtype), keep.sum().to(torch.int32).reshape(1)


def scale(A, rows=None, rows_pow=1, cols=None, cols_pow=1, out=None):
    res = A.clone()
    if rows is not None:
        res = res * (rows.to(A.dtype) ** rows_pow)[:, None]
    if cols is not None:
        res = res * (cols.to(A.dtype) ** cols_pow)[None, :]
    if out is not None:
        out.copy_(res)
        return out
    return res


def center_columns_(A):
    A.sub_(A.mean(dim=0, keepdim=True))
    return A


def frobenius_norm(A):
    return torch.linalg.norm(A.to(torch.float64)).to(A.dtype).reshape(1)


def ccaloss_small(Cm, d1, d2, eps):
    C64 = Cm.to(torch.float64)
    S11 = C64[:d1, :d1] + eps * torch.eye(d1, dtype=torch.float64)
    S22 = C64[d1:, d1:] + eps * torch.eye(d2, dtype=torch.float64)
    S12 = C64[:d1, d1:]
    i11, i22 = torch.linalg.inv(S11), torch.linalg.inv(S22)
    P = i11 @ S12 @ i22
    loss = -(S12 * P).sum()                       # -tr(S11^-1 S12 S22^-1 S21)
    G11 = P @ S12.T @ i11
    G22 = i22 @ S12.T @ P
    minp = torch.minimum(torch.linalg.eigvalsh(S11)[0], torch.linalg.eigvalsh(S22)[0])
    dt = Cm.dtype
    return loss.reshape(1).to(dt), G11.to(dt), P.to(dt), G22.to(dt), minp.reshape(1).to(dt)


def potrf_inv_(A, pivot_tol=0.0):
    squeeze = A.dim() == 2
    Ab = A.unsqueeze(0) if squeeze else A
    n = Ab.shape[-1]
    idx = torch.tril_indices(n, n)
    infos, invs = [], []
    for a in Ab:
        sym = torch.tril(a) + torch.tril(a, -1).T
        L, info = torch.linalg.cholesky_ex(sym.to(torch.float64))
        flag = int(info.item())
        if flag == 0 and pivot_tol > 0.0:
            small = (L.diagonal() ** 2 <= pivot_tol).nonzero()
            flag = int(small[0].item()) + 1 if small.numel() else 0
        infos.append(flag)
        if flag == 0:
            a[idx[0], idx[1]] = L[idx[0], idx[1]].to(A.dtype)
            invs.append(torch.linalg.inv(torch.tril(a).to(torch.float64)).to(A.dtype))
        else:
            invs.append(torch.zeros_like(a))
    Linv = torch.stack(invs)
    return (Linv[0] if squeeze else Linv), torch.tensor(infos, dtype=torch.int32)


def gemm_batched(A, B, transa=False, transb=False, alpha=1.0):
    return torch.stack([gemm(A[i], B[i], transa=transa, transb=transb, alpha=alpha) for i in range(A.shape[0])])


def ccaloss_fwd(z1, z2, eps, precision="exact"):
    n, d1, d2 = z1.shape[0], z1.shape[1], z2.shape[1]
    dt = z1.dtype
    mom = moments([z1, z2])
    flags = torch.zeros(3, dtype=torch.int32)
    if not bool(torch.isfinite(mom).all()):
        flags[2] = 1
    C, _ = covariance(mom, [d1, d2], n, True, torch.float64)
    S11 = C[:d1, :d1] + eps * torch.eye(d1, dtype=torch.float64)
    S22 = C[d1:, d1:] + eps * torch.eye(d2, dtype=torch.float64)
    S12 = C[:d1, d1:]
    for i, S in enumerate((S11, S22)):
        L, info = torch.linalg.cholesky_ex(S)
        if int(info) != 0 or bool((L.diagonal() ** 2 <= 0.25 * eps).any()):
            flags[i] = 1
    A1, A2 = torch.linalg.inv(S11), torch.linalg.inv(S22)
    P = A1 @ S12 @ A2
    G11 = P @ S12.T @ A1
    G22 = A2 @ S12.T @ P
    loss = -(P * S12).sum()
    means = torch.cat([z1.to(torch.float64).mean(dim=0), z2.to(torch.float64).mean(dim=0)])
    saved = torch.cat([G11.reshape(-1), P.reshape(-1), G22.reshape(-1), means]).to(dt)
    return loss.reshape(1).to(dt), saved, flags


def ccaloss_bwd(z1, z2, saved, grad_out):
    n, d1, d2 = z1.shape[0], z1.shape[1], z2.shape[1]
    s64 = saved.to(torch.float64)
    G11 = s64[:d1 * d1].reshape(d1, d1)
    P = s64[d1 * d1:d1 * d1 + d1 * d2].reshape(d1, d2)
    G22 = s64[d1 * d1 + d1 * d2:d1 * d1 + d1 * d2 + d2 * d2].reshape(d2, d2)
    a = 2.0 / (n - 1)
    x1, x2 = z1.to(torch.float64), z2.to(torch.float64)
    g1 = a * (x1 @ G11 - x2 @ P.T)
    g2 = a * (x2 @ G22 - x1 @ P)
    go = float(grad_out.reshape(-1)[0]) if grad_out is not None else 1.0
    g1 = (g1 - g1.mean(dim=0, keepdim=True)) * go
    g2 = (g2 - g2.mean(dim=0, keepdim=True)) * go
    return g1.to(z1.dtype), g2.to(z1.dtype)


# ---- device-side fit (csrc/fit.cu) stand-in: same result-block layout and status bits, LAPACK arithmetic ----
FIT_NOT_POSITIVE_DEFINITE, FIT_NOT_CONVERGED, FIT_NON_FINITE, FIT_TOO_FEW_SAMPLES = 1, 2, 4, 8
FIT_HEADER_DOUBLES = 32


def _al256(x):
    return (x + 255) // 256 * 256


def rcca_fit(mom, dims, n_host, n_dev, center, c, k, p, iters, dtype):
    from cca_zoo_b200.ops import decode_fit_block  # noqa: F401  (layout documented there)

    item = 4 if dtype == torch.float32 else 8
    D = int(sum(dims))
    o_mean = 8 * FIT_HEADER_DOUBLES
    o_sig = o_mean + _al256(8 * D)
    o_w1 = o_sig + _al256(item * k)
    o_w2 = o_w1 + _al256(item * dims[0] * k)
    total = o_w2 + _al256(item * dims[1] * k)
    offsets = [o_mean, o_sig, o_w1, o_w2, total]
    block = torch.zeros(total, dtype=torch.uint8)
    buf = block.numpy()
    hdr = buf[:8 * FIT_HEADER_DOUBLES].view(np.float64)
    n = float(n_host) if n_host is not None else float(n_dev[0])
    status = 0
    if not bool(torch.isfinite(mom).all()):
        status |= FIT_NON_FINITE
    if not n > max(dims):
        status |= FIT_TOO_FEW_SAMPLES
    hdr[1] = n
    if status == 0:
        C, mean = covariance(mom, dims, n, center, torch.float64)
        d1 = dims[0]
        Linv = []
        for i, sl in enumerate((slice(0, d1), slice(d1, D))):
            R = (1.0 - c[i]) * C[sl, sl] + c[i] * torch.eye(dims[i], dtype=torch.float64)
            L, info = torch.linalg.cholesky_ex(R)
            tol = dims[i] * float(torch.finfo(dtype).eps) * ((1.0 - c[i]) * float(C[sl, sl].diagonal().max()) + c[i])
            if int(info) != 0 or bool((L.diagonal() ** 2 <= tol).any()):
                status |= FIT_NOT_POSITIVE_DEFINITE
                break
            Linv.append(torch.linalg.inv(L))
        if status == 0:
            T = Linv[0] @ C[:d1, d1:] @ Linv[1].T
            U, S, Vh = torch.linalg.svd(T, full_matrices=False)
            np_dt = np.float32 if dtype == torch.float32 else np.float64
            buf[o_mean:o_mean + 8 * D].view(np.float64)[:] = mean.numpy()
            buf[o_sig:o_sig + item * k].view(np_dt)[:] = S[:k].numpy()
            buf[o_w1:o_w1 + item * dims[0] * k].view(np_dt)[:] = (Linv[0].T @ U[:, :k]).numpy().reshape(-1)
            buf[o_w2:o_w2 + item * dims[1] * k].view(np_dt)[:] = (Linv[1].T @ Vh[:k].T).numpy().reshape(-1)
            hdr[3] = float(S[0])
    hdr[0] = status
    return block, offsets


def mcca_fit(mom, dims, n_host, n_dev, center, c, eps, k, p, iters, dtype):
    item = 4 if dtype == torch.float32 else 8
    m, D = len(dims), int(sum(dims))
    offsets = [8 * FIT_HEADER_DOUBLES]
    offsets.append(offsets[-1] + _al256(8 * D))
    offsets.append(offsets[-1] + _al256(item * k))
    for d in dims:
        offsets.append(offsets[-1] + _al256(item * d * k))
    block = torch.zeros(offsets[-1], dtype=torch.uint8)
    buf = block.numpy()
    hdr = buf[:8 * FIT_HEADER_DOUBLES].view(np.float64)
    n = float(n_host) if n_host is not None else float(n_dev[0])
    status = 0
    if not bool(torch.isfinite(mom).all()):
        status |= FIT_NON_FINITE
    if not n > max(dims):
        status |= FIT_TOO_FEW_SAMPLES
    hdr[1] = n
    if status == 0:
        C, mean = covariance(mom, dims, n, center, torch.float64)
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        Linv = []
        for i in range(m):
            sl = slice(off[i], off[i + 1])
            R = (1.0 - c[i]) * C[sl, sl] + c[i] * torch.eye(dims[i], dtype=torch.float64)
            L, info = torch.linalg.cholesky_ex(R)
            tol = max(eps, dims[i] * float(torch.finfo(dtype).eps) * ((1.0 - c[i]) * float(C[sl, sl].diagonal().max()) + c[i]))
            if int(info) != 0 or bool((L.diagonal() ** 2 <= tol).any()):
                status |= FIT_NOT_POSITIVE_DEFINITE
                break
            Linv.append(torch.linalg.inv(L))
        if status == 0:
            K = torch.zeros((D, D), dtype=torch.float64)
            for i in range(m):
                for j in range(m):
                    if i != j:
                        K[off[i]:off[i + 1], off[j]:off[j + 1]] = Linv[i] @ C[off[i]:off[i + 1], off[j]:off[j + 1]] @ Linv[j].T
            w, V = torch.linalg.eigh(K)
            w, V = w.flip(0)[:k], V.flip(1)[:, :k]
            np_dt = np.float32 if dtype == torch.float32 else np.float64
            buf[offsets[0]:offsets[0] + 8 * D].view(np.float64)[:] = mean.numpy()
            buf[offsets[1]:offsets[1] + item * k].view(np_dt)[:] = w.numpy()
            for i in range(m):
                wi = (m ** 0.5) * Linv[i].T @ V[off[i]:off[i + 1]]
                buf[offsets[2 + i]:offsets[2 + i] + item * dims[i] * k].view(np_dt)[:] = wi.numpy().reshape(-1)
            hdr[3] = float(w[0])
    hdr[0] = status
    return block, offsets


def decode_fit_block(host, offsets, dims, k, dtype):
    from cca_zoo_b200.ops import decode_fit_block as real

    return real(host, offsets, dims, k, dtype)


@contextlib.contextmanager
def _no_streams(device):
    yield [None, None]


def install(monkeypatch):
    """Route the host logic of the package through this module for the duration of one test."""
    import sys

    import cca_zoo_b200
    from cca_zoo_b200 import _base, _solvers
    from cca_zoo_b200.linear import _grcca, _mcca, _partialcca, _rcca

    from cca_zoo_b200.deep import objectives

    me = sys.modules[__name__]
    for mod in (_base, _solvers, _partialcca, _grcca, _rcca, _mcca, objectives):
        monkeypatch.setattr(mod, "ops", me)
    monkeypatch.setattr(objectives, "_require_cuda", lambda name, *tensors: None)
    monkeypatch.setattr(cca_zoo_b200, "ops", me, raising=False)
    monkeypatch.setattr(_solvers, "_two_streams", _no_streams)
    monkeypatch.setattr(_base.BaseModel, "_device", lambda self: torch.device("cpu"))
