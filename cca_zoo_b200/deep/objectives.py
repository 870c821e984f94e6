"""Differentiable CCA objectives on the GPU (mirrors cca_zoo/deep/objectives.py:24-220).

``CCALoss.forward([z1, z2])`` returns ``-|| S11^-1/2 S12 S22^-1/2 ||_F^2`` with
``Sii = cov(zi) + eps I`` and eigenvalues clamped at ``eps`` exactly as the reference
(objectives.py:86-102, ``_inv_sqrtm`` :9-21).  Plug into ``DCCA(objective=...)``
(cca_zoo/deep/_dcca.py:61,73) unchanged: it is an ``nn.Module`` taking ``list[Tensor]`` and returning
a 0-dim tensor.

Forward  : ONE library call (``ccab_ccaloss_fwd``, csrc/fit.cu): moment pass over [z1 z2] -> S -> batched Cholesky +
           explicit inverse of S_11, S_22 -> P = S11^-1 S12 S22^-1 and the two small gradient matrices ->
           loss = -<P, S12> (the reference's third eigensolve, eigvalsh(T^T T).sum(), is a trace).  Nothing is read
           back on this path: the Cholesky status lands in a device flag that is checked LAZILY (at the next call, or
           by ``check()``).  Batches that are rank deficient by shape (n - 1 < width: the eigenvalue clamp of the
           reference is then active for certain) take the eigen route, which reproduces
           ``clamp(eigh(S + eps I), min=eps)`` literally with two Jacobi eigendecompositions.
Backward : analytic (SURVEY.md §3.4), no eigh-backward, ONE library call (``ccab_ccaloss_bwd``): with
           P = S11^-1 S12 S22^-1,  dL/dz1 = 2/(n-1) * center(z1 (P S21 S11^-1) - z2 P^T),  dL/dz2 symmetric.

Global batch (``global_batch=True`` under data parallelism, CCALoss / MCCALoss / GCCALoss): each rank's moment buffer
is summed over the ranks with ONE exchange (``parallel.allreduce_moments_lazy``, the step of the sharded fit), and the
loss stage runs on the global moments with the global count N read on the device (``ccab_ccaloss_fwd_moments``,
``ccab_covariance_ndev``).  The loss is the loss of the concatenated global batch, replicated on every rank; each rank's
backward is the exact derivative of that loss with respect to its own rows, centred by the saved global means, with no
collective (``ccab_ccaloss_bwd_global``, ``ccab_row_sub_scale``).  Every route decision is taken from exchanged data, so
all ranks take the same route and raise at the same call.  TCCALoss needs a second exchange: after the moments, the
local contraction of the whitened rows and, for 3 or more views, its marginals are summed with one all-reduce; its
backward then takes every global row sum from the global tensor and those marginals, again with no collective (see
``_TCCALossGlobalFn``).

bfloat16 / float16 representations (an encoder under ``torch.autocast``; all four losses) take the global-batch route
also in a single process, where nothing is exchanged and N is a device scalar holding n: the moment pass reads the
16-bit representations as they are (16-bit wgmma, or fp32 FMA for narrow batches), the loss stage runs in float32
and returns a float32 loss, and the backward runs the float32 global backward on float32 copies of the saved
representations made inside ``backward`` (TCCALoss: every stage after the moment pass in float64, on float64 copies
made inside ``forward``); the gradients come back in the representation's dtype.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops, parallel
from ..ops import HALF_DTYPES


def _require_cuda(name, *tensors):
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError(f"cca_zoo_b200.{name} needs CUDA tensors (sm_90a); there is no CPU fallback.")


def _row_major(z):
    z = z.detach()
    return z if (z.stride(1) == 1 and z.stride(0) >= z.shape[1]) else z.contiguous()


def _resolve_precision(precision, zs):
    """"auto": exact FMA moments for narrow batches (HBM / latency bound), the wgmma 3xTF32 kernel once the block
    covariance is wide enough to be a real contraction -- if TMA can address the representations."""
    if zs[0].dtype == torch.float64:
        return "exact"
    if precision == "auto":
        precision = "tf32x3b" if sum(z.shape[1] for z in zs) > 256 else "exact"
    if precision != "exact" and not all(z.data_ptr() % 16 == 0 and (z.stride(0) * z.element_size()) % 16 == 0
                                        for z in zs):
        return "exact"
    return precision


class _LazyStatus:
    """Device-side status flags of past evaluations, copied to pinned memory asynchronously and inspected without
    ever blocking the stream: ``poll`` looks at the copies that have already landed, ``check`` waits for all."""

    def __init__(self, what, nan_last=True):
        self.what = what
        self.nan_last = nan_last       # the last flag reports NaN / inf in the input
        self.pending = []
        self.free = []                 # recycled (pinned buffer, event) pairs: cudaHostAlloc costs ~0.1 ms

    def push(self, flags):
        if not flags.is_cuda:          # host-logic tests (tests/fake_ops.py): nothing is asynchronous there
            self._inspect(flags)
            return
        n = flags.numel()
        slot = next((i for i, (h, _) in enumerate(self.free) if h.numel() >= n), None)
        if slot is None:
            buf, ev = torch.empty(max(n, 16), dtype=flags.dtype, pin_memory=True), torch.cuda.Event()
        else:
            buf, ev = self.free.pop(slot)
        host = buf[:n]
        host.copy_(flags, non_blocking=True)
        ev.record(torch.cuda.current_stream(flags.device))
        self.pending.append((host, ev, buf))

    def _inspect(self, host):
        vals = host.tolist()
        if any(v != 0 for v in vals):
            self.pending.clear()
            if self.nan_last and vals[-1]:
                raise ValueError(f"{self.what}: a representation contained NaN or infinity.")
            raise RuntimeError(
                f"{self.what}: a within-view covariance S_ii + eps I of an earlier batch was not numerically positive "
                f"definite (Cholesky status {vals}); that loss value and its gradients are unreliable.  Use "
                f"verify='sync' to take the eigen route for such batches automatically, or a larger eps.")

    def poll(self):
        while self.pending and self.pending[0][1].query():
            host, ev, buf = self.pending.pop(0)
            self.free.append((buf, ev))
            self._inspect(host)

    def check(self):
        while self.pending:
            host, ev, buf = self.pending.pop(0)
            ev.synchronize()
            self.free.append((buf, ev))
            self._inspect(host)


def _eigen_route(z1d, z2d, eps, precision):
    """clamp(eigh(S + eps I), min=eps) literally (objectives.py:19-21): rank-deficient batches, verify='sync' fallback."""
    n, d1 = z1d.shape[0], z1d.shape[1]
    mom = ops.moments([z1d, z2d], precision=precision)
    C, _ = ops.covariance(mom, [d1, z2d.shape[1]], n, center=True, dtype=z1d.dtype)
    means = torch.cat([z1d.mean(dim=0), z2d.mean(dim=0)])     # the fused narrow backward centres algebraically
    return _eigen_stage(C, d1, eps, means)


def _eigen_stage(C, d1, eps, means):
    """The eigen route from the block covariance C of [z1 z2]: (loss, saved = G11 | P | G22 | means)."""
    S12 = C[:d1, d1:].contiguous()
    whiten = []
    for blk in (C[:d1, :d1], C[d1:, d1:]):
        lam, Vt = ops.syevj(blk.contiguous())
        Wt, _, _ = ops.whiten_rows(lam, Vt, 0.0, floor_add=eps, rank_tol=-1.0, lam_floor=0.0)
        whiten.append(Wt)
    W1t, W2t = whiten
    T = ops.gemm(ops.gemm(W1t, S12), W2t, transb=True)
    fro = ops.frobenius_norm(T)
    loss = -(fro * fro)
    S1inv = ops.gemm(W1t, W1t, transa=True)              # S11^-1 = W1 W1^T (W_i^T = Lam^-1/2 V^T)
    S2inv = ops.gemm(W2t, W2t, transa=True)
    P = ops.gemm(ops.gemm(S1inv, S12), S2inv)
    g11 = ops.gemm(ops.gemm(P, S12, transb=True), S1inv)
    g22 = ops.gemm(ops.gemm(S2inv, S12, transb=True), P)
    saved = torch.cat([g11.reshape(-1), P.reshape(-1), g22.reshape(-1), means])
    return loss, saved


def _is_global(global_batch, group):
    """Global-batch statistics apply only with more than one rank; otherwise the per-replica route runs unchanged."""
    return bool(global_batch) and parallel.is_distributed(group)


def _exchange(zd, precision, group, exchange=True):
    """The ONE collective of a global-batch forward: this rank's moment buffer summed over the ranks.  Returns
    (moments of the global batch, N as a 1-element float64 device tensor) -- nothing is read back.  ``exchange=False``
    (16-bit representations in a single process): the local moments, and n as that device scalar."""
    dims = [int(z.shape[1]) for z in zd]
    n_local = int(zd[0].shape[0])
    if n_local > 0:
        mom = ops.moments(zd, precision=precision)
    else:   # no rows here: contribute zeros (raising would leave the other ranks waiting in the exchange)
        mom = torch.zeros(ops.moments_size(dims), dtype=torch.float64, device=zd[0].device)
    if not exchange:
        return mom, torch.full((1,), float(n_local), dtype=torch.float64, device=mom.device)
    mom, _, n_dev = parallel.allreduce_moments_lazy(mom, n_local, group, dims)
    return mom, n_dev


def _compute_dtype(dt):
    """dtype of the loss stage and the backward: float32 for 16-bit representations."""
    return torch.float32 if dt in HALF_DTYPES else dt


def _widen(zs):
    """float32 copies of saved 16-bit representations (made inside ``backward``), the others as they are."""
    return [z.float() if z.dtype in HALF_DTYPES else z for z in zs]


def _global_count(n_dev, what):
    """N on the host (one read-back, taken only where the route depends on it)."""
    N = int(round(float(n_dev.reshape(-1)[0].item())))
    if N < 2:
        raise ValueError(f"{what}: a global batch needs at least 2 samples over all ranks, got N = {N}.")
    return N


def _check_finite(C, what):
    if not bool(torch.isfinite(C).all()):          # only on routes that read back anyway
        raise ValueError(f"{what}: a representation contained NaN or infinity.")


def _eigen_route_global(mom, n_dev, d1, d2, eps, dtype):
    """The eigen route from the global moments: (loss, saved = G11 | P | G22 | global means | N)."""
    _global_count(n_dev, "CCALoss")
    C, mean = ops.covariance(mom, [d1, d2], n_dev, center=True, dtype=dtype)
    _check_finite(C, "CCALoss")
    loss, saved = _eigen_stage(C, d1, eps, mean)
    return loss, torch.cat([saved, n_dev.to(dtype).reshape(1)])


_LOSS_DTYPES = (torch.float32, torch.float64, torch.bfloat16, torch.float16)


def _check_pair(z1, z2, name):
    _require_cuda(name, z1, z2)
    if z1.dtype != z2.dtype or z1.dtype not in _LOSS_DTYPES:
        raise ValueError("representations must share a float32/float64/bfloat16/float16 dtype")


class _CCALossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z1, z2, eps, precision, status, sync):
        _require_cuda("CCALoss", z1, z2)
        if z1.dtype != z2.dtype or z1.dtype not in (torch.float32, torch.float64):
            raise ValueError("representations must share a float32/float64 dtype")
        n = z1.shape[0]
        z1d, z2d = _row_major(z1), _row_major(z2)
        prec = _resolve_precision(precision, [z1d, z2d])
        if n - 1 < max(z1d.shape[1], z2d.shape[1]):          # rank deficient by shape: the clamp is active for certain
            loss, saved = _eigen_route(z1d, z2d, eps, prec)
        else:
            loss, saved, flags = ops.ccaloss_fwd(z1d, z2d, eps, prec)
            if sync:
                f = flags.tolist()                            # verify='sync': one read-back per step
                if f[2]:
                    raise ValueError("CCALoss: a representation contained NaN or infinity.")
                if f[0] or f[1]:
                    loss, saved = _eigen_route(z1d, z2d, eps, prec)
            else:
                status.push(flags)
        ctx.save_for_backward(z1d, z2d, saved)
        return loss.reshape(()).clone()

    @staticmethod
    def backward(ctx, grad_out):
        z1, z2, saved = ctx.saved_tensors
        go = grad_out.to(z1.dtype).reshape(1).contiguous()
        g1, g2 = ops.ccaloss_bwd(z1, z2, saved, go)
        return g1, g2, None, None, None, None


class _CCALossGlobalFn(torch.autograd.Function):
    """CCALoss of the global batch: this rank's rows, the moments of all ranks (see the module docstring).  With
    ``glob=False`` (16-bit representations in a single process) the same body without the exchange."""

    @staticmethod
    def forward(ctx, z1, z2, eps, precision, status, sync, group, glob=True):
        _check_pair(z1, z2, "CCALoss")
        n, d1, d2 = int(z1.shape[0]), int(z1.shape[1]), int(z2.shape[1])
        dt = _compute_dtype(z1.dtype)
        z1d, z2d = _row_major(z1), _row_major(z2)
        mom, n_dev = _exchange([z1d, z2d], _resolve_precision(precision, [z1d, z2d]), group, glob)
        width = max(d1, d2)
        # n - 1 >= width here implies N - 1 >= width: no read-back.  Only a narrower shard reads N, and N (exchanged)
        # decides for every rank alike.
        eigen = n - 1 < width and _global_count(n_dev, "CCALoss") - 1 < width
        if not eigen:
            loss, saved, flags = ops.ccaloss_fwd_moments(mom, n_dev, d1, d2, eps, dt)
            if sync:
                f = flags.tolist()                            # flags of the global moments: the same on every rank
                if f[2]:
                    raise ValueError("CCALoss: a representation contained NaN or infinity.")
                eigen = bool(f[0] or f[1])
            else:
                status.push(flags)
        if eigen:
            loss, saved = _eigen_route_global(mom, n_dev, d1, d2, eps, dt)
        ctx.save_for_backward(z1d, z2d, saved)
        return loss.reshape(()).clone()

    @staticmethod
    def backward(ctx, grad_out):
        z1, z2, saved = ctx.saved_tensors
        z1w, z2w = _widen([z1, z2])
        go = grad_out.to(z1w.dtype).reshape(1).contiguous()
        g1, g2 = ops.ccaloss_bwd_global(z1w, z2w, saved, go)
        return g1.to(z1.dtype), g2.to(z2.dtype), None, None, None, None, None, None


class CCALoss(nn.Module):
    r"""Andrew et al. (2013) deep-CCA loss for two views (cca_zoo/deep/objectives.py:24-102).

    Args:
        eps: ridge added to the within-view covariances and eigenvalue floor (default 1e-5).
        precision: arithmetic of the covariance kernel for float32 inputs: ``"auto"`` (default: exact CUDA-core FMA
            for narrow representations, wgmma 3xTF32 beyond a total width of 256), ``"exact"``, ``"tf32x3"``, ``"tf32"``.
        verify: ``"lazy"`` (default) never reads anything back in ``forward``: the Cholesky status of every
            evaluation is copied to the host asynchronously and inspected at the next call / by ``check()``, which
            raise if an earlier batch had a numerically indefinite covariance.  ``"sync"`` reads the status back in
            every call and takes the eigen route (the reference's ``clamp(eigh(.))`` literally) for such batches.
        global_batch: under data parallelism (an initialised process group of more than one rank), compute the loss
            of the concatenated global batch instead of each replica's own: the block moments are summed over the
            ranks with one exchange per forward, every rank gets the same loss, and each rank's backward (no
            collective) is the exact derivative of that loss with respect to its own rows.  A rank may hold 0 rows.
            DDP averages parameter gradients over the W ranks, so they come out as (1/W) dL_global/dθ.  Without a
            process group, or with one rank, the per-replica route runs unchanged.  Default False (the reference's
            per-replica statistics).
        process_group: the ranks whose batches form the global batch (``None``: the default group, as in
            ``torch.nn.SyncBatchNorm``).

    Representations may be float32, float64, bfloat16 or float16 (both of one dtype).  16-bit representations are
    read by the moment pass as they are; the loss (float32) and the float32 backward follow the global-batch route
    (see the module docstring), and the gradients have the representations' dtype.
    """

    def __init__(self, eps: float = 1e-5, precision: str = "auto", verify: str = "lazy", global_batch: bool = False,
                 process_group=None) -> None:
        super().__init__()
        if verify not in ("lazy", "sync"):
            raise ValueError("verify must be 'lazy' or 'sync'")
        self.eps = eps
        self.precision = precision
        self.verify = verify
        self.global_batch = global_batch
        self.process_group = process_group
        self._status = _LazyStatus("CCALoss")

    def check(self) -> None:
        """Wait for the status of every evaluation issued so far and raise if one of them was unreliable."""
        self._status.check()

    def forward(self, representations: list[torch.Tensor]) -> torch.Tensor:
        if len(representations) != 2:
            raise ValueError(
                "CCALoss expects exactly 2 representations, "
                f"got {len(representations)}."
            )
        self._status.poll()
        z1, z2 = representations
        glob = _is_global(self.global_batch, self.process_group)
        if glob or z1.dtype in HALF_DTYPES:
            return _CCALossGlobalFn.apply(z1, z2, float(self.eps), self.precision, self._status, self.verify == "sync",
                                          self.process_group, glob)
        return _CCALossFn.apply(z1, z2, float(self.eps), self.precision, self._status, self.verify == "sync")


def _mcca_cholesky_inverses(C, off, dims, eps):
    """A_i = (C_ii + eps I)^-1 by batched Cholesky + inverse; returns (A, Cholesky status tensors)."""
    m = len(dims)
    A, flags = [], []
    if len(set(dims)) == 1:                                  # one batched factorisation for all views
        R = torch.stack([C[off[i]:off[i + 1], off[i]:off[i + 1]] for i in range(m)])
        R.diagonal(dim1=1, dim2=2).add_(eps)
        Linv, info = ops.potrf_inv_(R, pivot_tol=0.25 * eps)
        flags.append(info)
        Ab = ops.gemm_batched(Linv, Linv, transa=True)
        A = [Ab[i] for i in range(m)]
    else:
        for i in range(m):
            R = C[off[i]:off[i + 1], off[i]:off[i + 1]].contiguous()
            R.diagonal().add_(eps)
            Linv, info = ops.potrf_inv_(R, pivot_tol=0.25 * eps)
            flags.append(info)
            A.append(ops.gemm(Linv, Linv, transa=True))
    return A, flags


def _mcca_eigen_inverses(C, off, dims, eps):
    """A_i = clamp(eigh(C_ii + eps I), min=eps)^-1 = W_i^T W_i, the inverse each pair's eigen route uses; returns the
    A_i and the whitening rows W_i."""
    A, W = [], []
    for i in range(len(dims)):
        lam, Vt = ops.syevj(C[off[i]:off[i + 1], off[i]:off[i + 1]].contiguous())
        Wt, _, _ = ops.whiten_rows(lam, Vt, 0.0, floor_add=eps, rank_tol=-1.0, lam_floor=0.0)
        A.append(ops.gemm(Wt, Wt, transa=True))
        W.append(Wt)
    return A, W


def _mcca_pairs(C, off, dims, A, W=None):
    """P_ij = A_i S_ij A_j, G_i = sum_j P_ij S_ji A_i and the loss terms <P_ij, S_ij> over the pairs i < j.  With the
    whitening rows W of the eigen route the terms are ||W_i S_ij W_j^T||_F^2 instead, as in CCALoss's eigen route: the
    same value, without the cancellation of the trace form when a clamped eigenvalue makes A_i huge."""
    m, dt = len(dims), C.dtype
    G = [torch.zeros((d, d), dtype=dt, device=C.device) for d in dims]
    P = {}
    terms = []
    for i in range(m):
        for j in range(i + 1, m):
            Sij = C[off[i]:off[i + 1], off[j]:off[j + 1]]
            Q = ops.gemm(A[i], Sij)                          # A_i S_ij
            Q2 = ops.gemm(Sij, A[j])                         # S_ij A_j
            Pij = ops.gemm(Q, A[j])
            ops.gemm(Pij, Q, transb=True, beta=1.0, out=G[i])            # += P_ij S_ji A_i
            ops.gemm(Q2, Pij, transa=True, beta=1.0, out=G[j])           # += A_j S_ji P_ij
            P[(i, j)] = Pij
            if W is None:
                terms.append((Pij * Sij).sum())
            else:
                f = ops.frobenius_norm(ops.gemm(ops.gemm(W[i], Sij), W[j], transb=True))
                terms.append((f * f).reshape(()))
    return G, P, terms


def _mcca_products(xs, G, P, alpha):
    """x_i G_i - sum_{j != i} x_j P_ji for every view (alpha times), x_i = z_i rows or a mean row."""
    m = len(xs)
    out = []
    for i in range(m):
        g = ops.gemm(xs[i], G[i], alpha=alpha)
        for j in range(m):
            if j == i:
                continue
            if i < j:
                ops.gemm(xs[j], P[(i, j)], transb=True, alpha=-alpha, beta=1.0, out=g)   # - x_j P_ij^T
            else:
                ops.gemm(xs[j], P[(j, i)], alpha=-alpha, beta=1.0, out=g)                # - x_j P_ji
        out.append(g)
    return out


class _MCCALossFn(torch.autograd.Function):
    """Sum of the pairwise CCA losses from ONE moment pass over all views, every S_ii factored ONCE
    (the reference calls CCALoss per pair, objectives.py:148-153: m - 1 eigendecompositions of every S_ii and m - 1
    passes over every z_i).  With A_i = S_ii^-1 (batched Cholesky + inverse), P_ij = A_i S_ij A_j:
        loss = - sum_{i<j} <P_ij, S_ij>,
        dL/dz_i = 2/(n-1) center( z_i G_i - sum_{j != i} z_j P_ji ),   G_i = sum_{j != i} P_ij S_ji A_i,  P_ji = P_ij^T.
    """

    @staticmethod
    def forward(ctx, eps, precision, status, *zs):
        _require_cuda("MCCALoss", *zs)
        dt = zs[0].dtype
        if dt not in (torch.float32, torch.float64) or any(z.dtype != dt for z in zs):
            raise ValueError("representations must share a float32/float64 dtype")
        n, m = zs[0].shape[0], len(zs)
        zd = [_row_major(z) for z in zs]
        dims = [int(z.shape[1]) for z in zd]
        off = [0]
        for d in dims:
            off.append(off[-1] + d)
        mom = ops.moments(zd, precision=_resolve_precision(precision, zd))
        C, _ = ops.covariance(mom, dims, n, center=True, dtype=dt)
        A, flags = _mcca_cholesky_inverses(C, off, dims, eps)
        G, P, terms = _mcca_pairs(C, off, dims, A)
        status.push(torch.cat(flags))
        ctx.n, ctx.m = n, m
        ctx.pairs = sorted(P)
        ctx.save_for_backward(*zd, *G, *[P[k] for k in ctx.pairs])
        return -torch.stack(terms).sum()

    @staticmethod
    def backward(ctx, grad_out):
        m, n = ctx.m, ctx.n
        t = ctx.saved_tensors
        zs, G = t[:m], t[m:2 * m]
        P = dict(zip(ctx.pairs, t[2 * m:]))
        a = 2.0 / (n - 1)
        go = grad_out.to(zs[0].dtype)
        grads = []
        for i in range(m):
            g = ops.gemm(zs[i], G[i], alpha=a)
            for j in range(m):
                if j == i:
                    continue
                if i < j:
                    ops.gemm(zs[j], P[(i, j)], transb=True, alpha=-a, beta=1.0, out=g)   # - z_j P_ij^T
                else:
                    ops.gemm(zs[j], P[(j, i)], alpha=-a, beta=1.0, out=g)                # - z_j P_ji
            ops.center_columns_(g)
            grads.append(g * go)
        return (None, None, None, *grads)


class _MCCALossGlobalFn(torch.autograd.Function):
    """MCCALoss of the global batch: one exchange, the pairs from the global C; backward with the global means.  With
    ``glob=False`` (16-bit representations in a single process) the same body without the exchange."""

    @staticmethod
    def forward(ctx, eps, precision, status, sync, group, glob, *zs):
        _require_cuda("MCCALoss", *zs)
        if zs[0].dtype not in _LOSS_DTYPES or any(z.dtype != zs[0].dtype for z in zs):
            raise ValueError("representations must share a float32/float64/bfloat16/float16 dtype")
        dt = _compute_dtype(zs[0].dtype)
        n, m = int(zs[0].shape[0]), len(zs)
        zd = [_row_major(z) for z in zs]
        dims = [int(z.shape[1]) for z in zd]
        off = [0]
        for d in dims:
            off.append(off[-1] + d)
        mom, n_dev = _exchange(zd, _resolve_precision(precision, zd), group, glob)
        C, mean = ops.covariance(mom, dims, n_dev, center=True, dtype=dt)
        eigen = n - 1 < max(dims) and _global_count(n_dev, "MCCALoss") - 1 < max(dims)
        W = None                                   # whitening rows, on the eigen route only
        if not eigen:
            A, flags = _mcca_cholesky_inverses(C, off, dims, eps)
            flags = torch.cat(flags + [(~torch.isfinite(C).all()).to(torch.int32).reshape(1)])
            if sync:
                f = flags.tolist()                 # from the global C: the same on every rank
                if f[-1]:
                    raise ValueError("MCCALoss: a representation contained NaN or infinity.")
                eigen = any(f[:-1])
            else:
                status.push(flags)
        if eigen:                                  # every pair through the eigen route, from the same global C
            _global_count(n_dev, "MCCALoss")
            _check_finite(C, "MCCALoss")
            A, W = _mcca_eigen_inverses(C, off, dims, eps)
        G, P, terms = _mcca_pairs(C, off, dims, A, W)
        ctx.m = m
        ctx.pairs = sorted(P)
        ctx.save_for_backward(mean, n_dev, *zd, *G, *[P[k] for k in ctx.pairs])
        return -torch.stack(terms).sum()

    @staticmethod
    def backward(ctx, grad_out):
        m = ctx.m
        mean, n_dev, *t = ctx.saved_tensors
        in_dt = [z.dtype for z in t[:m]]
        zs, G = _widen(t[:m]), t[m:2 * m]
        P = dict(zip(ctx.pairs, t[2 * m:]))
        dt = zs[0].dtype
        # dL/dz_i = 2/(N-1) (z_i G_i - sum_j z_j P_ji - 1 r_i^T) go, r_i the same product of the global mean rows
        s = (2.0 / (n_dev - 1.0)).to(dt) * grad_out.to(dt).reshape(1)
        mus, o = [], 0
        for z in zs:
            mus.append(mean[o:o + z.shape[1]].reshape(1, -1))
            o += z.shape[1]
        if zs[0].shape[0] == 0:
            return (None, None, None, None, None, None, *[torch.zeros_like(z, dtype=d) for z, d in zip(zs, in_dt)])
        rows = _mcca_products(mus, G, P, 1.0)
        grads = _mcca_products(list(zs), G, P, 1.0)
        for g, r in zip(grads, rows):
            ops.row_sub_scale_(g, r.reshape(-1), s)
        return (None, None, None, None, None, None, *[g.to(d) for g, d in zip(grads, in_dt)])


class MCCALoss(nn.Module):
    r"""Sum of pairwise CCA losses over all view pairs (cca_zoo/deep/objectives.py:105-153), computed from one
    moment pass with every within-view covariance factored once.  Same ``verify`` semantics as ``CCALoss``
    (``"lazy"``: status checked at the next call; ``"sync"``: per-pair ``CCALoss`` evaluations with the eigen-route
    fallback, i.e. the reference's loop).

    ``global_batch`` / ``process_group`` as in ``CCALoss`` (2 to 8 views): one exchange per forward, and all pairs come
    from the global block covariance.  There ``verify="sync"`` reads the replicated status and, if some S_ii failed,
    evaluates every pair through the eigen route from the same global covariance (no per-pair exchanges).
    bfloat16 / float16 representations (2 to 8, one dtype) take that route in a single process too, without the
    exchange (see the module docstring)."""

    def __init__(self, eps: float = 1e-5, precision: str = "auto", verify: str = "lazy", global_batch: bool = False,
                 process_group=None) -> None:
        super().__init__()
        if verify not in ("lazy", "sync"):
            raise ValueError("verify must be 'lazy' or 'sync'")
        self.eps = eps
        self.precision = precision
        self.verify = verify
        self.global_batch = global_batch
        self.process_group = process_group
        self._status = _LazyStatus("MCCALoss", nan_last=False)
        self._global_status = _LazyStatus("MCCALoss")
        self._cca_loss = CCALoss(eps=eps, precision=precision, verify="sync")

    def check(self) -> None:
        self._status.check()
        self._global_status.check()

    def forward(self, representations: list[torch.Tensor]) -> torch.Tensor:
        n_views = len(representations)
        glob = _is_global(self.global_batch, self.process_group)
        if glob or (n_views and representations[0].dtype in HALF_DTYPES):
            if not 2 <= n_views <= 8:
                what = "with global_batch=True" if glob else "with 16-bit representations"
                raise ValueError(f"MCCALoss {what} takes 2 to 8 representations, got {n_views}.")
            self._global_status.poll()
            return _MCCALossGlobalFn.apply(float(self.eps), self.precision, self._global_status, self.verify == "sync",
                                           self.process_group, glob, *representations)
        n = representations[0].shape[0]
        lazy_ok = (self.verify == "lazy" and 2 <= n_views <= 8
                   and n - 1 >= max(int(z.shape[1]) for z in representations))
        if lazy_ok:
            self._status.poll()
            return _MCCALossFn.apply(float(self.eps), self.precision, self._status, *representations)
        total = torch.zeros((), device=representations[0].device, dtype=representations[0].dtype)
        for i in range(n_views):
            for j in range(i + 1, n_views):
                total = total + self._cca_loss([representations[i], representations[j]])
        return total


class _GCCALossFn(torch.autograd.Function):
    """MAX-VAR GCCA objective in its primal form (SURVEY.md §8f rank 2).

    The reference (objectives.py:196-220) builds the n x n matrix M = sum_i H_i H_i^T, H_i = Zc_i S_i^-1/2, and
    sums its top-k eigenvalues: O(n^2) memory, O(n^3) work per step.  With H = [H_1 .. H_m] (n x D) the non-zero
    spectrum of M = H H^T equals that of K = H^T H = (n-1) Wt C Wt^T (D x D), Wt = blkdiag(Wt_i) with
    Wt_i = diag(clamp(lam_i + eps, min=eps)^-1/2) V_i^T -- all of it a function of the block covariance C that
    one K1 pass provides.  Backward is analytic (Hellmann-Feynman on the eigenvalue sum, no eigh-backward):
        Q = Wt^T U_k Lam_k^-1/2,  A = (n-1) C Q,  B = blkdiag(S_i^-1) A,
        dL/dz_i = center( -2 (Z Q) B_i^T + 2/(n-1) z_i B_i B_i^T ).
    """

    @staticmethod
    def forward(ctx, eps, precision, glob, group, *zs):
        _require_cuda("GCCALoss", *zs)
        if zs[0].dtype not in _LOSS_DTYPES or any(z.dtype != zs[0].dtype for z in zs):
            raise ValueError("representations must share a float32/float64/bfloat16/float16 dtype")
        dt = _compute_dtype(zs[0].dtype)
        # 16-bit representations take the global-batch body in a single process too, without the exchange
        route_global = glob or zs[0].dtype in HALF_DTYPES
        n = zs[0].shape[0]
        dims = [int(z.shape[1]) for z in zs]
        D, k = sum(dims), dims[0]
        zd = [z.detach() for z in zs]
        mean = None
        if route_global:
            # global batch: one exchange; N is read back (the Jacobi sweeps below read back anyway) and replaces n
            mom, n_dev = _exchange(zd, precision, group, glob)
            C, mean = ops.covariance(mom, dims, n_dev, center=True, dtype=dt)
            n = _global_count(n_dev, "GCCALoss")
            _check_finite(C, "GCCALoss")
        else:
            mom = ops.moments(zd, precision=precision)
            C, _ = ops.covariance(mom, dims, n, center=True, dtype=dt)
        Wt = torch.zeros((D, D), dtype=dt, device=C.device)
        off = 0
        for d in dims:
            lam, Vt = ops.syevj(C[off:off + d, off:off + d].contiguous())
            Wi, _, _ = ops.whiten_rows(lam, Vt, 0.0, floor_add=eps, rank_tol=-1.0, lam_floor=0.0)
            Wt[off:off + d, off:off + d] = Wi
            off += d
        K = ops.gemm(ops.gemm(Wt, C), Wt, transb=True, alpha=float(n - 1))
        K = 0.5 * (K + K.T)
        evals, Ut = ops.syevj(K)                              # descending; rows of Ut are eigenvectors
        lam_k = evals[:k].contiguous()
        ctx.n, ctx.dims, ctx.glob = n, dims, route_global
        ctx.save_for_backward(C, Wt, lam_k, Ut[:k].contiguous(), mean, *zd)
        return -lam_k.sum()

    @staticmethod
    def backward(ctx, grad_out):
        C, Wt, lam_k, Ut_k, mean, *zs = ctx.saved_tensors
        n, dims = ctx.n, ctx.dims
        k = lam_k.shape[0]
        safe = lam_k.clamp_min(torch.finfo(lam_k.dtype).tiny * 1e8)
        Qt = ops.scale(Ut_k, rows=safe, rows_pow=-0.5)                    # k x D : Lam^-1/2 U_k^T
        Q = ops.gemm(Wt, Qt, transa=True, transb=True)                    # D x k
        A = ops.gemm(C, Q, alpha=float(n - 1))                            # D x k
        B = ops.gemm(Wt, ops.gemm(Wt, A), transa=True)                    # blkdiag(S_i^-1) A
        if ctx.glob:
            grads = _gcca_global_grads(_widen(zs), dims, Q, B, mean, n, grad_out)
            return (None, None, None, None, *[g.to(z.dtype) for g, z in zip(grads, zs)])
        Y = torch.zeros((n, k), dtype=C.dtype, device=C.device)
        off = 0
        for z, d in zip(zs, dims):
            ops.gemm(z, Q[off:off + d], beta=1.0, out=Y)
            off += d
        go = grad_out.to(C.dtype)
        grads, off = [], 0
        for z, d in zip(zs, dims):
            Bi = B[off:off + d]
            g = ops.gemm(Y, Bi, transb=True, alpha=-2.0)
            ops.gemm(z, ops.gemm(Bi, Bi, transb=True), alpha=2.0 / (n - 1), beta=1.0, out=g)
            ops.center_columns_(g)
            grads.append(g * go)
            off += d
        return (None, None, None, None, *grads)


def _gcca_global_grads(zs, dims, Q, B, mean, N, grad_out):
    """This shard's rows of the global GCCA gradient: the local products, centred by the same products of the global
    mean row, times grad_out -- no collective."""
    dt = Q.dtype

    def products(xs):
        Y = torch.zeros((xs[0].shape[0], Q.shape[1]), dtype=dt, device=Q.device)
        off = 0
        for x, d in zip(xs, dims):
            ops.gemm(x, Q[off:off + d], beta=1.0, out=Y)
            off += d
        out, off = [], 0
        for x, d in zip(xs, dims):
            Bi = B[off:off + d]
            g = ops.gemm(Y, Bi, transb=True, alpha=-2.0)
            ops.gemm(x, ops.gemm(Bi, Bi, transb=True), alpha=2.0 / (N - 1), beta=1.0, out=g)
            out.append(g)
            off += d
        return out

    mus, off = [], 0
    for d in dims:
        mus.append(mean[off:off + d].reshape(1, d))
        off += d
    if zs[0].shape[0] == 0:
        return [torch.zeros_like(z) for z in zs]
    rows = products(mus)
    go = grad_out.to(dt).reshape(1)
    grads = products(list(zs))
    for g, r in zip(grads, rows):
        ops.row_sub_scale_(g, r.reshape(-1), go)
    return grads


class GCCALoss(nn.Module):
    r"""Generalised (MAX-VAR) CCA loss for two or more views (cca_zoo/deep/objectives.py:156-220):
    :math:`-\sum_{d \le k} \lambda_d(\sum_i H_i H_i^\top)` with ``k`` the width of the first representation.
    Same constructor and ``forward(list[Tensor]) -> 0-dim Tensor`` as the reference, so it plugs into
    ``DCCA(objective=...)`` and is what ``DGCCA`` uses (cca_zoo/deep/_dgcca.py:70).  At most 8 views.
    ``global_batch`` / ``process_group`` as in ``CCALoss``: one exchange per forward, and the eigenproblem of the
    global block covariance (its Jacobi sweeps read back, as the per-replica route's do, and so does N).
    bfloat16 / float16 representations take that route in a single process too, without the exchange (see the module
    docstring)."""

    def __init__(self, eps: float = 1e-5, precision: str = "exact", global_batch: bool = False,
                 process_group=None) -> None:
        super().__init__()
        self.eps = eps
        self.precision = precision
        self.global_batch = global_batch
        self.process_group = process_group

    def forward(self, representations: list[torch.Tensor]) -> torch.Tensor:
        prec = _resolve_precision(self.precision, [_row_major(z) for z in representations])
        glob = _is_global(self.global_batch, self.process_group)
        return _GCCALossFn.apply(float(self.eps), prec, glob, self.process_group if glob else None, *representations)


def _tcca_divided_differences(lam, eps):
    """F_ab = (f(l_a) - f(l_b)) / (l_a - l_b), F_aa = f'(l_a) for f(l) = max(l, eps)^-1/2 (f' = 0 where the clamp is
    active); where both eigenvalues are unclamped the closed form -1 / (s_a s_b (s_a + s_b)), s = sqrt(l), which has
    no cancellation and is the finite limit at a repeated eigenvalue."""
    s = lam.clamp_min(eps).sqrt()
    f = 1.0 / s
    la, lb = lam[:, None], lam[None, :]
    d = la - lb
    mixed = torch.where(d != 0, (f[:, None] - f[None, :]) / torch.where(d != 0, d, torch.ones_like(d)),
                        torch.zeros_like(d))
    both = (la > eps) & (lb > eps)
    return torch.where(both, -1.0 / (s[:, None] * s[None, :] * (s[:, None] + s[None, :])), mixed)


def _tcca_eigen_whiten(C, z64, off, dims, eps):
    """clamp(eigh(S_i), min=eps) whitening, S_i = C_ii + eps I, literally: H_i = Zc_i W_i, W_i = V f(Lam) V^T.
    Returns the H_i and, per view, what the backward needs: (Zc_i, W_i, V^T, F)."""
    H, parts = [], []
    for i, d in enumerate(dims):
        lam, Vt = ops.syevj(C[off[i]:off[i + 1], off[i]:off[i + 1]].clone())
        Wt, _, _ = ops.whiten_rows(lam, Vt, 0.0, floor_add=eps, rank_tol=-1.0, lam_floor=0.0)
        W = ops.gemm(Vt, Wt, transa=True)
        Zc = ops.center_columns_(z64[i].clone())
        H.append(ops.gemm(Zc, W))
        parts.append((Zc, W, Vt, _tcca_divided_differences(lam + eps, eps)))
    return H, parts


def _tcca_cholesky_factors(C, off, dims, eps):
    """L_i^-1 with S_i = C_ii + eps I = L_i L_i^T (batched when the widths agree); C stays intact for the eigen route.
    Returns the factors and their Cholesky status tensors."""
    m = len(dims)
    if len(set(dims)) == 1:                        # one batched factorisation for all views
        S = torch.stack([C[off[i]:off[i + 1], off[i]:off[i + 1]] for i in range(m)])
        S.diagonal(dim1=1, dim2=2).add_(eps)
        L, info = ops.potrf_inv_(S, pivot_tol=0.25 * eps)
        return [L[i] for i in range(m)], [info]
    Linv, flags = [], []
    for i in range(m):
        S = C[off[i]:off[i + 1], off[i]:off[i + 1]].clone()
        S.diagonal().add_(eps)
        L, info = ops.potrf_inv_(S, pivot_tol=0.25 * eps)
        Linv.append(L)
        flags.append(info)
    return Linv, flags


class _TCCALossFn(torch.autograd.Function):
    """-||M||_F, M = (1/n) sum_s H_1[s] x ... x H_m[s], in float64 for every input dtype (see TCCALoss)."""

    @staticmethod
    def forward(ctx, eps, precision, status, sync, *zs):
        dt = zs[0].dtype
        n, m = int(zs[0].shape[0]), len(zs)
        zd = [_row_major(z) for z in zs]
        dims = [int(z.shape[1]) for z in zd]
        off = [0]
        for d in dims:
            off.append(off[-1] + d)
        mom = ops.moments(zd, precision=_resolve_precision(precision, zd))
        C, _ = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
        z64 = [z if z.dtype == torch.float64 else z.to(torch.float64) for z in zd]
        eigen = n - 1 < max(dims)                      # rank deficient by shape: the clamp is active for certain
        if eigen and not bool(torch.isfinite(C).all()):       # the eigen route reads back anyway
            raise ValueError("TCCALoss: a representation contained NaN or infinity.")
        if not eigen:
            Linv, flags = _tcca_cholesky_factors(C, off, dims, eps)
            flags.append((~torch.isfinite(C).all()).to(torch.int32).reshape(1))
            flags = torch.cat(flags)
            # H_i = Zc_i R_i with R_i = L_i^-T: centring commutes with the right factor
            H = [ops.center_columns_(ops.gemm(z, L, transb=True)) for z, L in zip(z64, Linv)]
            if sync:
                f = flags.tolist()                     # verify='sync': one read-back per step
                if f[-1]:
                    raise ValueError("TCCALoss: a representation contained NaN or infinity.")
                eigen = any(f[:-1])
            else:
                status.push(flags)
        if eigen:
            if dt != torch.float64:    # the clamp at eps is decided on the eigenvalues: float64 moments for those
                C, _ = ops.covariance(ops.moments(z64), dims, n, center=True, dtype=torch.float64)
            H, parts = _tcca_eigen_whiten(C, z64, off, dims, eps)
        M = ops.tcca_moment(H)
        norm = ops.frobenius_norm(M)
        ctx.n, ctx.m, ctx.dt, ctx.eigen = n, m, dt, eigen
        saved = [M, norm, *H]
        if eigen:
            for p in parts:
                saved += list(p)
        else:
            saved += Linv
        ctx.save_for_backward(*saved)
        return (-norm).reshape(()).to(dt).clone()

    @staticmethod
    def backward(ctx, grad_out):
        n, m = ctx.n, ctx.m
        t = ctx.saved_tensors
        M, norm, H = t[0], t[1], t[2:2 + m]
        rest = t[2 + m:]
        go = grad_out.to(torch.float64).reshape(1)
        # Gamma_i = dL/dH_i = -Y_i / (n ||M||) * grad_out; 0 at ||M|| = 0 (torch's subgradient of the norm)
        coef = torch.where(norm > 0, -go / (n * norm), torch.zeros_like(norm))
        gam = ops.tcca_moment_adjoint(M, list(H), scale_dev=coef)
        grads = []
        for i in range(m):
            g = gam[i]
            if ctx.eigen:
                Zc, W, Vt, F = rest[4 * i:4 * i + 4]
                B = ops.gemm(Zc, g, transa=True)
                B = 0.5 * (B + B.T)
                X = ops.gemm(Vt, F * ops.gemm(ops.gemm(Vt, B), Vt, transb=True), transa=True)
                X = ops.gemm(X, Vt)
                out = ops.gemm(g, W)
                ops.gemm(Zc, X, alpha=2.0 / (n - 1), beta=1.0, out=out)
                ops.center_columns_(out)
            else:
                # (Gamma_i - H_i (H_i^T Gamma_i) / (n - 1)) R_i^T, centred; R_i^T = L_i^-1
                T = ops.gemm(H[i], g, transa=True)
                ops.gemm(H[i], T, alpha=-1.0 / (n - 1), beta=1.0, out=g)
                ops.center_columns_(g)
                out = ops.gemm(g, rest[i])
            grads.append(out.to(ctx.dt))
        return (None, None, None, None, *grads)


def _unfolding_products(M, dims, i, pbar=None):
    """(M_(i) M_(i)^T, M_(i) vec(pbar) or None) for the mode-i unfolding M_(i) (k_i x prod_{j != i} k_j, the other
    modes in C order, as ``tcca_moment`` orders the marginal pbar).  Both are one two-view contraction over the
    prod_{j != i} k_j positions on ``tcca_moment``, whose sample splits spread that long reduction over the GPU (a GEMM
    with a k_i x k_i output would run it in one CTA): X^T [X | vec(pbar)] with X = M_(i)^T, one copy of M."""
    k, Q = dims[i], M.numel() // dims[i]
    Y = torch.empty((Q, k if pbar is None else k + 1), dtype=M.dtype, device=M.device)
    Y[:, :k] = M.reshape(dims).movedim(i, -1).reshape(Q, k)
    if pbar is not None:
        Y[:, k] = pbar.reshape(-1)
    G = ops.tcca_moment([Y[:, :k], Y], scale=1.0)
    return G[:, :k], (G[:, k] if pbar is not None else None)


def _tcca_sizes(dims):
    """Entries of M and of the marginals P_i = sum_s (x)_{j != i} H_j[s] (sent for m >= 3 only: for m = 2, P_i is the
    column sum of a view centred with the global mean, which is 0)."""
    P = 1
    for d in dims:
        P *= d
    return P, ([P // d for d in dims] if len(dims) >= 3 else [])


class _TCCALossGlobalFn(torch.autograd.Function):
    """TCCALoss of the global batch: this rank's rows, the moments and the cross-moment tensor of all ranks (see the
    module docstring).  With ``exchange=False`` (16-bit representations in a single process) the same body without the
    exchanges, N a device scalar holding n.

    Forward: exchange 1 (moments) gives the global C and means mu_i; the whitening (Cholesky R_i = L_i^-T, or the
    eigen route W_i) and H_i = (z_i - mu_i) R_i are replicated / local; exchange 2 sums [sum_s (x)_i H_i[s] | P_i] over
    the ranks, scaled by 1/N on the device to [M | Pbar_i].  Backward, with Gamma_i = coef Y_i, coef = -g / (N ||M||)
    and Y_i the adjoint of the global M against the local H_j, every global row sum follows from M and Pbar_i:
        T_i = sum H_i^T Gamma_i = coef N M_(i) M_(i)^T,   (1/N) sum Gamma_i = r_i = coef M_(i) vec(Pbar_i),
        Cholesky: dL/dz_i = (Gamma_i - H_i T_i / (N - 1) - 1 r_i^T) R_i^T,
        eigen:    dL/dz_i = Gamma_i W_i + 2/(N - 1) Zc_i X_i - 1 r_i^T W_i,  X_i from B_i = W_i^-1 T_i,
    so the backward issues no collective."""

    @staticmethod
    def forward(ctx, eps, precision, status, sync, group, exchange, *zs):
        in_dt = zs[0].dtype
        n, m = int(zs[0].shape[0]), len(zs)
        zd = [_row_major(z) for z in zs]
        dims = [int(z.shape[1]) for z in zd]
        off = [0]
        for d in dims:
            off.append(off[-1] + d)
        dev = zd[0].device
        mom, n_dev = _exchange(zd, _resolve_precision(precision, zd), group, exchange)
        C, mean = ops.covariance(mom, dims, n_dev, center=True, dtype=torch.float64)
        width = max(dims)
        # n - 1 >= width here implies N - 1 >= width: no read-back.  Only a narrower shard reads N, and N (exchanged)
        # decides for every rank alike.
        eigen = n - 1 < width and _global_count(n_dev, "TCCALoss") - 1 < width
        if not eigen:
            Linv, flags = _tcca_cholesky_factors(C, off, dims, eps)
            flags = torch.cat(flags + [(~torch.isfinite(C).all()).to(torch.int32).reshape(1)])
            if sync:
                f = flags.tolist()                     # flags of the global C: the same on every rank
                if f[-1]:
                    raise ValueError("TCCALoss: a representation contained NaN or infinity.")
                eigen = any(f[:-1])
            else:
                status.push(flags)
        z64 = [z.to(torch.float64, copy=True) for z in zd]
        one = torch.ones(1, dtype=torch.float64, device=dev)
        if eigen:
            _global_count(n_dev, "TCCALoss")
            _check_finite(C, "TCCALoss")
            if not exchange and in_dt != torch.float64:
                # the clamp at eps is decided on the eigenvalues: float64 moments of the float64 copies, as the
                # per-replica route takes them (with an exchange, the exchanged moments are all there is)
                C, mean = ops.covariance(ops.moments(z64), dims, n, center=True, dtype=torch.float64)
        H, saved = [], []
        for i, d in enumerate(dims):
            Zc = z64[i]
            if n:
                ops.row_sub_scale_(Zc, mean[off[i]:off[i + 1]], one)       # centred with the global mean
            if eigen:
                lam, Vt = ops.syevj(C[off[i]:off[i + 1], off[i]:off[i + 1]].clone())
                Wt, g, _ = ops.whiten_rows(lam, Vt, 0.0, floor_add=eps, rank_tol=-1.0, lam_floor=0.0)
                W = ops.gemm(Vt, Wt, transa=True)
                Winv = ops.gemm(Vt, ops.scale(Vt, rows=g, rows_pow=-1), transa=True)    # V clamp(Lam, eps)^1/2 V^T
                H.append(ops.gemm(Zc, W) if n else Zc)
                saved += [Zc, W, Vt, _tcca_divided_differences(lam + eps, eps), Winv]
            else:
                H.append(ops.gemm(Zc, Linv[i], transb=True) if n else Zc)        # R_i = L_i^-T
                saved.append(Linv[i])
        P, marg = _tcca_sizes(dims)
        buf = (torch.empty if n else torch.zeros)(P + sum(marg), dtype=torch.float64, device=dev)
        if n:                                          # no rows here: zeros, and no kernel on an empty batch
            ops.tcca_moment(H, scale=1.0, out=buf[:P])
            o = P
            for i, q in enumerate(marg):
                ops.tcca_moment([H[j] for j in range(m) if j != i], scale=1.0, out=buf[o:o + q])
                o += q
        if exchange:
            parallel.allreduce_sum_(buf, group)
        row = buf.view(1, -1)
        ops.scale(row, rows=n_dev, rows_pow=-1, out=row)                  # [M | Pbar_i]: sums over all ranks / N
        norm = ops.frobenius_norm(buf[:P].view(dims[0], -1))
        ctx.m, ctx.dims, ctx.in_dt, ctx.eigen = m, dims, in_dt, eigen
        ctx.save_for_backward(buf, norm, n_dev, *H, *saved)
        return (-norm).reshape(()).to(_compute_dtype(in_dt)).clone()

    @staticmethod
    def backward(ctx, grad_out):
        m, dims, in_dt = ctx.m, ctx.dims, ctx.in_dt
        buf, norm, n_dev, *t = ctx.saved_tensors
        H, rest = t[:m], t[m:]
        head = (None,) * 6
        if H[0].shape[0] == 0:
            return (*head, *[torch.zeros((0, d), dtype=in_dt, device=buf.device) for d in dims])
        P, marg = _tcca_sizes(dims)
        M = buf[:P]
        go = grad_out.to(torch.float64).reshape(1)
        cN = torch.where(norm > 0, -go / norm, torch.zeros_like(norm))   # coef N; 0 at ||M|| = 0
        coef = cN / n_dev
        one = torch.ones(1, dtype=torch.float64, device=buf.device)
        gam = ops.tcca_moment_adjoint(M, list(H), scale_dev=coef)
        grads, o = [], P
        for i in range(m):
            G, r = _unfolding_products(M, dims, i, buf[o:o + marg[i]] if marg else None)
            if r is not None:                                               # r_i = coef M_(i) vec(Pbar_i)
                r = r * coef
                o += marg[i]
            g = gam[i]
            if ctx.eigen:
                Zc, W, Vt, F, Winv = rest[5 * i:5 * i + 5]
                B = ops.gemm(Winv, G) * cN                                  # sum over all rows of Zc_i^T Gamma_i
                B = 0.5 * (B + B.T)
                X = ops.gemm(Vt, F * ops.gemm(ops.gemm(Vt, B), Vt, transb=True), transa=True)
                X = ops.gemm(X, Vt) * (2.0 / (n_dev - 1.0))
                out = ops.gemm(g, W)
                ops.gemm(Zc, X, beta=1.0, out=out)
                if r is not None:
                    ops.row_sub_scale_(out, ops.gemm(r.reshape(1, -1), W).reshape(-1), one)
            else:
                ops.gemm(H[i], G * (cN / (n_dev - 1.0)), alpha=-1.0, beta=1.0, out=g)
                if r is not None:
                    ops.row_sub_scale_(g, r, one)
                out = ops.gemm(g, rest[i])                                  # R_i^T = L_i^-1
            grads.append(out.to(in_dt))
        return (*head, *grads)


class TCCALoss(nn.Module):
    r"""Deep tensor-CCA loss for 2 to 8 views (cca_zoo/deep/objectives.py:223-289): :math:`-\|M\|_F` with
    :math:`M = \frac1n \sum_s H_1[s] \otimes \cdots \otimes H_m[s]` the cross-moment tensor of the whitened
    representations :math:`H_i = \tilde Z_i\,\mathrm{clamp}(S_i)^{-1/2}`, :math:`S_i = \mathrm{cov}(z_i) + \epsilon I`.
    Views may have different widths; the product of the widths is at most 2^25.  Plugs into ``DTCCA``, which sets
    its objective in its constructor: assign ``model.objective = TCCALoss(eps=model.eps)`` afterwards.

    The reference materialises the n x k_1 x ... x k_m outer-product array and keeps it for autograd.  Here M is
    contracted on the fp64 tensor pipe without that array (``ccab_tcca_moment``), and the backward is analytic: one
    launch of the Khatri-Rao adjoint (``ccab_tcca_moment_adjoint``) gives every dL/dH_i, then a few k_i x k_i
    products per view.  ||M||_F does not change under an orthogonal change of basis in any mode, so the whitening is
    a Cholesky factor of S_i, which equals the reference whenever its eigenvalue clamp is inactive; batches that are
    rank deficient by shape (n - 1 < k_i) take the eigen route, the reference's ``clamp(eigh(S_i), min=eps)``
    literally.  All of it runs in float64, also for float32 representations (the moment pass then follows
    ``precision``); the loss and the gradients come back in the input dtype.  Where some S_i has a repeated
    eigenvalue (a constant representation: S_i = eps I) the reference's eigh backward returns NaN; the gradient here
    is the finite limit.  ||M||_F = 0 gives a zero gradient.

    Args:
        eps: ridge added to the within-view covariances and eigenvalue floor (default 1e-5).
        precision: arithmetic of the moment pass for float32 inputs, as in ``CCALoss``.
        verify: ``"lazy"`` (default) reads nothing back: the Cholesky status and a NaN flag are inspected at the next
            call or by ``check()``.  ``"sync"`` reads them back in every call, raises ``ValueError`` on NaN or
            infinity and takes the eigen route for a batch whose S_i is not numerically positive definite.
        global_batch: under data parallelism (an initialised process group of more than one rank), compute the loss
            of the concatenated global batch instead of each replica's own: the block moments are summed over the
            ranks, then the local contraction of the whitened rows (and, for 3 or more views, its marginals), so a
            forward runs two exchanges; every rank gets the same loss, and each rank's backward (no collective) is
            the exact derivative of that loss with respect to its own rows.  A rank may hold 0 rows.  DDP averages
            parameter gradients over the W ranks, so they come out as (1/W) dL_global/dθ.  Without a process group,
            or with one rank, the per-replica route runs unchanged.  Default False (the reference's per-replica
            statistics).
        process_group: the ranks whose batches form the global batch (``None``: the default group, as in
            ``torch.nn.SyncBatchNorm``).

    Representations may be float32, float64, bfloat16 or float16 (all of one dtype).  16-bit representations are read
    by the moment pass as they are and take the global-batch route (without an exchange in a single process);
    everything after the moment pass runs in float64, the loss is float32 and the gradients have the representations'
    dtype.
    """

    def __init__(self, eps: float = 1e-5, precision: str = "auto", verify: str = "lazy", global_batch: bool = False,
                 process_group=None) -> None:
        super().__init__()
        if verify not in ("lazy", "sync"):
            raise ValueError("verify must be 'lazy' or 'sync'")
        self.eps = eps
        self.precision = precision
        self.verify = verify
        self.global_batch = global_batch
        self.process_group = process_group
        self._status = _LazyStatus("TCCALoss")

    def check(self) -> None:
        """Wait for the status of every evaluation issued so far and raise if one of them was unreliable."""
        self._status.check()

    def forward(self, representations: list[torch.Tensor]) -> torch.Tensor:
        zs = list(representations)
        if not 2 <= len(zs) <= ops.TCCA_MAX_VIEWS:
            raise ValueError(f"TCCALoss takes 2 to {ops.TCCA_MAX_VIEWS} representations, got {len(zs)}.")
        _require_cuda("TCCALoss", *zs)
        dt = zs[0].dtype
        if dt not in _LOSS_DTYPES or any(z.dtype != dt for z in zs):
            raise ValueError("representations must share a float32/float64/bfloat16/float16 dtype")
        if any(z.dim() != 2 for z in zs) or any(z.shape[0] != zs[0].shape[0] for z in zs):
            raise ValueError("representations must be 2-D with the same number of rows")
        # every argument error is raised here, before any exchange; a global batch checks N >= 2 from exchanged data
        glob = _is_global(self.global_batch, self.process_group)
        n = int(zs[0].shape[0])
        if n < 2 and not glob:
            raise ValueError(f"TCCALoss needs at least 2 samples for a covariance, got n = {n}.")
        entries = 1
        for z in zs:
            if z.shape[1] < 1:
                raise ValueError("every representation needs at least one column")
            entries *= int(z.shape[1])
        if entries > ops.TCCA_MAX_ENTRIES:
            raise ValueError(f"the cross-moment tensor of widths {[int(z.shape[1]) for z in zs]} has {entries} entries; "
                             f"TCCALoss supports at most 2^25 = {ops.TCCA_MAX_ENTRIES} (the product of the widths).")
        self._status.poll()
        if glob or dt in HALF_DTYPES:
            return _TCCALossGlobalFn.apply(float(self.eps), self.precision, self._status, self.verify == "sync",
                                           self.process_group, glob, *zs)
        return _TCCALossFn.apply(float(self.eps), self.precision, self._status, self.verify == "sync", *zs)
