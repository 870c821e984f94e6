"""Base class of the H100 estimators: the reference's sklearn surface (cca_zoo/_base.py:19-258) with
the fit-time arithmetic moved to the GPU.

Drop-in contract kept from the reference:
  * ``__init__`` only stores keyword arguments (sklearn ``clone`` / ``get_params`` work);
  * ``fit(views, y=None) -> self`` sets ``weights_`` (list of ``(d_i, k)`` numpy arrays),
    ``means_``, ``n_views_``, ``n_features_in_``, ``n_samples_`` (_base.py:94-101);
  * ``transform / fit_transform / score / pairwise_correlations / average_pairwise_correlations /
    get_factor_loadings / weights`` behave as in the reference (numpy in, numpy out);
  * parameter constraints are validated at ``fit`` time with sklearn's machinery
    (``InvalidParameterError``), view errors are ``ValueError`` with the reference's messages.

Added (all defaulting to reference behaviour): ``precision`` selects the arithmetic of the
covariance kernel for float32 inputs, ``device`` the CUDA device.  Inputs may also be torch tensors
(CPU or CUDA); CUDA tensors are consumed in place, without a host round trip.  When
``torch.distributed`` is initialised with more than one rank, ``fit`` treats the views as this
rank's ROW SHARD and all-reduces the moments (SURVEY.md §8e).
"""
from __future__ import annotations

from abc import ABC, abstractmethod
from numbers import Integral
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.base import BaseEstimator
from sklearn.utils._param_validation import Interval, StrOptions
from sklearn.utils.validation import check_is_fitted

from . import ops, parallel
from .ops import HALF_DTYPES
from ._validation import validate_views


_COPY_STREAMS: dict = {}


def _copy_stream(device):
    """One side stream per device for host->device staging (kept off the estimator so that it stays picklable)."""
    key = (device.type, device.index)
    if key not in _COPY_STREAMS:
        _COPY_STREAMS[key] = torch.cuda.Stream(device)
    return _COPY_STREAMS[key]


def _shared_half_dtype(views):
    """The 16-bit dtype (torch.bfloat16 / torch.float16) all views share, else None.  numpy has no bfloat16; float16
    arrays count as torch.float16."""
    dts = {v.dtype if isinstance(v, torch.Tensor) else (torch.float16 if v.dtype == np.float16 else None)
           for v in views}
    dt = dts.pop() if len(dts) == 1 else None
    return dt if dt in HALF_DTYPES else None


def _as_tensor(v):
    return v if isinstance(v, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(v))


def _freeze(v):
    """A value-comparable snapshot of a constructor parameter (lists / arrays may be mutated in place between fits)."""
    if isinstance(v, (list, tuple)):
        return ("seq", type(v).__name__, tuple(_freeze(x) for x in v))
    if isinstance(v, np.ndarray):
        return ("nd", v.dtype.str, v.shape, v.tobytes())
    if isinstance(v, torch.Tensor):
        return ("tt", str(v.dtype), tuple(v.shape), v.detach().cpu().numpy().tobytes())
    if isinstance(v, dict):
        return ("map", tuple(sorted((repr(k), _freeze(x)) for k, x in v.items())))
    return (type(v).__name__, v)


class BaseModel(BaseEstimator, ABC):
    """Abstract base of all estimators (mirrors cca_zoo._base.BaseModel)."""

    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        "latent_dimensions": [Interval(Integral, 1, None, closed="left")],
        "center": ["boolean"],
        "precision": [StrOptions({"tf32", "tf32x3", "tf32x3b", "exact"})],
        "device": [None, str, int, torch.device],
    }

    #: dtype of the eigen-stage for float32 inputs: the reference keeps float32 in rCCA
    #: (numpy SVD) but upcasts to float64 in MCCA/GCCA (np.cov), see SURVEY.md §7.3-7.
    _solve_in_float64: ClassVar[bool] = False
    #: ``center=False`` only skips the mean subtraction of ``_setup_fit`` (cca_zoo/_base.py:96-99).  rCCA then works
    #: on the raw views (uncentred second moments); MCCA and its subclasses build A and B with ``np.cov``, which
    #: centres regardless (cca_zoo/linear/_mcca.py:150,166), so their covariance is always the centred one and
    #: ``center`` only decides ``means_``.
    _covariance_always_centred: ClassVar[bool] = False
    #: GCCA with ``center=False`` needs both: np.cov for the regularised blocks, raw products for the rest
    _wants_second_moment: ClassVar[bool] = False
    #: SCCA_IPLS with ``center=False`` carries the column means of the views through its deflation
    _wants_column_means: ClassVar[bool] = False

    def __init__(self, latent_dimensions: int = 1, center: bool = True, precision: str = "tf32x3b",
                 device=None) -> None:
        self.latent_dimensions = latent_dimensions
        self.center = center
        self.precision = precision
        self.device = device

    # ------------------------------------------------------------------ parameter validation
    _param_names_by_class: ClassVar[dict] = {}

    def _validate_params(self):
        """sklearn's constructor-parameter validation (InvalidParameterError at fit time, as in the reference:
        cca_zoo/_base.py:88).  It is reflection-heavy -- 0.1-0.2 ms of pure host time in front of the first kernel of a
        4 ms fit -- and a function of the parameters alone, so a re-fit of the same estimator with unchanged
        parameters does not repeat it."""
        cls = type(self)
        names = BaseModel._param_names_by_class.get(cls)
        if names is None:
            names = BaseModel._param_names_by_class[cls] = tuple(cls._get_param_names())
        snap = tuple(_freeze(getattr(self, n, None)) for n in names)
        if self.__dict__.get("_validated_params_") == snap:
            return
        super()._validate_params()
        self._validated_params_ = snap

    # ------------------------------------------------------------------ abstract
    @abstractmethod
    def fit(self, views, y=None):
        """Fit the model to multiview data (list of ``(n_samples, n_features_i)`` arrays)."""

    @abstractmethod
    def _solve(self, C: torch.Tensor, dims: list[int], n_total: int) -> list[torch.Tensor]:
        """Weights from the block covariance (device tensors)."""

    # ------------------------------------------------------------------ fit plumbing
    def _device(self) -> torch.device:
        if not torch.cuda.is_available():
            raise RuntimeError(
                "cca_zoo_b200 needs a CUDA device (sm_90a); there is no CPU fallback.  "
                "Use the reference cca_zoo package on CPU-only machines."
            )
        if self.device is None:
            return torch.device("cuda", torch.cuda.current_device())
        return torch.device(self.device)

    def _to_device(self, v, device):
        if isinstance(v, torch.Tensor):
            t = v
        else:
            arr = np.asarray(v)
            if arr.dtype not in (np.float32, np.float64):
                arr = arr.astype(np.float64)
            t = torch.from_numpy(np.ascontiguousarray(arr))
        if t.dtype not in (torch.float32, torch.float64):
            t = t.to(torch.float64)
        return t.to(device, non_blocking=True)

    #: host inputs larger than this many bytes are streamed to the device in row chunks (copy of chunk i+1
    #: overlaps the moment kernel of chunk i; device memory holds a few chunks instead of the whole data set)
    _stream_threshold_bytes: ClassVar[int] = 64 << 20
    _stream_chunk_rows: ClassVar[int] = 16384

    def _local_moments(self, validated, device):
        """Moment buffer of the rows this process holds.  Returns (moments, n_rows, dims, input dtype).

        Views that share one 16-bit dtype (bfloat16 / float16 tensors, float16 arrays) reach the moment kernel as they
        are, without a float64 copy; their input dtype is reported as float64, so every stage after the moment buffer
        runs as it does for a float64 copy of them."""
        half = _shared_half_dtype(validated)
        host = all(not (isinstance(v, torch.Tensor) and v.is_cuda) for v in validated)
        n_rows = int(validated[0].shape[0])
        nbytes = sum(int(np.prod(v.shape)) * (v.element_size() if isinstance(v, torch.Tensor) else v.dtype.itemsize)
                     for v in validated)
        if not (host and nbytes >= self._stream_threshold_bytes and n_rows >= 4 * self._stream_chunk_rows):
            if half is not None:
                dev_views = [_as_tensor(v).to(device, non_blocking=True) for v in validated]
            else:
                dev_views = [self._to_device(v, device) for v in validated]
                if len({v.dtype for v in dev_views}) > 1:
                    dev_views = [v.to(torch.float64) for v in dev_views]
            dims = [int(v.shape[1]) for v in dev_views]
            # shifted accumulation when a pilot over the leading rows finds badly centred columns (one-pass covariance
            # from raw moments would cancel: the reference centres first, cca_zoo/_base.py:96-99)
            mom, _ = ops.moments_safe(dev_views, precision=self.precision)
            return mom, n_rows, dims, torch.float64 if half is not None else dev_views[0].dtype
        # ---- streamed: the moments are additive over row chunks (the same identity the multi-GPU path uses) ----
        cpu_views = []
        for v in validated:
            t = _as_tensor(v)
            if t.dtype not in (torch.float32, torch.float64) and half is None:
                t = t.to(torch.float64)
            cpu_views.append(t)
        if len({t.dtype for t in cpu_views}) > 1:
            cpu_views = [t.to(torch.float64) for t in cpu_views]
        dims = [int(t.shape[1]) for t in cpu_views]
        main = torch.cuda.current_stream(device)
        copy = _copy_stream(device)
        mom = None
        step = self._stream_chunk_rows
        pending = None
        self._stream_x0 = "undecided"          # pilot origin of the shifted accumulation, fixed by the first chunk
        for lo in range(0, n_rows, step):
            hi = min(lo + step, n_rows)
            with torch.cuda.stream(copy):
                chunk = [t[lo:hi].to(device, non_blocking=True) for t in cpu_views]
                ready = torch.cuda.Event()
                ready.record(copy)
            if pending is not None:
                mom = self._accumulate(mom, pending, main)
            pending = (chunk, ready)
        mom = self._accumulate(mom, pending, main)
        return mom, n_rows, dims, torch.float64 if half is not None else cpu_views[0].dtype

    def _accumulate(self, mom, pending, main):
        chunk, ready = pending
        main.wait_event(ready)
        for c in chunk:
            c.record_stream(main)
        if isinstance(self._stream_x0, str):
            cand, ratio = ops.column_pilot(chunk)
            self._stream_x0 = cand if ratio > ops.SHIFT_RATIO[chunk[0].dtype] else None
        if self._stream_x0 is None:
            part = ops.moments(chunk, precision=self.precision)
        else:
            part, _ = ops.moments_safe(chunk, precision=self.precision, x0=self._stream_x0)
        if mom is None:
            return part
        mom.add_(part)
        return mom

    def _solve_dtype(self, in_dtype):
        """dtype of the covariance and of every solve after it, for views of ``in_dtype``."""
        return torch.float64 if (self._solve_in_float64 or in_dtype == torch.float64) else torch.float32

    def _covariance_stage(self, mom, n_local, dims, in_dtype, check_finite, reduced=False):
        """All-reduce (if sharded and not ``reduced`` already), finalise the covariance, record the fitted metadata
        (_base.py:94-101)."""
        if reduced:
            n_total = int(n_local)
        else:
            mom, n_total = parallel.allreduce_moments(mom, n_local, dims=dims)
        # NaN / inf anywhere in the inputs poisons the moments: one tiny device-side check replaces the
        # reference's host scan (check_array) for tensors that never visit the host
        if check_finite and not bool(torch.isfinite(mom).all()):
            raise ValueError("Input contains NaN or infinity.")
        solve_dtype = self._solve_dtype(in_dtype)
        centred = bool(self.center) or self._covariance_always_centred
        C, mean = ops.covariance(mom, dims, n_total, center=centred, dtype=solve_dtype)
        # estimators whose reference mixes np.cov (always centred) with products of the raw views (GCCA, center=False)
        self._second_moment = None
        if self._wants_second_moment and not self.center:
            self._second_moment, _ = ops.covariance(mom, dims, n_total, center=False, dtype=solve_dtype)
        self.n_views_ = len(dims)
        self.n_features_in_ = dims
        self.n_samples_ = n_total
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        mean_np = mean.to(torch.float64).cpu().numpy()
        if self._wants_column_means:
            self._column_means = mean_np if centred else ops.column_means(mom, dims, n_total)
        np_dtype = np.float32 if in_dtype == torch.float32 else np.float64
        if self.center:
            self.means_ = [mean_np[off[i]:off[i + 1]].astype(np_dtype) for i in range(len(dims))]
        else:
            self.means_ = [np.zeros(p) for p in dims]
        return C, dims, n_total

    def _fit_device(self, views, min_views: int = 2):
        """_setup_fit (cca_zoo/_base.py:78-102) + the covariance stage.  Returns (C, dims, n_total)."""
        self._validate_params()
        validated = validate_views(views, min_views)
        device = self._device()
        mom, n_local, dims, in_dtype = self._local_moments(validated, device)
        self._partial = None
        return self._covariance_stage(mom, n_local, dims, in_dtype, True)

    # ------------------------------------------------------------------ device-side fit (the fit behind the C ABI)
    def _device_fit_plan(self, dims, n_local, in_dtype):
        """None, or the arguments of the estimator's device-side fit (csrc/fit.cu) when this problem qualifies."""
        return None

    def _fit_moments(self, mom, n_local, dims, in_dtype):
        """From this process's moment buffer to ``weights_``: the exchange step, then either the device-side fit (one
        asynchronous library call, one copy of the result block, no other host synchronisation) or -- when the
        problem does not qualify or the device-side status word says so -- the host-assembled routes of
        ``_solvers.py``."""
        plan = self._device_fit_plan(dims, n_local, in_dtype)
        if plan is None:
            C, dims, n_total = self._covariance_stage(mom, n_local, dims, in_dtype, True)
            return self._finish(self._solve(C, dims, n_total))
        mom, n_host, n_dev = parallel.allreduce_moments_lazy(mom, n_local, dims=dims)
        solve_dtype = self._solve_dtype(in_dtype)
        attempts = plan.pop("iters")
        hdr = None
        for iters in attempts:
            block, offsets = plan["call"](mom, dims, n_host, n_dev, solve_dtype, iters)
            host = block.cpu()                                   # THE host synchronisation of the fit
            hdr, mean, sig, ws = ops.decode_fit_block(host, offsets, dims, plan["k"], solve_dtype)
            status = int(hdr[0])
            if status & ops.FIT_NON_FINITE:
                raise ValueError("Input contains NaN or infinity.")
            if status == 0:
                n_total = int(round(float(hdr[1])))
                self.n_views_ = len(dims)
                self.n_features_in_ = dims
                self.n_samples_ = n_total
                np_dtype = np.float32 if in_dtype == torch.float32 else np.float64
                off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
                if self.center:
                    self.means_ = [mean[off[i]:off[i + 1]].astype(np_dtype) for i in range(len(dims))]
                else:
                    self.means_ = [np.zeros(p) for p in dims]
                self._second_moment = None
                self.weights_ = [np.array(w) for w in ws]
                self._fit_info = {"route": "device", "iters": iters, "residual": float(hdr[2]), "sigma_1": float(hdr[3]),
                                  "ritz_sweeps": int(hdr[5])}
                return self
            if status != ops.FIT_NOT_CONVERGED:                  # only a missed tolerance is worth more iterations
                break
        # declined (a block is not positive definite, too few samples, no spectral gap): the host-assembled routes
        n_total = int(round(float(hdr[1])))
        C, dims, n_total = self._covariance_stage(mom, n_total, dims, in_dtype, False, reduced=True)
        self._fit_info = {"route": "host", "device_status": int(hdr[0])}
        return self._finish(self._solve(C, dims, n_total))

    def partial_fit(self, views, y=None, solve: bool = True):
        """Incremental fit on a batch of rows (a capability the reference lacks: its streaming answer is the
        stochastic EY family).  The block moments are additive over rows, so batches can arrive from disk or a
        loader in any split; the result after the last batch is the same as one ``fit`` on all rows (up to
        floating-point summation order).  ``solve=False`` only accumulates (use it for all but the last batch
        when the intermediate models are not needed)."""
        self._validate_params()
        validated = validate_views(views)
        device = self._device()
        mom, n_local, dims, in_dtype = self._local_moments(validated, device)
        state = getattr(self, "_partial", None)
        if state is not None:
            if state["dims"] != dims or state["dtype"] != in_dtype:
                raise ValueError(f"partial_fit batches must keep the view widths/dtype: {state['dims']} vs {dims}")
            mom = state["mom"].to(device).add_(mom)
            n_local += state["n"]
        self._partial = {"mom": mom, "n": n_local, "dims": dims, "dtype": in_dtype}
        if solve:
            self._fit_from_moments(mom.clone(), n_local, dims, in_dtype)
        return self

    _requires_two_views: ClassVar[bool] = False

    def _fit_from_moments(self, mom, n_local, dims, in_dtype):
        """Parameter validation, the view-count check and the solve from a moment buffer (consumed): the end of
        ``partial_fit``, and how ``model_selection.GridSearchCV`` fits each candidate from a split's train moments."""
        self._validate_params()
        if type(self)._requires_two_views and len(dims) != 2:
            raise ValueError(f"rCCA requires exactly 2 views, got {len(dims)}. Use MCCA for more than 2 views.")
        return self._fit_moments(mom, n_local, dims, in_dtype)

    def __getstate__(self):
        """Estimators stay picklable like the reference's (SURVEY.md §5): fitted state is numpy; an open
        partial_fit accumulator travels as a host tensor."""
        state = super().__getstate__()
        part = state.get("_partial")
        if part is not None:
            state = dict(state)
            state["_partial"] = {**part, "mom": part["mom"].detach().cpu()}
        return state

    def _finish(self, weights: list[torch.Tensor]):
        self.weights_ = [w.cpu().numpy() for w in weights]
        return self

    # ------------------------------------------------------------------ public API (reference semantics)
    @staticmethod
    def _as_numpy_views(views):
        out = []
        for v in views:
            out.append(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v)
        return out

    def transform(self, views):
        """Project views with the fitted weights: ``(v - mean_) @ weights_`` per view (cca_zoo/_base.py:108-123).

        CUDA tensors, and host inputs above ``_device_score_threshold`` elements, are projected on the device:
        ``Z_i = X_i W_i - 1 (mean_i^T W_i)`` is one GEMM per view (wgmma for float32, DMMA for float64) whose output
        is pre-loaded with the mean term, so neither a centred copy of the data nor a second pass exists.  Returns
        numpy arrays like the reference."""
        check_is_fitted(self)
        on_gpu = any(isinstance(v, torch.Tensor) and v.is_cuda for v in views)
        big = sum(int(np.prod(getattr(v, "shape", (0,)))) for v in views) >= self._device_score_threshold
        if on_gpu or (big and torch.cuda.is_available()):
            return self._transform_device(validate_views(views))
        validated = validate_views(self._as_numpy_views(views))
        return [(v - m) @ w for v, m, w in zip(validated, self.means_, self.weights_)]

    def _transform_device(self, validated, weights=None):
        device = self._device()
        out = []
        for v, m, w in zip(validated, self.means_, self.weights_ if weights is None else weights):
            X = self._to_device(v, device)
            np_dt = np.result_type(X.cpu().numpy().dtype if False else (np.float32 if X.dtype == torch.float32
                                                                         else np.float64), w.dtype)
            dt = torch.float32 if np_dt == np.float32 else torch.float64
            X = X.to(dt)
            W = torch.from_numpy(np.ascontiguousarray(w, dtype=np_dt)).to(device)
            mw = -(np.asarray(m, dtype=np.float64) @ np.asarray(w, dtype=np.float64))          # (k,) on the host: tiny
            Z = torch.from_numpy(mw.astype(np_dt)).to(device).expand(X.shape[0], -1).contiguous()
            ops.gemm(X, W, beta=1.0, out=Z)                                                  # Z <- X W + Z
            out.append(Z.cpu().numpy())
        return out

    def fit_transform(self, views, y=None):
        return self.fit(views, y).transform(views)

    def score(self, views, y=None):
        """Average pairwise canonical correlations per dimension (cca_zoo/_base.py:140-151)."""
        return self.average_pairwise_correlations(views)

    #: element count above which host inputs are scored on the device as well (one K1 pass instead of
    #: m tall numpy products); CUDA tensors always are
    _device_score_threshold: ClassVar[int] = 1 << 24

    def _pairwise_correlations_device(self, validated):
        """Correlations of the variates from the block covariance of ``views`` (SURVEY.md §8f-1):
        corr(X_i w_i, X_j w_j) = w_i^T C_ij w_j / sqrt(w_i^T C_ii w_i * w_j^T C_jj w_j)  per latent dimension,
        exactly what cca_zoo/_base.py:153-174 computes from the transformed samples (its centring makes the
        stored ``means_`` irrelevant) -- at the cost of one moment pass (K1) instead of m tall products."""
        device = self._device()
        dev_views = [self._to_device(v, device) for v in validated]
        if len({v.dtype for v in dev_views}) > 1:
            dev_views = [v.to(torch.float64) for v in dev_views]
        dims = [int(v.shape[1]) for v in dev_views]
        if dims != list(self.n_features_in_):
            raise ValueError(f"views have {dims} features, the model was fitted on {self.n_features_in_}")
        mom, _ = ops.moments_safe(dev_views, precision=self.precision)
        mom, n_total = parallel.allreduce_moments(mom, int(dev_views[0].shape[0]), dims=dims)
        C, _ = ops.covariance(mom, dims, n_total, center=True, dtype=torch.float64)
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        sl = [slice(int(off[i]), int(off[i + 1])) for i in range(len(dims))]
        W = [torch.from_numpy(np.ascontiguousarray(w, dtype=np.float64)).to(device) for w in self.weights_]
        m, k = len(dims), W[0].shape[1]
        S = torch.empty((m, m, k), dtype=torch.float64, device=device)
        for i in range(m):
            Ti = ops.gemm(C[:, sl[i]], W[i])                      # D x k : C[:, i] w_i
            for j in range(m):
                S[j, i] = ops.gemm(W[j], Ti[sl[j]], transa=True).diagonal()
        S = S.cpu().numpy()
        norms = np.sqrt(np.stack([S[i, i] for i in range(m)]) * (n_total - 1))     # ||centred variate||
        denom = np.where(norms > 1e-12, norms, 1.0) / np.sqrt(n_total - 1)
        return S / (denom[:, None, :] * denom[None, :, :])

    def pairwise_correlations(self, views):
        """(n_views, n_views, k) Pearson correlations of the variates (cca_zoo/_base.py:153-174)."""
        check_is_fitted(self)
        on_gpu = any(isinstance(v, torch.Tensor) and v.is_cuda for v in views)
        big = sum(int(np.prod(getattr(v, "shape", (0,)))) for v in views) >= self._device_score_threshold
        if on_gpu or (big and torch.cuda.is_available()):
            return self._pairwise_correlations_device(validate_views(views))
        transformed = self.transform(views)
        T = np.stack(transformed, axis=0)
        T = T - T.mean(axis=1, keepdims=True)
        norms = np.sqrt((T**2).sum(axis=1, keepdims=True))
        T_norm = T / np.where(norms > 1e-12, norms, 1.0)
        return np.einsum("isd,jsd->ijd", T_norm, T_norm)

    def average_pairwise_correlations(self, views):
        """Mean off-diagonal pairwise correlation per dimension (cca_zoo/_base.py:176-194)."""
        corrs = self.pairwise_correlations(views)
        n_views = corrs.shape[0]
        off_diag_sum = corrs.sum(axis=(0, 1)) - sum(corrs[i, i, :] for i in range(n_views))
        return off_diag_sum / (n_views * (n_views - 1))

    @property
    def weights(self):
        check_is_fitted(self)
        return self.weights_

    def get_factor_loadings(self, views):
        """Feature/variate correlations (cca_zoo/_base.py:208-234)."""
        validated = validate_views(self._as_numpy_views(views))
        transformed = self.transform(views)
        loadings = []
        for v, t in zip(validated, transformed):
            v_c = v - v.mean(axis=0)
            t_c = t - t.mean(axis=0)
            cov = v_c.T @ t_c / (v.shape[0] - 1)
            std_v = np.maximum(v_c.std(axis=0, ddof=1), 1e-12)
            std_t = np.maximum(t_c.std(axis=0, ddof=1), 1e-12)
            loadings.append(cov / np.outer(std_v, std_t))
        return loadings

    def __sklearn_tags__(self):
        tags = super().__sklearn_tags__()
        tags.no_validation = True
        tags.input_tags.two_d_array = False
        tags._skip_test = True
        return tags
