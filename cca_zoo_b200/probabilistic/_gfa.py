"""GFA (Group Factor Analysis) on the GPU (mirrors cca_zoo/probabilistic/_gfa.py).

The reference runs closed-form mean-field variational Bayes over the full n x d views: four n x d_m x k products per
iteration, for up to ``max_iter`` iterations.  From the first Z update on the latent mean is z = X B with
B = [tau_1 W_1; ...; tau_m W_m] cov_z, so every later quantity of the loop is a function of the Gram matrix
G = X^T X (centred when ``center``) and of G B.  A fit here is therefore:

  1. the moment pass (the block moments of every other estimator), giving G and the data variances;
  2. the random start z0, drawn on the host exactly as the reference draws it, and X^T z0 (one GEMM per view);
  3. ONE ``ccab_gfa_fit`` call of ``max_iter`` iterations (each one D x D x k product, whatever n is);
  4. one copy of the state back, then z = X B (one GEMM per view) for the posterior samples, which the host draws
     with the reference's generator in the reference's order.

``partial_fit`` and the sharded fit are not supported: z0 is drawn over one global row order.
"""
from __future__ import annotations

from numbers import Integral, Real
from typing import Any, ClassVar

import numpy as np
import torch
from sklearn.utils._param_validation import Interval
from sklearn.utils.validation import check_is_fitted

from .. import ops, parallel
from .._base import BaseModel
from .._validation import validate_views


class GFA(BaseModel):
    r"""Group Factor Analysis: Bayesian CCA with per-view ARD (cca_zoo/probabilistic/_gfa.py).

    Same arguments, defaults and fitted attributes as the reference (``weights_``, ``view_relevance_``,
    ``n_components_``, ``n_iter_``, ``posterior_samples_``, ``means_``, ``n_views_``, ``n_features_in_``,
    ``n_samples_``), plus ``precision`` (arithmetic of the moment pass for float32 views) and ``device``.  The loop
    runs in float64 on the device; ``latent_dimensions`` may be at most 64.  ``transform`` returns a single-element
    list (the posterior mean of the shared z), as in the reference."""

    _solve_in_float64 = True
    _covariance_always_centred = True     # datavar uses np.var(ddof=1): always centred
    _wants_second_moment = True           # center=False iterates on the raw Gram matrix
    _parameter_constraints: ClassVar[dict[str, list[Any]]] = {
        **BaseModel._parameter_constraints,
        "max_iter": [Interval(Integral, 0, None, closed="left")],
        "tol": [Interval(Real, None, None, closed="neither")],
        "drop_k": ["boolean"],
        "num_posterior_samples": [Interval(Integral, 0, None, closed="left")],
        "random_state": [Interval(Integral, None, None, closed="neither")],
    }

    def __init__(self, latent_dimensions: int = 1, center: bool = True, max_iter: int = 10000, tol: float = 1e-4,
                 drop_k: bool = True, num_posterior_samples: int = 1000, random_state: int = 0,
                 precision: str = "tf32x3b", device=None) -> None:
        super().__init__(latent_dimensions=latent_dimensions, center=center, precision=precision, device=device)
        self.max_iter = max_iter
        self.tol = tol
        self.drop_k = drop_k
        self.num_posterior_samples = num_posterior_samples
        self.random_state = random_state

    # ------------------------------------------------------------------ fit
    def fit(self, views, y=None):
        self._validate_params()
        k = int(self.latent_dimensions)
        if k > ops.GFA_MAX_K:
            raise ValueError(f"latent_dimensions = {k}: GFA supports at most {ops.GFA_MAX_K} latent dimensions")
        if parallel.is_distributed():
            raise NotImplementedError("GFA has no sharded fit: its random start z0 takes one global row order")
        validated = validate_views(views)
        device = self._device()
        dev_views = [self._to_device(v, device) for v in validated]
        if len({v.dtype for v in dev_views}) > 1:
            dev_views = [v.to(torch.float64) for v in dev_views]
        mom, n_local, dims, in_dtype = self._local_moments(dev_views, device)
        self._partial = None
        C, dims, n = self._covariance_stage(mom, n_local, dims, in_dtype, True)
        off = np.concatenate([[0], np.cumsum(dims)]).astype(int)
        G = (C if self.center else self._second_moment).mul(n - 1)
        gdiag = G.diagonal().cpu().numpy()
        cdiag = C.diagonal().cpu().numpy()
        y_const = np.array([gdiag[off[i]:off[i + 1]].sum() for i in range(len(dims))])
        datavar = np.array([cdiag[off[i]:off[i + 1]].sum() for i in range(len(dims))])

        rng = np.random.default_rng(self.random_state)
        z0 = rng.standard_normal((n, k))
        XtZ0 = self._xt_z0(dev_views, z0, off)
        fit = ops.gfa_fit(dims, G, n, XtZ0, z0.T @ z0, datavar, y_const, float(self.tol), bool(self.drop_k))
        fit.run(int(self.max_iter))
        st = fit.result()

        kf = st["k"]
        self.n_iter_ = int(self.max_iter) if not st["stop"] else st["iters"]
        self.n_components_ = kf
        self.weights_ = [np.ascontiguousarray(st["W"][off[i]:off[i + 1]]) for i in range(len(dims))]
        self.view_relevance_ = st["alpha"].copy()
        z = self._latent_mean(dev_views, st["B"], off)
        a_ard = ops.GFA_ARD_ALPHA_0 + np.array(dims) / 2.0
        a_tau = ops.GFA_TAU_ALPHA_0 + n * np.array(dims) / 2.0
        self._draw_posterior_samples(rng, z, st["cov_z"], self.weights_, list(st["cov_w"]), a_ard,
                                     list(st["b_ard"]), a_tau, st["b_tau"], dims)
        self._fit_info = {"iters": st["iters"], "prunes": st["prunes"], "index": st["index"]}
        return self

    def partial_fit(self, views, y=None, solve: bool = True):
        raise NotImplementedError("GFA has no partial_fit: its random start z0 takes one global row order")

    def _solve(self, C, dims, n_total):
        raise NotImplementedError("GFA iterates in ccab_gfa_fit, not on a solved covariance")

    @staticmethod
    def _gemm(A, B, transa=False):
        """A product with a view: DMMA for float64, 3xTF32 tensor cores for float32 (FMA when TMA cannot address)."""
        if A.dtype == torch.float32:
            Bf = B.to(torch.float32).contiguous()
            try:
                return ops.gemm_tc(A, Bf, transa=transa).to(torch.float64)
            except ValueError:
                return ops.gemm(A, Bf, transa=transa).to(torch.float64)
        return ops.gemm(A, B, transa=transa)

    def _xt_z0(self, views, z0, off):
        """X^T z0 (D x k float64, CUDA) of the views as the loop sees them (centred when ``center``)."""
        device = views[0].device
        z0d = torch.from_numpy(z0).to(device)
        parts = [self._gemm(v, z0d, transa=True) for v in views]
        if self.center:
            s = torch.from_numpy(z0.sum(axis=0)).to(device)
            for i, p in enumerate(parts):
                mu = torch.from_numpy(np.asarray(self.means_[i], dtype=np.float64)).to(device)
                p.sub_(torch.outer(mu, s))
        return torch.cat(parts).contiguous()

    def _latent_mean(self, views, B, off):
        """z = X B (n x k float64, host): one GEMM per view; the centring is a rank-one correction of the sum."""
        device = views[0].device
        z = None
        shift = np.zeros(B.shape[1])
        for i, v in enumerate(views):
            Bi = np.ascontiguousarray(B[off[i]:off[i + 1]])
            zi = self._gemm(v, torch.from_numpy(Bi).to(device))
            z = zi if z is None else z.add_(zi)
            if self.center:
                shift += np.asarray(self.means_[i], dtype=np.float64) @ Bi
        z = z.cpu().numpy()
        return z - shift if self.center else z

    # ------------------------------------------------------------------ posterior sampling (host, reference order)
    def _draw_posterior_samples(self, rng, z, cov_z, w, cov_w, a_ard, b_ard, a_tau, b_tau, d):
        """The reference's draws, in its order, with its generator (cca_zoo/probabilistic/_gfa.py:301-352)."""
        s = int(self.num_posterior_samples)
        m_views = len(w)
        k = z.shape[1]
        samples: dict[str, np.ndarray] = {}
        chol_z = np.linalg.cholesky(cov_z)
        z_noise = rng.standard_normal((s, *z.shape)) @ chol_z.T
        samples["z"] = z[np.newaxis, :, :] + z_noise
        tau_samples = np.stack([rng.gamma(a_tau[m], 1.0 / b_tau[m], size=s) for m in range(m_views)], axis=1)
        samples["alpha"] = np.stack([rng.gamma(a_ard[m], 1.0 / b_ard[m], size=(s, k)) for m in range(m_views)],
                                    axis=1)
        for m in range(m_views):
            chol_w = np.linalg.cholesky(cov_w[m])
            w_noise = rng.standard_normal((s, d[m], k)) @ chol_w.T
            samples[f"W_{m}"] = w[m][np.newaxis, :, :] + w_noise
            psi_m = 1.0 / tau_samples[:, m]
            samples[f"log_psi_{m}"] = np.log(psi_m)[:, np.newaxis] * np.ones((1, d[m]))
        self.posterior_samples_ = samples

    # ------------------------------------------------------------------ PosteriorMeanTransformMixin
    def _psi(self):
        return [np.exp(np.array(self.posterior_samples_[f"log_psi_{i}"])).mean(axis=0) for i in range(self.n_views_)]

    def _use_device(self, views):
        on_gpu = any(isinstance(v, torch.Tensor) and v.is_cuda for v in views)
        big = sum(int(np.prod(getattr(v, "shape", (0,)))) for v in views) >= self._device_score_threshold
        return on_gpu or (big and torch.cuda.is_available())

    def _projections(self, views, weights):
        """(v_i - mean_i) @ weights_i per view: one GEMM per view on the device for CUDA tensors and large inputs."""
        if self._use_device(views):
            return self._transform_device(validate_views(views), weights)
        validated = validate_views(self._as_numpy_views(views))
        return [(v - m) @ w for v, m, w in zip(validated, self.means_, weights)]

    def transform(self, views):
        """The posterior mean of the shared latent variable, as a single-element list (cca_zoo/probabilistic/
        _utils.py:25-56,219-250): one GEMM per view with the psi^-1-scaled weights, summed, times Sigma_z."""
        check_is_fitted(self)
        psi_inv = [1.0 / np.maximum(p, 1e-8) for p in self._psi()]
        k = self.weights_[0].shape[1]
        precision = np.eye(k)
        for w, pi in zip(self.weights_, psi_inv):
            precision = precision + w.T @ (w * pi[:, np.newaxis])
        scaled = [w * pi[:, np.newaxis] for w, pi in zip(self.weights_, psi_inv)]
        information = sum(self._projections(views, scaled))
        return [information @ np.linalg.inv(precision)]

    def _per_view_projections(self, views):
        return self._projections(views, self.weights_)

    def pairwise_correlations(self, views):
        """(n_views, n_views, k) correlations of the per-view projections v_i @ W_i (not of ``transform``)."""
        check_is_fitted(self)
        if self._use_device(views):
            return self._pairwise_correlations_device(validate_views(views))
        T = np.stack(self._per_view_projections(views), axis=0)
        T = T - T.mean(axis=1, keepdims=True)
        norms = np.sqrt((T ** 2).sum(axis=1, keepdims=True))
        T_norm = T / np.where(norms > 1e-12, norms, 1.0)
        return np.einsum("isd,jsd->ijd", T_norm, T_norm)

    def get_factor_loadings(self, views):
        """Correlations of every feature with its view's own projection (cca_zoo/probabilistic/_utils.py:320-357)."""
        validated = validate_views(self._as_numpy_views(views))
        loadings = []
        for v, t in zip(validated, self._per_view_projections(views)):
            v_c = v - v.mean(axis=0)
            t_c = t - t.mean(axis=0)
            cov = v_c.T @ t_c / (v.shape[0] - 1)
            std_v = np.maximum(v_c.std(axis=0, ddof=1), 1e-12)
            std_t = np.maximum(t_c.std(axis=0, ddof=1), 1e-12)
            loadings.append(cov / np.outer(std_v, std_t))
        return loadings

    def log_likelihood(self, views) -> float:
        """Mean per-sample marginal log-likelihood of held-out views (cca_zoo/probabilistic/_utils.py:59-122), from
        one moment pass: with G_t the Gram matrix of the views centred by ``means_`` and V = Psi^-1 W,
        quad = tr(Psi^-1 G_t) - tr(M^-1 V^T G_t V),  M = I + W^T Psi^-1 W."""
        check_is_fitted(self)
        validated = validate_views(views)
        device = self._device()
        dev_views = [self._to_device(v, device) for v in validated]
        if len({v.dtype for v in dev_views}) > 1:
            dev_views = [v.to(torch.float64) for v in dev_views]
        dims = [int(v.shape[1]) for v in dev_views]
        if dims != list(self.n_features_in_):
            raise ValueError(f"views have {dims} features, the model was fitted on {self.n_features_in_}")
        mom, _ = ops.moments_safe(dev_views, precision=self.precision)
        n = int(dev_views[0].shape[0])
        C, mean = ops.covariance(mom, dims, n, center=True, dtype=torch.float64)
        psi = np.concatenate(self._psi())
        psi_inv = 1.0 / np.maximum(psi, 1e-8)
        W = np.vstack(self.weights_)
        V = W * psi_inv[:, np.newaxis]
        Vd = torch.from_numpy(np.ascontiguousarray(V)).to(device)
        VCV = ops.gemm(Vd, ops.gemm(C, Vd), transa=True).cpu().numpy()
        delta = mean.cpu().numpy() - np.concatenate([np.asarray(m, dtype=np.float64) for m in self.means_])
        gdiag = (n - 1) * C.diagonal().cpu().numpy() + n * delta ** 2
        Vd_ = V.T @ delta
        VGV = (n - 1) * VCV + n * np.outer(Vd_, Vd_)
        k = W.shape[1]
        M = np.eye(k) + W.T @ V
        quad = float(psi_inv @ gdiag) - float(np.sum(np.linalg.inv(M) * VGV.T))
        log_det = float(np.sum(np.log(np.maximum(psi, 1e-300)))) + np.linalg.slogdet(M)[1]
        return float(-0.5 * (W.shape[0] * np.log(2 * np.pi) + log_det + quad / n))
