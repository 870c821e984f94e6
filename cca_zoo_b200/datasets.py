"""Synthetic multiview inputs for parity tests and the benchmark.

``joint_data`` reproduces, draw for draw, the linear latent-variable generator the
reference uses for its examples (cca_zoo/datasets/_simulated.py:49-130: ``JointData``):
``W_i ~ N(0,1)^{d_i x k}`` are drawn first (constructor, :75-78), then ``z ~ N(0, I_k)`` and
per-view ``x_i = z W_i^T + N(0, 1/snr_i)`` in view order (``sample``, :113-125), all from one
``numpy.random.default_rng(random_state)`` stream.  Host-side numpy only: it feeds the
pipeline, it is not part of it.
"""
from __future__ import annotations

import numpy as np


def _per_view(value, m, name):
    if isinstance(value, (list, tuple)):
        if len(value) != m:
            raise ValueError(
                f"Parameter '{name}' must be a scalar or a list of length {m}, got {len(value)}."
            )
        return list(value)
    return [value] * m


def joint_data(n_views=2, n_samples=100, latent_dimensions=1, n_features=10,
               signal_to_noise=1.0, random_state=None, dtype=np.float64):
    """Return a list of ``n_views`` arrays ``(n_samples, n_features_i)``."""
    rng = np.random.default_rng(random_state)
    feats = _per_view(n_features, n_views, "n_features")
    snrs = _per_view(signal_to_noise, n_views, "signal_to_noise")
    weights = [rng.standard_normal((p, latent_dimensions)) for p in feats]
    z = rng.standard_normal((n_samples, latent_dimensions))
    views = []
    for w, snr in zip(weights, snrs):
        signal = z @ w.T
        noise_std = 1.0 / np.sqrt(snr) if snr > 0 else 1.0
        noise = rng.standard_normal(signal.shape) * noise_std
        views.append((signal + noise).astype(dtype, copy=False))
    return views


def joint_data_device(n_views=2, n_samples=100, latent_dimensions=1, n_features=10, signal_to_noise=1.0,
                      random_state=0, dtype=None, device=None, weights_seed=None):
    """The same latent-variable model (cca_zoo/datasets/_simulated.py:113-125) generated ON THE DEVICE: the views of a
    large configuration (BASELINE configs 4 and 5: 16 GB and 65 GB of float64 on the host) never exist in host memory.
    ``x_i = z W_i^T + N(0, 1/snr_i)`` with ``W_i`` drawn from ``weights_seed`` (default: ``random_state``) and the
    latent draws / noise from ``random_state`` -- ranks of a sharded fit pass one ``weights_seed`` and their own
    ``random_state`` so that their row shards are samples of ONE population.  Not draw-for-draw identical to the
    host generator (different RNG); returns a list of CUDA tensors."""
    import torch

    from . import ops

    dtype = torch.float32 if dtype is None else dtype
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    feats = _per_view(n_features, n_views, "n_features")
    snrs = _per_view(signal_to_noise, n_views, "signal_to_noise")
    gw = torch.Generator(device=device).manual_seed(int(random_state if weights_seed is None else weights_seed))
    g = torch.Generator(device=device).manual_seed(int(random_state) + 7919)
    weights = [torch.randn((p, latent_dimensions), generator=gw, device=device, dtype=dtype) for p in feats]
    z = torch.randn((n_samples, latent_dimensions), generator=g, device=device, dtype=dtype)
    views = []
    for w, snr in zip(weights, snrs):
        x = torch.randn((n_samples, w.shape[0]), generator=g, device=device, dtype=dtype)
        noise_std = 1.0 / float(np.sqrt(snr)) if snr > 0 else 1.0
        ops.gemm(z, w, transb=True, alpha=1.0, beta=noise_std, out=x)      # x <- z W^T + noise_std * x
        views.append(x)
    return views


def conftest_views(name):
    """The seeded fixtures of the reference test-suite (tests/conftest.py:9-59)."""
    rng = np.random.default_rng(42 if name == "two_views_test" else 0)
    if name == "two_views":
        return [rng.standard_normal((50, 10)), rng.standard_normal((50, 8))]
    if name == "three_views":
        return [rng.standard_normal((50, 10)), rng.standard_normal((50, 8)),
                rng.standard_normal((50, 6))]
    if name == "correlated_views":
        z = rng.standard_normal((50, 2))
        x1 = z @ rng.standard_normal((2, 10)) + 0.1 * rng.standard_normal((50, 10))
        x2 = z @ rng.standard_normal((2, 8)) + 0.1 * rng.standard_normal((50, 8))
        return [x1, x2]
    if name == "two_views_test":
        return [rng.standard_normal((20, 10)), rng.standard_normal((20, 8))]
    if name == "three_correlated_views":       # cca_zoo tests/linear/test_gradient.py:19-26
        z = rng.standard_normal((300, 2))
        return [z @ rng.standard_normal((2, p)) + 0.1 * rng.standard_normal((300, p)) for p in (10, 8, 6)]
    raise KeyError(name)
