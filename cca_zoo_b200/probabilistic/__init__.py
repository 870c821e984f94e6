"""Probabilistic (Bayesian) CCA methods, at the reference's import path ``cca_zoo.probabilistic``.

``GFA`` is closed-form variational Bayes and runs on the device.  ``ProbabilisticCCA`` and ``VariationalBayesCCA``
need numpyro and jax in the reference and are not provided."""
from ._gfa import GFA

__all__ = ["GFA"]
