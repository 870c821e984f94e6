"""Estimators on the hot path: same names and constructor arguments as ``cca_zoo.linear`` (every one of them, CCAR3
included)."""
from ._rcca import CCA, PLS, rCCA
from ._mcca import MCCA
from ._gcca import GCCA
from ._partialcca import PartialCCA
from ._grcca import GRCCA
from ._tcca import TCCA
from ._ccar3 import CCAR3
from ._iterative import PLS_ALS, SCCA_ADMM, SCCA_IPLS, SCCA_PMD, ElasticCCA, ParkhomenkoCCA, SCCA_Span
from .gradient import CCA_EY, MCCA_EY, PLS_EY

__all__ = ["CCA", "rCCA", "PLS", "MCCA", "GCCA", "PartialCCA", "GRCCA", "PLS_ALS", "SCCA_PMD", "ParkhomenkoCCA",
           "SCCA_Span", "SCCA_ADMM", "SCCA_IPLS", "ElasticCCA", "PLS_EY", "CCA_EY", "MCCA_EY",
           "TCCA", "CCAR3"]
