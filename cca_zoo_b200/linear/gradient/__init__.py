"""Gradient-descent (Eckart-Young) estimators, at the reference's import path ``cca_zoo.linear.gradient``."""
from .._gradient import CCA_EY, MCCA_EY, PLS_EY

__all__ = ["PLS_EY", "CCA_EY", "MCCA_EY"]
