"""Kernel (nonparametric) CCA methods, at the reference's import path ``cca_zoo.nonparametric``.

``KCCA`` runs on the device: pairwise kernel matrices from ``ccab_pairwise_kernel`` and the kernel eigenproblem
solved in each kernel matrix's eigenbasis.  ``KGCCA`` and ``KTCCA`` are not provided."""
from ._kcca import KCCA

__all__ = ["KCCA"]
