"""Kernel (nonparametric) CCA methods, at the reference's import path ``cca_zoo.nonparametric``.

All three run on the device, each solved in the eigenbases of its pairwise kernel matrices (``ccab_pairwise_kernel``
and ``syevj``): ``KCCA`` whitens the kernel eigenproblem there, ``KGCCA`` sums the kernel GCCA matrix there and
``KTCCA`` whitens each kernel matrix there before the cross-moment contraction and the CP-ALS of TCCA.

``__all__`` lists KCCA alone, as it did before KGCCA and KTCCA were added, so that a star import binds the same names
as before; import the other two by name."""
from ._kcca import KCCA
from ._kgcca import KGCCA
from ._ktcca import KTCCA

__all__ = ["KCCA"]
