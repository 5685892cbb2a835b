"""
gpax_b200 -- H100-native exact-GP posterior path behind the gpax API (ExactGP / viGP / viSparseGP
`.predict()`, `.predict_in_batches()`, `.get_mvn_posterior()`, and the RBF / Matern / Periodic kernel
functions).  Python host code + ctypes -> libb200gp.so (hand-written sm_90a CUDA).  No JAX, no torch,
no CPU fallback on the product path.
"""
from . import kernels, utils
from .kernels import MaternKernel, PeriodicKernel, RBFKernel, get_kernel
from .gp import ExactGP
from .vigp import viGP
from .sparse_gp import viSparseGP
from .variants import MeasuredNoiseGP, UIGP, VarNoiseGP, vExactGP
from .mtgp import CoregGP, MultiTaskGP
from .dkl import DKL, viDKL, viMTDKL
from .ibnn import iBNN, vi_iBNN
from .bnn import BNN
from .spm import sPM
from .hypo import sample_next
from . import acquisition, diagnostics, hypo, mtkernels
from .kernels import NNGPKernel
from .mtkernels import LCMKernel, MultitaskKernel, MultivariateKernel
from ._ffi import B200GPError, Context, default_context

__version__ = "0.1.0"
__all__ = ["ExactGP", "iBNN", "vi_iBNN", "BNN", "sPM", "sample_next", "DKL", "viDKL", "viMTDKL", "MultiTaskGP", "CoregGP", "viGP", "viSparseGP", "MeasuredNoiseGP", "VarNoiseGP", "vExactGP", "UIGP", "acquisition", "RBFKernel", "MaternKernel", "PeriodicKernel", "NNGPKernel", "MultitaskKernel", "MultivariateKernel", "LCMKernel", "mtkernels", "get_kernel",
           "kernels", "utils", "Context", "default_context", "B200GPError"]
