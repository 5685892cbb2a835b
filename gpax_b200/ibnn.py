"""
ibnn.py -- `iBNN` and `vi_iBNN`, the infinite-width Bayesian neural networks (gpax/models/ibnn.py, gpax/models/vi_ibnn.py):
an ExactGP / viGP on the NNGP kernel (gpax/kernels/kernels.py:120-224) with `var_b` and `var_w` as the sampled kernel
parameters.  The posterior is the fused b2gp_posterior on the NNGP kinds (Gram builds, factorisation, solves and the
variance epilogue with the input-dependent prior diagonal on the GPU); fit() evaluates the marginal likelihood and its
gradient w.r.t. log var_b / log var_w / log noise with b2gp_mll.
"""
from typing import Callable, Dict, Optional

import numpy as np

from . import priors as P
from .gp import ExactGP
from .kernels import get_kernel
from .vigp import viGP


def nngp_theta_rows(params: Dict[str, np.ndarray], d: int, depth: int, batched: bool) -> np.ndarray:
    """dict with var_b, var_w, noise -> theta rows [S, d+3] = (depth [d], var_w, noise, var_b), b2gp_gram's NNGP layout"""
    var_b = np.asarray(params["var_b"], dtype=np.float64).reshape(-1)
    var_w = np.asarray(params["var_w"], dtype=np.float64).reshape(-1)
    noise = np.asarray(params["noise"], dtype=np.float64).reshape(-1)
    S = var_b.shape[0] if batched else 1
    if not batched and (var_b.size, var_w.size, noise.size) != (1, 1, 1):
        raise ValueError("a single parameter set needs scalar var_b, var_w and noise")
    th = np.empty((S, d + 3), dtype=np.float64)
    th[:, :d] = float(depth)
    th[:, d], th[:, d + 1], th[:, d + 2] = var_w.reshape(S), noise.reshape(S), var_b.reshape(S)
    return th


class _NNGPModel:
    """What iBNN and vi_iBNN share: the kernel, the theta packing and the sites var_b / var_w."""

    def _nngp_setup(self, depth, activation):
        depth = int(depth)
        if not 0 <= depth <= 16:
            raise ValueError(f"depth must be an integer in [0, 16], got {depth}")
        self.depth = depth
        self.activation = "relu" if activation == "relu" else "erf"      # kernels.py:205 (anything else is erf)
        self.kernel = get_kernel("NNGP", activation=self.activation, depth=depth)
        self.kernel_name = None
        self._fused = "NNGP_relu" if self.activation == "relu" else "NNGP_erf"

    def _theta(self, params, d, batched):
        return nngp_theta_rows(params, d, self.depth, batched)

    def _nngp_site_priors(self):
        raise NotImplementedError

    def _sample_kernel_params(self) -> Dict[str, np.ndarray]:
        """the var_b / var_w sites with the model's default priors (ibnn.py:54-61, vi_ibnn.py:53-60), as a gpax_b200.priors
        program"""
        pb, pw = self._nngp_site_priors()
        return {"var_b": P.sample("var_b", pb), "var_w": P.sample("var_w", pw)}

    def _posterior_grad(self, X_new, params, batched, noiseless, **kwargs):
        raise NotImplementedError("posterior gradients w.r.t. the test inputs are not implemented for the NNGP kernels")


class iBNN(_NNGPModel, ExactGP):
    """
    Infinite-width Bayesian neural net (gpax/models/ibnn.py): ExactGP on the NNGP kernel, var_b, var_w ~ LogNormal(0, 1).

    Args:
        input_dim: number of input features
        depth: layers of the corresponding infinite-width network (0..16)
        activation: 'erf' or 'relu'
        mean_fn, mean_fn_prior, noise_prior, noise_prior_dist: as ExactGP
        nngp_prior: optional prior program returning {"var_b": ..., "var_w": ...} (the reference's kernel_prior slot)
        ctx: optional gpax_b200.Context
    """

    def __init__(self, input_dim: int, depth: int = 3, activation: str = "erf", mean_fn: Optional[Callable] = None,
                 nngp_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_prior: Optional[Callable] = None, noise_prior_dist=None, ctx=None) -> None:
        super().__init__(input_dim, None, mean_fn, nngp_prior, mean_fn_prior, noise_prior, noise_prior_dist, ctx=ctx)
        self._nngp_setup(depth, activation)

    def _nngp_site_priors(self):
        return P.LogNormal(0.0, 1.0), P.LogNormal(0.0, 1.0)              # ibnn.py:59-60


class vi_iBNN(_NNGPModel, viGP):
    """
    Variational infinite-width Bayesian neural net (gpax/models/vi_ibnn.py): viGP on the NNGP kernel,
    var_b ~ HalfNormal(1), var_w ~ LogNormal(0, 10), noise ~ LogNormal(0, 1).  Arguments as iBNN (no noise_prior_dist).
    """

    def __init__(self, input_dim: int, depth: int = 3, activation: str = "erf", mean_fn: Optional[Callable] = None,
                 nngp_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_prior: Optional[Callable] = None, ctx=None) -> None:
        super().__init__(input_dim, None, mean_fn, nngp_prior, mean_fn_prior, noise_prior, ctx=ctx)
        self._nngp_setup(depth, activation)

    def _nngp_site_priors(self):
        return P.HalfNormal(1.0), P.LogNormal(0.0, 10.0)                 # vi_ibnn.py:58-59
