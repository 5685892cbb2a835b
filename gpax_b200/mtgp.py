"""
mtgp.py -- `MultiTaskGP` and `CoregGP` with the reference's surface (gpax/models/mtgp.py:57-90, gpax/models/corgp.py:38-53):
exact GPs whose covariance is the linear model of coregionalisation (LCM) of mtkernels.py:197-233.  The posterior is one
b2gp_posterior_multitask call per predict (the LCM Gram matrices built on the GPU by gram_lcm_kernel, then ExactGP's
factorisation and solves), and b2gp_posterior_multitask_grad adds its gradient w.r.t. the test inputs; `fit` runs the
host NUTS on the multi-task log marginal likelihood and its gradient (b2gp_mll_multitask).  Both forms of the reference:
  * multitask form (shared_input_space=False, and CoregGP): one row per observation, its task id in the last column of X;
  * Kronecker form (MultiTaskGP with shared_input_space=True): every task observed at every input, y of length N*T in
    point-major order (point i, task t at i*T + t); predictions have length P*T in the same order.
"""
from typing import Callable, Dict, Optional

import numpy as np

from . import _ffi
from .gp import ExactGP, _eps_dtype
from .mtkernels import LCMKernel, MultitaskKernel
from .utils import posterior_eps

_BUILTIN = ("RBF", "Matern", "Periodic")


def _refuse_kernel(data_kernel):
    if data_kernel not in _BUILTIN:
        raise NotImplementedError("multi-task models take the data kernels 'RBF', 'Matern' and 'Periodic'")


def lcm_task_matrix(W, v):
    """B = W W^T + diag(v) (mtkernels.py:60-63) over any leading axes: W [..., T, R], v [..., T] -> B [..., T, T]"""
    W, v = np.asarray(W, dtype=np.float64), np.asarray(v, dtype=np.float64)
    return np.einsum("...tr,...ur->...tu", W, W) + v[..., None] * np.eye(W.shape[-2])


def lcm_points(X, T: int, shared: bool):
    """(data points [n, d], int32 task ids of the GP rows, group) of an input array.  The Kronecker form (shared) observes
    every point once per task: n * T rows, point-major, task index fastest; the multitask form reads the task id from the
    last column with astype(int) as the reference does, one row per point.  Task ids outside [0, T) raise ValueError (JAX
    would clamp the gather into B silently)."""
    X = np.asarray(X, dtype=np.float64)
    X = X if X.ndim > 1 else X[:, None]
    if shared:
        return X, np.tile(np.arange(T, dtype=np.int32), X.shape[0]), T
    t = X[:, -1].astype(int)
    if t.size and (t.min() < 0 or t.max() >= T):
        raise ValueError(f"task ids must lie in [0, {T}): got {t.min()} .. {t.max()}")
    return np.ascontiguousarray(X[:, :-1]), t.astype(np.int32), 1


class _LCMModel(ExactGP):
    """What MultiTaskGP and CoregGP share: parameter packing, task columns, the posterior and fit."""

    shared_input = False

    # ------------------------------------------------------------------ shapes
    def _num_tasks(self, X=None):
        """T: num_tasks, else the distinct labels of the task column of X_train (mtgp.py:106-107, corgp.py:66) -- or of
        X when given (the prior inputs of sample_from_prior)"""
        if self.num_tasks is None:
            X = np.asarray(self.X_train if X is None else X)
            return len(np.unique(X[:, -1]))
        return int(self.num_tasks)

    def _rank(self, T=None):
        return int(self.rank) if self.rank is not None else (self._num_tasks() if T is None else T) - 1   # mtgp.py:109-110

    def _data_dim(self, X):
        return X.shape[1] if self.shared_input else X.shape[1] - 1

    def _rows(self, X):
        """(data rows, int32 task ids, group) of an input array (lcm_points, each point repeated once per task in the
        Kronecker form)"""
        pts, t, group = lcm_points(X, self._num_tasks(), self.shared_input)
        return (np.repeat(pts, group, axis=0) if group > 1 else pts), t, group

    def _out_len(self, X_new):
        X_new = self._set_data(X_new)
        return X_new.shape[0] * (self._num_tasks() if self.shared_input else 1)

    def _scale_shape(self):
        return (self._num_latents(),) if self._num_latents() > 1 or isinstance(self, MultiTaskGP) else ()

    # ------------------------------------------------------------------ parameters
    def _pack(self, params: Dict[str, np.ndarray], batched: bool):
        """a params / samples dict with the reference's names and shapes -> theta [S, L, d+2] (lengthscale[d], k_scale,
        period), B [S, L, T, T] = W W^T + diag(v), noise [S, T]"""
        L, T, d = self._num_latents(), self._num_tasks(), self.kernel_dim
        W = np.asarray(params["W"], dtype=np.float64)
        S = W.shape[0] if batched else 1
        W = W.reshape(S, L, T, -1)
        v = np.asarray(params["v"], dtype=np.float64).reshape(S, L, T)
        ell = np.asarray(params["k_length"], dtype=np.float64).reshape(S, L, -1)
        if ell.shape[2] not in (1, d):
            raise ValueError(f"k_length has {ell.shape[2]} entries per latent for input_dim={d}")
        sc = params.get("k_scale")
        sc = np.ones((S, L)) if sc is None else np.broadcast_to(np.asarray(sc, dtype=np.float64).reshape(S, -1), (S, L))
        per = params.get("period")
        per = np.ones((S, L)) if per is None else np.broadcast_to(np.asarray(per, dtype=np.float64).reshape(S, -1), (S, L))
        theta = np.empty((S, L, d + 2))
        theta[:, :, :d] = ell
        theta[:, :, d], theta[:, :, d + 1] = sc, per
        B = lcm_task_matrix(W, v)
        noise = np.broadcast_to(np.asarray(params["noise"], dtype=np.float64).reshape(S, -1), (S, T)).copy()
        return theta, B, noise

    # ------------------------------------------------------------------ the posterior seam
    def _posterior_batched(self, X_new, params, batched, noiseless, want, eps=None, **kwargs):
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        if self._data_dim(X) != self.kernel_dim:
            raise ValueError(f"X_train has {self._data_dim(X)} input features, the model input_dim={self.kernel_dim}")
        theta, B, noise = self._pack(params, batched)
        S = theta.shape[0]
        Xd, ttr, group = self._rows(X)
        Xnd, tnew, _ = self._rows(Xn)
        yres = self._residuals(X, y, params, batched, S)
        out = self.ctx.posterior_multitask(self._fused, Xd, ttr, yres, Xnd, tnew, theta, B, noise, group, noiseless,
                                           float(kwargs.get("jitter", 1e-6)), want, eps)
        pm = self._prior_mean(Xn, params, batched, S)
        if pm is not None:
            if out["mean"] is not None:
                out["mean"] = out["mean"] + pm
            if out["y_sampled"] is not None:
                out["y_sampled"] = out["y_sampled"] + (pm[:, None, :] if pm.ndim == 2 else pm)
        return out

    def _posterior_grad(self, X_new, params, batched, noiseless, **kwargs):
        """Per-draw posterior mean [S, P], variance [S, P] and their gradients dmean, dvar [S, P, d + 1] w.r.t. the test
        inputs, task column included (b2gp_posterior_multitask_grad): what jax.grad through the acquisition w.r.t. x needs
        (optimize.py:70-88).  The task column reaches the kernel through astype(int), whose gradient is 0, so its entries
        are 0.  Multitask form only: the Kronecker form predicts T values per input, so its acquisition is not one scalar
        per x.  A mean function (an arbitrary host callable) has no analytic gradient either."""
        if self.shared_input:
            raise NotImplementedError("posterior gradients take the multitask form (task id in the last column of X)")
        if self.mean_fn is not None:
            raise NotImplementedError("posterior gradients need a model without a mean function")
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        Xn = Xn if Xn.ndim > 1 else Xn[:, None]
        if self._data_dim(X) != self.kernel_dim:
            raise ValueError(f"X_train has {self._data_dim(X)} input features, the model input_dim={self.kernel_dim}")
        theta, B, noise = self._pack(params, batched)
        Xd, ttr, group = self._rows(X)
        Xnd, tnew, _ = self._rows(Xn)
        out = self.ctx.posterior_multitask_grad(self._fused, Xd, ttr, y, Xnd, tnew, theta, B, noise, group, noiseless,
                                                float(kwargs.get("jitter", 1e-6)))
        dmean, dvar = (np.zeros(out[k].shape[:2] + (Xn.shape[1],)) for k in ("dmean", "dvar"))
        dmean[..., :-1], dvar[..., :-1] = out["dmean"], out["dvar"]
        return out["mean"], out["var"], dmean, dvar

    def _predict(self, rng_key, X_new, params, n: int, noiseless: bool = False, **kwargs):
        """gp.py:279-293: (mean [P'], samples [n, P']) with P' = P, or P*T for the Kronecker form"""
        Xn = self._set_data(X_new)
        eps = posterior_eps(rng_key, 1, n, self._out_len(Xn), _eps_dtype(), per_draw_keys=False)
        out = self._posterior_batched(Xn, params, False, noiseless, ("mean",), eps=eps, **kwargs)
        return out["mean"][0], out["y_sampled"][0]

    def predict(self, rng_key, X_new, samples=None, n: int = 1, filter_nans: bool = False, noiseless: bool = False,
                device=None, **kwargs):
        """gp.py:351-399: (mean over draws [P'], y_sampled [S, n, P']); P' = P, or P*T for the Kronecker form"""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(np.asarray(samples["W"]))
        eps = posterior_eps(rng_key, S, n, self._out_len(X_new), _eps_dtype())
        out = self._posterior_batched(X_new, samples, True, noiseless, ("mean",), eps=eps, **kwargs)
        y_means, y_sampled = out["mean"], out["y_sampled"]
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        dt = self._out_dtype(X_new)
        return y_means.mean(0).astype(dt, copy=False), y_sampled.astype(dt, copy=False)

    # ------------------------------------------------------------------ fit / prior
    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True,
            device=None, rng_key_predict=None, **kwargs) -> None:
        """gp.py:166-220 on the model's program: host NUTS, the likelihood and its gradient on the GPU (b2gp_mll_multitask)"""
        from .inference import MTLogJoint, run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        lj = MTLogJoint(self, kwargs.get("jitter", 1e-6))
        self.mcmc = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        if print_summary:
            self._print_summary()

    def sample_from_prior(self, rng_key, X, num_samples: int = 10) -> np.ndarray:
        """gp.py:401-408 with the model's program: samples [num_samples, N'] of the prior predictive at X"""
        from . import priors as P
        from .utils import seed_from_key
        X = np.asarray(self._set_data(X), dtype=np.float64)
        T = self._num_tasks(None if self.X_train is not None else X)
        R, L = self._rank(T), self._num_latents()
        rng = seed_from_key(rng_key)
        n_out, S = X.shape[0] * (T if self.shared_input else 1), int(num_samples)
        K, mean = np.empty((S, n_out, n_out)), np.zeros((S, n_out))
        for s in range(S):
            kp, noise, mp = P.run_program(lambda: self._model_program(T, R, L), rng=rng)[0]
            K[s] = np.asarray(self.kernel(X, X, {k: v for k, v in kp.items() if v is not None}, noise), dtype=np.float64)
            if self.mean_fn is not None:
                mean[s] = np.asarray(self.mean_fn(X, mp) if mp is not None else self.mean_fn(X), dtype=np.float64).squeeze()
        y, _ = self.ctx.mvn_sample(mean, K, rng.standard_normal((S, 1, n_out)))
        return y[:, 0, :]


class MultiTaskGP(_LCMModel):
    """
    Multi-task / multi-fidelity GP with the LCM kernel -- gpax/models/mtgp.py:57-90.

    Args:
        input_dim: number of input features (without the task column)
        data_kernel: 'RBF', 'Matern' or 'Periodic'
        num_latents: number of latent functions L (required unless shared_input_space)
        shared_input_space: every task observed at the same inputs (Kronecker form; needs num_tasks)
        num_tasks: T (inferred from the task column of X_train when not given and not shared)
        rank: rank of W (defaults to T - 1)
        mean_fn, data_kernel_prior, mean_fn_prior, noise_prior, noise_prior_dist, lengthscale_prior_dist,
        W_prior_dist, v_prior_dist, output_scale: as in the reference; priors are gpax_b200.priors objects / programs

    Limits of the GPU path: T <= 8, L <= 4, input_dim <= 16.  Task labels outside [0, T) raise ValueError (the reference's
    JAX gather would clamp them silently).  Acquisition functions work through `predict`.  In the multitask form without
    a mean function, `acquisition.optimize_acq` with EI / UCB / POI / UE takes the posterior's closed-form gradient w.r.t.
    x (one b2gp_posterior_multitask_grad call per evaluation, 0 on the task column); the Kronecker form and models with a
    mean function take finite differences.
    """

    def __init__(self, input_dim: int, data_kernel: str, num_latents: Optional[int] = None, shared_input_space: bool = False,
                 num_tasks: Optional[int] = None, rank: Optional[int] = None, mean_fn: Optional[Callable] = None,
                 data_kernel_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_prior: Optional[Callable] = None, noise_prior_dist=None, lengthscale_prior_dist=None,
                 W_prior_dist=None, v_prior_dist=None, output_scale: bool = False, ctx: Optional[_ffi.Context] = None,
                 **kwargs) -> None:
        _refuse_kernel(data_kernel)
        super().__init__(input_dim, data_kernel, mean_fn, None, mean_fn_prior, noise_prior, ctx=ctx)
        if shared_input_space:                                  # mtgp.py:71-76
            if num_tasks is None:
                raise ValueError("Please specify num_tasks")
        else:
            if num_latents is None:
                raise ValueError("Please specify num_latents")
        self.num_tasks = num_tasks
        self.num_latents = num_tasks if num_latents is None else num_latents
        self.rank = rank
        self.kernel = LCMKernel(data_kernel, shared_input_space, num_tasks, **kwargs)
        self.data_kernel_name = data_kernel
        self.data_kernel_prior = data_kernel_prior
        self.noise_prior_dist = noise_prior_dist
        self.lengthscale_prior_dist = lengthscale_prior_dist
        self.W_prior_dist = W_prior_dist
        self.v_prior_dist = v_prior_dist
        self.shared_input = shared_input_space
        self.output_scale = output_scale

    def _num_latents(self):
        return int(self.num_latents)

    def _model_program(self, T, R, L):
        from .inference import mtgp_model_program
        return mtgp_model_program(self, self.kernel_dim, T, R, L)


class CoregGP(_LCMModel):
    """
    Coregionalised GP -- gpax/models/corgp.py:38-53: the multitask form with one latent, k_scale fixed at 1, W [T, rank],
    v [T], noise [T]; T is the number of distinct task labels of X_train.  Task labels outside [0, T) raise ValueError.
    Acquisition functions work through `predict`.  Without a mean function, `acquisition.optimize_acq` with EI / UCB / POI
    / UE takes the posterior's closed-form gradient w.r.t. x (one b2gp_posterior_multitask_grad call per evaluation, 0 on
    the task column); with one it takes finite differences.
    """

    def __init__(self, input_dim: int, data_kernel: str, mean_fn: Optional[Callable] = None,
                 data_kernel_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_prior: Optional[Callable] = None, task_kernel_prior: Optional[Callable] = None, rank: int = 1,
                 ctx: Optional[_ffi.Context] = None, **kwargs) -> None:
        _refuse_kernel(data_kernel)
        super().__init__(input_dim, data_kernel, mean_fn, None, mean_fn_prior, noise_prior, ctx=ctx)
        self.num_tasks = None
        self.rank = rank
        self.kernel = MultitaskKernel(data_kernel, **kwargs)
        self.data_kernel_name = data_kernel
        self.data_kernel_prior = data_kernel_prior
        self.task_kernel_prior = task_kernel_prior

    def _num_tasks(self, X=None):
        return len(np.unique(np.asarray(self.X_train if X is None else X)[:, -1]))    # corgp.py:66

    def _num_latents(self):
        return 1

    def _model_program(self, T, R, L):
        from .inference import corgp_model_program
        return corgp_model_program(self, self.kernel_dim, T, R)
