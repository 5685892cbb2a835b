"""
gp.py -- `ExactGP` with the reference's surface (gpax/models/gp.py:96-106 constructor,
253-277 get_mvn_posterior, 279-293 _predict, 295-349 predict_in_batches, 351-399 predict,
410-428 _set_data / _set_training_data).  The numerical path -- Gram builds, the N x N factorisation,
triangular solves, mean / covariance / samples, batched over posterior draws -- is one C-ABI call
(b2gp_posterior) per predict; nothing is computed on the host.
"""
import warnings
from typing import Callable, Dict, Optional, Tuple, Union

import numpy as np

from . import _ffi
from .kernels import builtin_name, get_kernel
from .utils import posterior_eps, split_in_batches, x64_enabled

kernel_fn_type = Callable[[np.ndarray, np.ndarray, Dict[str, np.ndarray], np.ndarray], np.ndarray]


def _theta_rows(params: Dict[str, np.ndarray], d: int, batched: bool) -> np.ndarray:
    """dict of hyper-parameters -> rows [S, d+3] = (lengthscale[d], k_scale, noise, period).
    `batched`: values carry a leading draw axis (gp.py:386-387) -- otherwise a single theta."""
    def get(name, default=None):
        v = params.get(name, default)
        return default if v is None else v
    ell = np.asarray(get("k_length"), dtype=np.float64)
    scale = np.asarray(get("k_scale"), dtype=np.float64)
    noise = np.asarray(get("noise"), dtype=np.float64)
    if batched:
        S = scale.shape[0]
        ell = ell.reshape(S, -1)
        period = np.asarray(get("period", np.ones(S)), dtype=np.float64).reshape(S)
        scale, noise = scale.reshape(S), noise.reshape(S)
    else:
        S = 1
        ell = ell.reshape(1, -1)
        period = np.asarray(get("period", 1.0), dtype=np.float64).reshape(1)
        scale, noise = scale.reshape(1), noise.reshape(1)
    if ell.shape[1] not in (1, d):
        raise ValueError(f"k_length has {ell.shape[1]} entries for input_dim={d}")
    th = np.empty((S, d + 3), dtype=np.float64)
    th[:, :d] = ell                       # scalar lengthscale broadcasts over the d features
    th[:, d], th[:, d + 1], th[:, d + 2] = scale, noise, period
    return th


GRAM_CHUNK_BYTES = 1 << 30      # host Gram bytes of one b2gp_posterior_gram call (user kernel callables)


def gram_chunks(S, N, P, full_kpp=True, budget=GRAM_CHUNK_BYTES):
    """[(start, stop)] over S draws such that each chunk's k_XX [N, N], k_pX [P, N] and k_pp ([P, P], or its diagonal
    [P]) stay under `budget` bytes; a draw larger than the budget is a chunk of its own"""
    per_draw = 8 * (N * N + P * N + (P * P if full_kpp else P))
    step = max(1, int(budget) // per_draw)
    return [(a, min(a + step, S)) for a in range(0, S, step)]


def _eps_dtype():
    return np.float64 if x64_enabled() else np.float32


class ExactGP:
    """
    Gaussian process with the reference's constructor (gpax/models/gp.py:96-106).

    Args:
        input_dim: number of input features
        kernel: 'RBF', 'Matern', 'Periodic' (fused GPU Gram build) or a callable
            ``k(X, Z, params, noise, jitter)`` (evaluated by the caller's function on the host, then
            factorised / solved on the GPU)
        mean_fn, kernel_prior, mean_fn_prior, noise_prior, noise_prior_dist, lengthscale_prior_dist:
            as in the reference; the priors matter to ``fit`` only
    """

    def __init__(self, input_dim: int, kernel: Union[str, kernel_fn_type],
                 mean_fn: Optional[Callable] = None, kernel_prior: Optional[Callable] = None,
                 mean_fn_prior: Optional[Callable] = None, noise_prior: Optional[Callable] = None,
                 noise_prior_dist=None, lengthscale_prior_dist=None, ctx: Optional[_ffi.Context] = None) -> None:
        if noise_prior is not None:      # gp.py:108-115
            warnings.warn("`noise_prior` is deprecated and will be removed in a future version. "
                          "Please use `noise_prior_dist` instead.", FutureWarning)
        if kernel_prior is not None:     # gp.py:116-123
            warnings.warn("`kernel_prior` will remain available for complex priors. However, for modifying "
                          "only the lengthscales, it is recommended to use `lengthscale_prior_dist` instead.",
                          UserWarning)
        self.kernel_dim = input_dim
        self.kernel = get_kernel(kernel)
        self.kernel_name = kernel if isinstance(kernel, str) else None
        self._fused = builtin_name(kernel)          # name of the fused GPU kernel, or None for a user callable
        self.mean_fn = mean_fn
        self.kernel_prior = kernel_prior
        self.mean_fn_prior = mean_fn_prior
        self.noise_prior = noise_prior
        self.noise_prior_dist = noise_prior_dist
        self.lengthscale_prior_dist = lengthscale_prior_dist
        self.X_train = None
        self.y_train = None
        self.mcmc = None
        self._ctx = ctx

    # ------------------------------------------------------------------ plumbing
    @property
    def ctx(self) -> _ffi.Context:
        if self._ctx is None:
            self._ctx = _ffi.default_context()
        return self._ctx

    def _set_data(self, X, y=None):
        """gp.py:410-414."""
        X = np.asarray(X)
        X = X if X.ndim > 1 else X[:, None]
        if y is not None:
            return X, np.asarray(y).squeeze()
        return X

    def _set_training_data(self, X_train_new=None, y_train_new=None, device=None) -> None:
        """gp.py:416-428 (`device` is accepted and ignored: the ctx owns the device)."""
        self.X_train = self.X_train if X_train_new is None else X_train_new
        self.y_train = self.y_train if y_train_new is None else y_train_new

    def _train_arrays(self):
        X = np.asarray(self.X_train, dtype=np.float64)
        X = X if X.ndim > 1 else X[:, None]
        y = np.asarray(self.y_train, dtype=np.float64).reshape(-1)
        return X, y

    def _residuals(self, X, y, params, batched, S):
        """gp.py:262-265: y_train minus the mean function, per draw when the mean function has parameters."""
        if self.mean_fn is None:
            return y
        if self.mean_fn_prior is None:
            return y - np.asarray(self.mean_fn(X), dtype=np.float64).squeeze()
        if not batched:
            return y - np.asarray(self.mean_fn(X, params), dtype=np.float64).squeeze()
        out = np.empty((S, y.shape[0]))
        for s in range(S):
            ps = {k: np.asarray(v)[s] for k, v in params.items()}
            out[s] = y - np.asarray(self.mean_fn(X, ps), dtype=np.float64).squeeze()
        return out

    def _prior_mean(self, X_new, params, batched, S):
        """gp.py:274-276."""
        if self.mean_fn is None:
            return None
        if self.mean_fn_prior is None:
            return np.asarray(self.mean_fn(X_new), dtype=np.float64).squeeze()
        if not batched:
            return np.asarray(self.mean_fn(X_new, params), dtype=np.float64).squeeze()
        return np.stack([np.asarray(self.mean_fn(X_new, {k: np.asarray(v)[s] for k, v in params.items()}),
                                    dtype=np.float64).squeeze() for s in range(S)])

    def _out_dtype(self, X_new):
        return np.float32 if np.asarray(X_new).dtype == np.float32 else np.float64

    # ------------------------------------------------------------------ the posterior seam
    def _theta(self, params, d, batched):
        """the posterior's theta rows [S, d+3] from a parameter dict (the NNGP models pack theirs differently)"""
        return _theta_rows(params, d, batched)

    def _f32_io(self, X_new):
        """the reference's default precision: float32 training data and test inputs go over the C-ABI as float32 and the
        results come back float32 (B2GP_FLAG_F32; gpax/utils/utils.py:19-21) -- no host-side casts of the big arrays"""
        return (np.asarray(self.X_train).dtype == np.float32 and np.asarray(self.y_train).dtype == np.float32
                and np.asarray(X_new).dtype == np.float32 and self.mean_fn is None)

    def _posterior_batched(self, X_new, params, batched, noiseless, want, eps=None, **kwargs):
        if self._fused is not None and self._f32_io(X_new):
            X = np.asarray(self.X_train)
            X = X if X.ndim > 1 else X[:, None]
            theta = self._theta(params, X.shape[1], batched)
            return self.ctx.posterior(self._fused, X, np.asarray(self.y_train).reshape(-1), self._set_data(X_new), theta, noiseless,
                                      float(kwargs.get("jitter", 1e-6)), want, eps, f32=True)
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        d = X.shape[1]
        jitter = float(kwargs.get("jitter", 1e-6))
        if self._fused is None:
            return self._posterior_gram(X, y, Xn, params, batched, noiseless, want, eps, jitter)
        theta = self._theta(params, d, batched)
        S = theta.shape[0]
        yres = self._residuals(X, y, params, batched, S)
        out = self.ctx.posterior(self._fused, X, yres, Xn, theta, noiseless, jitter, want, eps)
        return self._add_prior_mean(out, Xn, params, batched, S)

    def _add_prior_mean(self, out, Xn, params, batched, S):
        pm = self._prior_mean(Xn, params, batched, S)
        if pm is not None:
            if out["mean"] is not None:
                out["mean"] = out["mean"] + pm
            if out["y_sampled"] is not None:
                out["y_sampled"] = out["y_sampled"] + (pm[:, None, :] if pm.ndim == 2 else pm)
        return out

    def _posterior_gram(self, X, y, Xn, params, batched, noiseless, want, eps, jitter):
        """User kernel callable: per draw the three Gram blocks of gp.py:267-269 from the callable (host), then one
        b2gp_posterior_gram call per chunk of draws (GRAM_CHUNK_BYTES of host Grams) for the factorisation, solves, mean,
        variance, covariance and samples on the GPU"""
        S = len(next(np.asarray(v) for v in params.values() if v is not None)) if batched else 1
        yres = np.broadcast_to(self._residuals(X, y, params, batched, S), (S, X.shape[0]))
        N, P = X.shape[0], Xn.shape[0]
        full_kpp = "cov" in want or eps is not None
        chunks = []
        for a, b in gram_chunks(S, N, P, full_kpp):
            Kxx, Kpx, Kpp = np.empty((b - a, N, N)), np.empty((b - a, P, N)), np.empty((b - a, P, P) if full_kpp else (b - a, P))
            for s in range(a, b):
                ps = {k: (None if v is None else np.asarray(v)[s]) for k, v in params.items()} if batched else params
                noise = ps["noise"]
                noise_p = noise * (1 - int(bool(noiseless)))                                       # gp.py:260-261
                k_pp = np.asarray(self.kernel(Xn, Xn, ps, noise_p, jitter=jitter), dtype=np.float64)   # gp.py:267
                Kpp[s - a] = k_pp if full_kpp else np.diagonal(k_pp)
                Kpx[s - a] = self.kernel(Xn, X, ps, jitter=0.0)                                      # gp.py:268
                Kxx[s - a] = self.kernel(X, X, ps, noise, jitter=jitter)                             # gp.py:269
            chunks.append(self.ctx.posterior_gram(Kxx, Kpx, Kpp, yres[a:b], want, None if eps is None else eps[a:b],
                                                  kpp_diag=not full_kpp))
        out = {k: (None if chunks[0][k] is None else np.concatenate([c[k] for c in chunks]))
               for k in ("mean", "var", "cov", "y_sampled", "info")}
        return self._add_prior_mean(out, Xn, params, batched, S)

    def _posterior_grad(self, X_new, params, batched, noiseless, **kwargs):
        """Per-draw posterior mean [S, P], variance [S, P] and their gradients w.r.t. the test inputs dmean, dvar
        [S, P, d] (b2gp_posterior_grad): what jax.grad through the acquisition w.r.t. x needs (optimize.py:70-88).  fp32
        inputs are cast to fp64 here.  A model with a mean function has no analytic gradient (the mean function is an
        arbitrary host callable), nor has a user kernel callable.  Subclasses inherit this method but predict a different
        posterior; acquisition.optimize_acq uses it for ExactGP and viGP only."""
        if self.mean_fn is not None or self._fused is None:
            raise NotImplementedError("posterior gradients need a built-in kernel and no mean function")
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        theta = _theta_rows(params, X.shape[1], batched)
        out = self.ctx.posterior_grad(self._fused, X, y, Xn, theta, noiseless, float(kwargs.get("jitter", 1e-6)))
        return out["mean"], out["var"], out["dmean"], out["dvar"]

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], noiseless: bool = False,
                          **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """
        Mean [P] and covariance [P, P] of the multivariate-normal posterior for a single sample of GP
        parameters -- gpax/models/gp.py:253-277, with the explicit inverse of gp.py:271 replaced by a
        Cholesky factorisation and triangular solves on the GPU.  A non-positive-definite k_XX gives
        NaNs (the reference's LU path returns finite numbers there; SURVEY.md section 9).
        """
        if self._fused is None:
            return self._posterior_callable(X_new, params, noiseless, **kwargs)
        out = self._posterior_batched(X_new, params, False, noiseless, ("mean", "cov"), **kwargs)
        dt = self._out_dtype(X_new)
        return out["mean"][0].astype(dt, copy=False), out["cov"][0].astype(dt, copy=False)

    def _posterior_callable(self, X_new, params, noiseless=False, **kwargs):
        """User kernel callable: the three Gram matrices come from the callable (host), the factorisation
        and the solves run on the GPU (b2gp_potrf / b2gp_trsm_lower / b2gp_gemm_nt)."""
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        noise = params["noise"]
        noise_p = noise * (1 - int(bool(noiseless)))
        yres = self._residuals(X, y, params, False, 1)
        k_pp = np.asarray(self.kernel(Xn, Xn, params, noise_p, **kwargs), dtype=np.float64)
        k_pX = np.asarray(self.kernel(Xn, X, params, jitter=0.0), dtype=np.float64)
        k_XX = np.asarray(self.kernel(X, X, params, noise, **kwargs), dtype=np.float64)
        L, info = self.ctx.potrf(k_XX)
        rhs = np.concatenate([k_pX, yres[None, :]], axis=0)
        V = self.ctx.trsm_lower(L, rhs)
        mean = V[:-1] @ V[-1]
        cov = self.ctx.gemm_nt(V[:-1], V[:-1], k_pp, alpha=-1.0, beta=1.0)
        if info != 0:
            mean[:] = np.nan
            cov[:] = np.nan
        pm = self._prior_mean(Xn, params, False, 1)
        if pm is not None:
            mean = mean + pm
        return mean, cov

    # ------------------------------------------------------------------ predict
    def _predict(self, rng_key, X_new, params: Dict[str, np.ndarray], n: int, noiseless: bool = False,
                 **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """Prediction with a single sample of GP parameters (gp.py:279-293): (mean [P], samples [n, P])."""
        Xn = self._set_data(X_new)
        eps = posterior_eps(rng_key, 1, n, Xn.shape[0], _eps_dtype(), per_draw_keys=False)
        if self._fused is None:
            mean, cov = self._posterior_callable(Xn, params, noiseless, **kwargs)
            Lc, info = self.ctx.potrf(cov)
            y = mean[None, :] + eps[0] @ np.tril(Lc).T if info == 0 else np.full((n, Xn.shape[0]), np.nan)
            return mean, y
        out = self._posterior_batched(Xn, params, False, noiseless, ("mean",), eps=eps, **kwargs)
        return out["mean"][0], out["y_sampled"][0]

    def get_samples(self, chain_dim: bool = False) -> Dict[str, np.ndarray]:
        """gp.py:249-251: posterior samples of the hyper-parameters after `fit`."""
        if self.mcmc is None:
            raise RuntimeError("no posterior samples: call fit() first or pass `samples=` to predict()")
        return self.mcmc.get_samples(group_by_chain=chain_dim)

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1,
                filter_nans: bool = False, noiseless: bool = False, device=None,
                **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """
        Prediction at X_new with posterior samples of the GP parameters -- gpax/models/gp.py:351-399.
        The reference vmaps `_predict` over the S draws (gp.py:393-395), materialising S copies of k_XX;
        here the draws stream through a small ring of N x N workspaces on the GPU.

        Returns (mean over draws [P], y_sampled [S, n, P]).
        """
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        P = X_new.shape[0]
        eps = posterior_eps(rng_key, S, n, P, _eps_dtype())
        out = self._posterior_batched(X_new, samples, True, noiseless, ("mean",), eps=eps, **kwargs)
        y_means, y_sampled = out["mean"], out["y_sampled"]
        if filter_nans:                                     # gp.py:396-398
            keep = [i for i in range(S) if not np.isnan(y_sampled[i]).any()]
            y_sampled = y_sampled[keep]
        dt = self._out_dtype(X_new)
        return y_means.mean(0).astype(dt, copy=False), y_sampled.astype(dt, copy=False)

    def _predict_in_batches(self, rng_key, X_new, batch_size: int = 100, batch_dim: int = 0,
                            samples=None, n: int = 1, filter_nans: bool = False, predict_fn=None,
                            noiseless: bool = False, device=None, **kwargs):
        """gp.py:295-323."""
        if predict_fn is None:
            predict_fn = lambda xi: self.predict(rng_key, xi, samples, n, filter_nans, noiseless, device, **kwargs)  # noqa: E731
        y_out1, y_out2 = [], []
        for Xi in split_in_batches(np.asarray(X_new), batch_size, dim=batch_dim):
            out1, out2 = predict_fn(Xi)
            y_out1.append(out1)
            y_out2.append(out2)
        return y_out1, y_out2

    def predict_in_batches(self, rng_key, X_new, batch_size: int = 100, samples=None, n: int = 1,
                           filter_nans: bool = False, predict_fn=None, noiseless: bool = False, device=None,
                           **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """gp.py:325-349: chunk X_new, predict each chunk, concatenate."""
        y_pred, y_sampled = self._predict_in_batches(rng_key, X_new, batch_size, 0, samples, n, filter_nans,
                                                     predict_fn, noiseless, device, **kwargs)
        return np.concatenate(y_pred, 0), np.concatenate(y_sampled, -1)

    # ------------------------------------------------------------------ fit (host-side inference, see inference.py)
    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True,
            device=None, rng_key_predict=None, **kwargs: float) -> None:
        """gp.py:166-220.  The reference runs NumPyro's NUTS over the hyper-parameters; here a host-side NUTS
        (gpax_b200/inference.py) samples the same posterior with the log marginal likelihood and its gradient
        evaluated on the GPU (b2gp_mll), LogNormal(0, 1) priors by default (gp.py:222-247)."""
        from .inference import fit_exact_gp
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        self.mcmc = fit_exact_gp(self, rng_key, num_warmup, num_samples, num_chains, progress_bar, **kwargs)
        if print_summary:
            self._print_summary()

    def sample_from_prior(self, rng_key, X, num_samples: int = 10) -> np.ndarray:
        """gp.py:401-408: samples [num_samples, N] from the prior predictive at X -- hyper-parameters (and mean-function
        parameters) drawn from their priors, y ~ N(mean_fn(X), k(X, X) + (noise + jitter) I) per draw.  The Gram matrices
        are built and the draws made on the device (kernel call, b2gp_mvn_sample); the key seeds NumPy's generator (the
        distribution is the reference's, NumPyro's own key stream is not reproduced)."""
        from .inference import prior_draws
        from .utils import seed_from_key
        X = np.asarray(self._set_data(X), dtype=np.float64)
        N, S = X.shape[0], int(num_samples)
        rng = seed_from_key(rng_key)
        K, mean = np.empty((S, N, N)), np.zeros((S, N))
        for s, (kp, noise, mp) in enumerate(prior_draws(self, rng, S, X.shape[1])):
            K[s] = np.asarray(self.kernel(X, X, kp, noise), dtype=np.float64)              # gp.py:157
            if self.mean_fn is not None:                                                    # gp.py:150-155
                mean[s] = np.asarray(self.mean_fn(X, mp) if mp is not None else self.mean_fn(X), dtype=np.float64).squeeze()
        y, _ = self.ctx.mvn_sample(mean, K, rng.standard_normal((S, 1, N)))
        return y[:, 0, :]

    def _print_summary(self):
        samples = self.get_samples(1)
        for k, v in samples.items():
            v = np.asarray(v)
            print(f"{k:>12s}  mean {np.mean(v, axis=(0, 1))}  std {np.std(v, axis=(0, 1))}")
