"""
sparse_gp.py -- `viSparseGP` with the reference's surface (gpax/models/sparse_gp.py:49-60 constructor,
116-171 fit, 173-223 get_mvn_posterior).  The Nystrom / VFE posterior is one b2gp_sparse_posterior call, or with a user
kernel callable one b2gp_sparse_posterior_gram call on the blocks the callable returns.
"""
from typing import Callable, Dict, Optional, Tuple

import numpy as np

from .gp import _theta_rows
from .utils import initialize_inducing_points
from .vigp import viGP


class viSparseGP(viGP):
    """Variational-inference sparse GP (inducing points)."""

    def __init__(self, input_dim: int, kernel, mean_fn: Optional[Callable] = None,
                 kernel_prior: Optional[Callable] = None, mean_fn_prior: Optional[Callable] = None,
                 noise_prior: Optional[Callable] = None, noise_prior_dist=None, lengthscale_prior_dist=None,
                 guide: str = "delta", ctx=None) -> None:
        super().__init__(input_dim, kernel, mean_fn, kernel_prior, mean_fn_prior, noise_prior,
                         noise_prior_dist, lengthscale_prior_dist, guide, ctx=ctx)
        self.Xu = None

    def fit(self, rng_key, X, y, inducing_points_ratio: float = 0.1, inducing_points_selection: str = "random",
            num_steps: int = 1000, step_size: float = 5e-3, progress_bar: bool = True, print_summary: bool = True,
            device=None, **kwargs: float) -> None:
        """sparse_gp.py:116-171."""
        from .inference import fit_sparse_gp
        X, y = self._set_data(X, y)
        Xu0 = initialize_inducing_points(np.array(X, copy=True), inducing_points_ratio, inducing_points_selection, rng_key)
        self.X_train, self.y_train = X, y
        self.svi, self.kernel_params = fit_sparse_gp(self, rng_key, Xu0, num_steps, step_size, progress_bar, **kwargs)
        self.Xu = self.kernel_params.pop("Xu")
        if print_summary:
            self._print_summary()

    KSS_CHUNK = 256      # rows of the diagonal blocks k(X_new[a:b], X_new[a:b]) predict takes diag(Kss) from (P * KSS_CHUNK entries)

    def _posterior_callable_sparse(self, X_new, params, noiseless, want, **kwargs):
        """User kernel callable: the blocks of sparse_gp.py:193-215 from the reference's own kernel calls, then one
        b2gp_sparse_posterior_gram call.  Without "cov" only diag(Kss) is needed: it is taken from diagonal blocks
        k(X_new[a:b], X_new[a:b], ...) of KSS_CHUNK rows, which put noise_p and the jitter on their diagonal by the same
        shape rule as the full call, so no P x P matrix is formed."""
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        Xu = np.asarray(self._set_data(self.Xu), dtype=np.float64)
        noise = float(np.asarray(params["noise"]).reshape(-1)[0])
        noise_p = noise * (1 - int(bool(noiseless)))
        yres = self._residuals(X, y, params, False, 1)
        k = self.kernel
        Kuu = np.asarray(k(Xu, Xu, params, **kwargs), dtype=np.float64)
        Kuf = np.asarray(k(Xu, X, params, jitter=0), dtype=np.float64)
        Kus = np.asarray(k(Xu, Xn, params, jitter=0), dtype=np.float64)
        if "cov" in want:
            Kss = np.asarray(k(Xn, Xn, params, noise_p, **kwargs), dtype=np.float64)
        else:
            P, c = Xn.shape[0], self.KSS_CHUNK
            Kss = np.concatenate([np.diagonal(np.asarray(k(Xn[a:a + c], Xn[a:a + c], params, noise_p, **kwargs), dtype=np.float64))
                                  for a in range(0, P, c)])
        out = self.ctx.sparse_posterior_gram(Kuu, Kuf, yres, noise, Kus, Kss, want, kss_diag="cov" not in want)
        pm = self._prior_mean(Xn, params, False, 1)
        if pm is not None:
            out["mean"] = out["mean"] + pm
        return out

    def get_mvn_posterior(self, X_new, params: Dict[str, np.ndarray], noiseless: bool = False,
                          **kwargs: float) -> Tuple[np.ndarray, np.ndarray]:
        """sparse_gp.py:173-223: mean [P] and covariance [P, P] for a single theta."""
        if self._fused is None:
            out = self._posterior_callable_sparse(X_new, params, noiseless, ("mean", "cov"), **kwargs)
            dt = self._out_dtype(X_new)
            return out["mean"].astype(dt, copy=False), out["cov"].astype(dt, copy=False)
        X, y = self._train_arrays()
        Xn = np.asarray(self._set_data(X_new), dtype=np.float64)
        Xu = np.asarray(self._set_data(self.Xu), dtype=np.float64)
        d = X.shape[1]
        theta = _theta_rows(params, d, False)[0]
        yres = self._residuals(X, y, params, False, 1)
        out = self.ctx.sparse_posterior(self._fused, Xu, X, yres, Xn, theta, noiseless,
                                        float(kwargs.get("jitter", 1e-6)), ("mean", "cov"))
        mean, cov = out["mean"], out["cov"]
        pm = self._prior_mean(Xn, params, False, 1)
        if pm is not None:
            mean = mean + pm
        dt = self._out_dtype(X_new)
        return mean.astype(dt, copy=False), cov.astype(dt, copy=False)

    def predict(self, rng_key, X_new, samples=None, noiseless: bool = False, device=None, **kwargs: float):
        """viGP.predict through the sparse posterior (vigp.py:178-185 calls self.get_mvn_posterior):
        (mean, diag cov) with the variance epilogue only."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples()
        if self._fused is None:
            out = self._posterior_callable_sparse(X_new, samples, noiseless, ("mean", "var"), **kwargs)
            dt = self._out_dtype(X_new)
            return out["mean"].astype(dt, copy=False), out["var"].astype(dt, copy=False)
        X, y = self._train_arrays()
        Xn = np.asarray(X_new, dtype=np.float64)
        Xu = np.asarray(self._set_data(self.Xu), dtype=np.float64)
        theta = _theta_rows(samples, X.shape[1], False)[0]
        yres = self._residuals(X, y, samples, False, 1)
        out = self.ctx.sparse_posterior(self._fused, Xu, X, yres, Xn, theta, noiseless,
                                        float(kwargs.get("jitter", 1e-6)), ("mean", "var"))
        mean = out["mean"]
        pm = self._prior_mean(Xn, samples, False, 1)
        if pm is not None:
            mean = mean + pm
        dt = self._out_dtype(X_new)
        return mean.astype(dt, copy=False), out["var"].astype(dt, copy=False)
