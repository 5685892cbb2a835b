"""
bnn.py -- the fully Bayesian MLP with the reference's surface: `BNN` (gpax/models/bnn.py) over `sPM` (gpax/models/spm.py).
A tanh MLP over `hidden_dim` (default [64, 32]) and a linear output layer map X [N, D] to the mean of y [N, O]; NUTS
samples every weight (Normal(0, 1)) and bias (Cauchy(0, 1)) together with the observation noise (LogNormal(0, 1) or
`noise_prior_dist`).  Every numerical step is on the GPU: b2gp_bnn_loglik evaluates sum log N(y; MLP(X), noise) and its
gradient w.r.t. the noise and every weight for each leapfrog step (b2gp_bnn_loglik_draws for every chain of a round under
chain_method="vectorized"), b2gp_bnn_predict runs the network for all draws at
once with the predictive sampling in the same epilogue.  The sampler is the host NUTS loop the other models use
(inference.run_nuts).

Sites, as the reference names them: w0, b0, ..., w{L}, b{L} (L = len(hidden_dim)), noise, and the deterministic `mu`
[S, N, O] (spm.py:70), which is computed once after sampling on the training inputs.  Initialisation is numpyro's
init_to_median(num_samples=10) (spm.py:112): every element of every site starts at the median of 10 prior draws, seeded
from `rng_key` (bitwise equality with a JAX run is not a goal).

Not supported: custom `nn` / `nn_prior` callables (NotImplementedError: the network and its prior are built in) and the
deprecated `noise_prior` program.  `device` is accepted and ignored: the context owns the device.
"""
from typing import Dict, List, Optional, Tuple

import numpy as np

from . import _ffi
from . import priors as P
from .dkl import _nn_log_prior
from .gp import _eps_dtype
from .utils import posterior_eps, seed_from_key

INIT_MEDIAN_DRAWS = 10        # spm.py:112, init_to_median(num_samples=10)


class BNNLogJoint:
    """log p(y, sites) of sPM.model with bnn.py's MLP (spm.py:63-77) over u = (unconstrained noise, w0, b0, ..., wL, bL)
    for run_nuts: the likelihood and its gradient from b2gp_bnn_loglik, Normal(0, 1) weights and Cauchy(0, 1) biases,
    the noise prior with its Jacobian.  X and y are uploaded once for the whole fit."""

    def __init__(self, model, X, y, rng):
        self.m, self.rng = model, rng
        self.Xd, self.yd = model.ctx.to_device(X), model.ctx.to_device(y)
        self.noise = model._noise_prior()
        self.wmask = model._weight_mask()
        self.dim = 1 + self.wmask.size
        self.n_evals = 0

    def close(self):
        self.Xd.free()
        self.yd.free()

    def _lik(self, flat, sigma):
        m = self.m
        return m.ctx.bnn_loglik(self.Xd, self.yd, m.widths, _ffi.ACT_TANH, flat, sigma)

    def init_u(self):
        """init_to_median(num_samples=10): the element-wise median of 10 prior draws of every site"""
        draws = self.noise.sample(self.rng, (INIT_MEDIAN_DRAWS,))
        u_noise = float(self.noise.inverse(np.median(draws)))
        n = self.wmask.size
        net = np.where(self.wmask, np.median(self.rng.standard_normal((INIT_MEDIAN_DRAWS, n)), axis=0),
                       np.median(self.rng.standard_cauchy((INIT_MEDIAN_DRAWS, n)), axis=0))
        return np.concatenate([[u_noise], net])

    def _sigma(self, u):
        """the noise of u, or None where it is not a valid scale (the likelihood is not evaluated there)"""
        sigma = float(self.noise.transform(u[0]))
        return sigma if np.isfinite(sigma) and sigma > 0.0 else None

    def __call__(self, u, jacobian):
        self.n_evals += 1
        sigma = self._sigma(u)
        if sigma is None:
            return -np.inf, np.zeros(self.dim)
        val, gs, gp = self._lik(u[1:], sigma)
        return self._joint(u, sigma, val, gs, gp, jacobian)

    def batch(self, U, jacobian):
        """`batch(U, jacobian) -> (values [k], grads [k, dim])` for run_nuts' vectorized chains: the rows with a valid noise
        in one b2gp_bnn_loglik_draws call on the resident X and y, each finished as __call__ finishes it, so row r is
        self(U[r], jacobian) bit for bit"""
        U = np.asarray(U, dtype=np.float64)
        self.n_evals += len(U)
        vals, grads = np.full(len(U), -np.inf), np.zeros((len(U), self.dim))
        sig = [self._sigma(u) for u in U]
        ok = [r for r, s in enumerate(sig) if s is not None]
        if ok:
            m = self.m
            v, gs, gp = m.ctx.bnn_loglik_draws(self.Xd, self.yd, m.widths, _ffi.ACT_TANH, U[ok, 1:], [sig[r] for r in ok])
            for i, r in enumerate(ok):
                vals[r], grads[r] = self._joint(U[r], sig[r], float(v[i]), float(gs[i]), gp[i], jacobian)
        return vals, grads

    def _joint(self, u, sigma, val, gs, gp, jacobian):
        """the log joint and its gradient w.r.t. u from the likelihood's value and gradients at sigma = noise(u)"""
        pr, flat = self.noise, u[1:]
        ds = float(pr.dtheta_du(u[0]))
        val += float(pr.log_prob(sigma))
        gu = (gs + float(pr.dlog_prob(sigma))) * ds
        if jacobian:
            val += float(pr.log_abs_jac(u[0]))
            gu += float(pr.dlog_abs_jac(u[0]))
        lp, glp = _nn_log_prior(self.wmask, flat)
        val += lp
        g = np.concatenate([[gu], gp + glp])
        if not (np.isfinite(val) and np.all(np.isfinite(g))):
            return -np.inf, np.zeros(self.dim)
        return val, g

    def to_dict(self, U):
        U = np.atleast_2d(U)
        out = self.m.from_flat(U[:, 1:])
        out["noise"] = np.asarray(self.noise.transform(U[:, 0]), dtype=np.float64)
        return out


class BNN:
    """
    Fully Bayesian MLP (gpax/models/bnn.py): `BNN(input_dim, output_dim, noise_prior_dist=None, hidden_dim=None, ctx=None)`.
    The surface of the reference's BNN / sPM: fit (NUTS), get_samples, get_param_means, sample_from_prior,
    sample_single_posterior_predictive and predict.
    """

    def __init__(self, input_dim: int, output_dim: int, noise_prior_dist=None, hidden_dim: Optional[List[int]] = None,
                 ctx: Optional[_ffi.Context] = None, **kwargs) -> None:
        if "nn" in kwargs or "nn_prior" in kwargs:
            raise NotImplementedError("custom nn / nn_prior callables are not supported: the tanh MLP and its Normal(0, 1) "
                                      "weight / Cauchy(0, 1) bias prior are built in")
        hidden = [64, 32] if not hidden_dim else [int(h) for h in hidden_dim]      # bnn.py:24
        self.input_dim, self.output_dim = int(input_dim), int(output_dim)
        self.hidden_dim = hidden
        self.widths = hidden + [self.output_dim]
        self.noise_prior_dist = noise_prior_dist
        self.mcmc = None
        self.X_train = self.y_train = None
        self._ctx = ctx

    @property
    def ctx(self) -> _ffi.Context:
        if self._ctx is None:
            self._ctx = _ffi.default_context()
        return self._ctx

    # ---- layout
    def _shapes(self):
        """[(in, out)] per layer"""
        ins = [self.input_dim] + self.widths[:-1]
        return list(zip(ins, self.widths))

    def _weight_mask(self):
        """True at the weights, False at the biases of the flat layout"""
        return np.concatenate([np.r_[np.ones(i * w), np.zeros(w)] for i, w in self._shapes()]).astype(bool)

    def _noise_prior(self):
        return self.noise_prior_dist if self.noise_prior_dist is not None else P.LogNormal(0.0, 1.0)

    def site_names(self) -> List[str]:
        return [n for i in range(len(self.widths)) for n in (f"w{i}", f"b{i}")] + ["noise"]

    def to_flat(self, params) -> np.ndarray:
        """site dict -> flat parameters [S, P] (leading draw axis) or [P]"""
        lead = np.asarray(params["w0"]).shape[:-2]
        parts = []
        for i in range(len(self.widths)):
            parts += [np.asarray(params[f"w{i}"], np.float64).reshape(lead + (-1,)),
                      np.asarray(params[f"b{i}"], np.float64).reshape(lead + (-1,))]
        return np.concatenate(parts, axis=-1)

    def from_flat(self, flat) -> Dict[str, np.ndarray]:
        flat = np.asarray(flat, dtype=np.float64)
        lead, out, o = flat.shape[:-1], {}, 0
        for l, (i, w) in enumerate(self._shapes()):
            out[f"w{l}"] = flat[..., o:o + i * w].reshape(lead + (i, w))
            o += i * w
            out[f"b{l}"] = flat[..., o:o + w]
            o += w
        return out

    def _set_data(self, X, y=None):
        """bnn.py:31-37: X [N] -> [N, 1]; y [N] -> [N, 1].  X must have input_dim columns and y output_dim columns, or one
        column, which is broadcast over the outputs as the reference's Normal(mu, noise) broadcasts it."""
        X = np.asarray(X, dtype=np.float64)
        X = X if X.ndim > 1 else X[:, None]
        if X.ndim != 2 or X.shape[1] != self.input_dim:
            raise ValueError(f"X has shape {X.shape}; the network takes {self.input_dim} input column(s)")
        if y is not None:
            y = np.asarray(y, dtype=np.float64)
            y = y[:, None] if y.ndim < 2 else y
            if y.ndim != 2 or y.shape[0] != X.shape[0] or y.shape[1] not in (1, self.output_dim):
                raise ValueError(f"y has shape {y.shape}; expected ({X.shape[0]}, {self.output_dim})")
            if y.shape[1] != self.output_dim:
                y = np.ascontiguousarray(np.broadcast_to(y, (y.shape[0], self.output_dim)))
            return X, y
        return X

    def _predict_draws(self, X, flat, sigma=None, eps=None):
        return self.ctx.bnn_predict(X, self.widths, _ffi.ACT_TANH, flat, sigma, eps)

    # ---- fit
    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None) -> None:
        """spm.py:88-130: NUTS over the weights and the noise, then `mu` on X_train.  chain_method "vectorized" runs the
        chains in lock-step, each round's likelihoods in one b2gp_bnn_loglik_draws call; any other value runs them one
        after another.  Both give the same samples bit for bit."""
        from .inference import MCMCResult, run_nuts
        X, y = self._set_data(X, y)
        self.X_train, self.y_train = X, y
        lj = BNNLogJoint(self, X, y, seed_from_key(rng_key))
        try:
            res = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        finally:
            lj.close()
        by_chain = res.get_samples(group_by_chain=True)
        C, S = by_chain["noise"].shape[:2]
        flat = self.to_flat({k: v.reshape((C * S,) + v.shape[2:]) for k, v in by_chain.items() if k != "noise"})
        mu, _ = self._predict_draws(X, flat)
        by_chain["mu"] = mu.reshape((C, S) + mu.shape[1:])
        self.mcmc = MCMCResult(by_chain, res.stats)
        if print_summary:
            self._print_summary()

    def get_samples(self, chain_dim: bool = False) -> Dict[str, np.ndarray]:
        """spm.py:132-134"""
        return self.mcmc.get_samples(group_by_chain=chain_dim)

    def get_param_means(self) -> Dict[str, object]:
        """spm.py:136-144: the mean over draws of every site but `mu`.  Scalar sites come back as floats and weight / bias
        sites as arrays; the reference calls `.item()` on every mean and so raises on the weight sites."""
        out = {}
        for k, v in self.get_samples().items():
            if k == "mu":
                continue
            m = np.asarray(v).mean(0)
            out[k] = float(m) if m.size == 1 and m.ndim == 0 else m
        return out

    # ---- prior and posterior predictive
    def sample_from_prior(self, rng_key, X, num_samples: int = 10) -> np.ndarray:
        """spm.py:146-150: y [num_samples, N, O] from the prior predictive.  Weights, biases and noise are drawn on the
        host from their priors (seeded from rng_key), mu and y = mu + noise * eps on the GPU."""
        X = self._set_data(X)
        rng = seed_from_key(rng_key)
        wmask = self._weight_mask()
        S = int(num_samples)
        flat = np.where(wmask, rng.standard_normal((S, wmask.size)), rng.standard_cauchy((S, wmask.size)))
        sigma = np.asarray(self._noise_prior().sample(rng, (S,)), dtype=np.float64)
        eps = rng.standard_normal((S, 1, X.shape[0], self.output_dim))
        _, y = self._predict_draws(X, flat, sigma, eps)
        return y

    def sample_single_posterior_predictive(self, rng_key, X_new, params, n_draws) -> Tuple[np.ndarray, np.ndarray]:
        """spm.py:152-156 for one draw of the sites: (loc [P, O], mean of n_draws Normal(loc, noise) samples [P, O]).  The
        standard normals are jax.random.normal(rng_key, (n_draws, P, O))."""
        X_new = self._set_data(X_new)
        Pn, O = X_new.shape[0], self.output_dim
        eps = posterior_eps(rng_key, 1, int(n_draws), Pn * O, _eps_dtype(), per_draw_keys=False)
        loc, y = self._predict_draws(X_new, self.to_flat(params), params["noise"], eps.reshape(1, -1, Pn, O))
        return loc[0], y[0]

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                take_point_predictions_mean: bool = True, device=None, noiseless: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        """spm.py:173-208: (mean over draws of loc [P, O], or loc [S, P, O] without take_point_predictions_mean; y_sampled
        [S, P, O]).  Draw s uses the s-th key of jax.random.split(rng_key, S) and jax.random.normal(key, (n, P, O)); the
        whole batch of draws is one b2gp_bnn_predict call.  noiseless=True (not in the reference; the analogue of the GP's
        noiseless predictive, which the acquisition functions pass on) returns y_sampled = loc: the network's output
        without the observation noise, and draws no normals."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        flat = np.atleast_2d(self.to_flat(samples))
        S, Pn, O = flat.shape[0], X_new.shape[0], self.output_dim
        if noiseless:
            y_pred, _ = self._predict_draws(X_new, flat)
            y_sampled = y_pred.copy()
        else:
            eps = posterior_eps(rng_key, S, int(n), Pn * O, _eps_dtype()).reshape(S, int(n), Pn, O)
            y_pred, y_sampled = self._predict_draws(X_new, flat, np.asarray(samples["noise"]).reshape(S), eps)
        if filter_nans:
            y_sampled = y_sampled[[i for i in range(S) if not np.isnan(y_sampled[i]).any()]]
        if take_point_predictions_mean:
            y_pred = y_pred.mean(0)
        return y_pred, y_sampled

    def _print_summary(self):
        s = self.get_samples()
        noise = np.asarray(s["noise"])
        print(f"{'noise':>12s}  mean {noise.mean():.4g}  std {noise.std():.4g}")
        st = self.mcmc.stats
        print(f"{'divergences':>12s}  {sum(c['divergences'] for c in st)}  step size {st[-1]['step_size']:.3g}")
