"""
spm.py -- `sPM`, the structured probabilistic model, with the reference's surface (gpax/models/spm.py:29-218).

A deterministic model `model(X, params)` of the system, priors over its parameters written as a prior program, and a
normal observation noise:

    params = model_prior()                          sites of the program (a, b, ...)
    mu     = model(X, params)                       deterministic site "mu"
    sigma  = sample("noise", LogNormal(0, 1))       or noise_prior_dist, or the deprecated noise_prior() program
    y      ~ Normal(mu, sigma)

`fit` samples the sites with the host NUTS of inference.run_nuts over SPMLogJoint.  Everything here runs on the host:
each evaluation is the caller's own Python `model`, which nothing compiled can replace, and the arithmetic around it is
O(N p) for the N of tens to hundreds of measurements this model serves (hypothesis learning, gpax_b200/hypo.py).  A
device round trip per evaluation would cost more than that arithmetic.

`X` reaches `model` exactly as it was passed -- a 1-D array stays 1-D (spm.py:213-218); unlike ExactGP nothing is
reshaped.  `device` is accepted and ignored.
"""
import math
import warnings
from typing import Callable, Dict, Optional, Tuple

import numpy as np

from . import priors as P
from .gp import _eps_dtype
from .inference import MCMCResult, ProgramLogJoint, run_nuts
from .utils import posterior_eps, seed_from_key

_HALF_LOG_2PI = 0.5 * math.log(2 * math.pi)


class SPMLogJoint(ProgramLogJoint):
    """log p(y, sites) of sPM.model (spm.py:63-77) over the unconstrained vector u of the prior program's sites:

      value = sum log N(y; model(X, params(u)), sigma(u))  +  sum_sites log p(site)  (+ log |d site / du|)

    Gradient.  d value / d sigma = sum ((r / sigma)^2 - 1) / sigma with r = y - mu, and d value / d mu = r / sigma^2, in
    closed form.  d sigma / du is the noise site's transform derivative (central differences of the program for the
    deprecated noise_prior program).  d mu / du_k of the model-prior coordinates are central differences of `model` over
    u with ProgramLogJoint's step: 2 model calls per coordinate.  Site densities as ProgramLogJoint (analytic, or
    differenced for hierarchical programs).  The sum broadcasts y against mu as Normal(mu, sigma).log_prob(y) does."""

    batch = None        # every evaluation is the caller's host Python: vectorized chains go row by row

    def __init__(self, spm, X, y):
        self.m, self.X = spm, X
        self.y = np.asarray(y, dtype=np.float64)
        self._find_sites()
        _, msites, _ = P.run_program(spm.model_prior)
        self.model_coord = np.concatenate([np.full(s.size, s.name in msites) for s in self.sites]) \
            if self.sites else np.zeros(0, dtype=bool)
        self.n_evals = 0

    def _model_program(self):
        return self.m._program()

    def _run(self, u):
        """u -> (the model's parameter dict, sigma, sites with values)"""
        (params, noise), sites, _ = P.run_program(self._model_program, self._site_values(u))
        return params, np.asarray(noise, dtype=np.float64), sites

    def mu(self, params):
        return np.asarray(self.m._model(self.X, params), dtype=np.float64)

    def mu_at(self, values):
        """mu for the site values of one draw ({name: value}): the program run at those values, then `model`"""
        (params, _), _, _ = P.run_program(self._model_program, values)
        return self.mu(params)

    def __call__(self, u, jacobian):
        u = np.asarray(u, dtype=np.float64)
        params, sigma, sites = self._run(u)
        self.n_evals += 1
        if not (np.all(np.isfinite(sigma)) and np.all(sigma > 0)):
            return -np.inf, np.zeros(self.dim)
        mu = self.mu(params)
        z = (self.y - mu) / sigma
        val = float(np.sum(-0.5 * z * z - np.log(sigma) - _HALF_LOG_2PI))
        if not np.isfinite(val):
            return -np.inf, np.zeros(self.dim)
        dmu = z / sigma                      # d value / d mu, on the broadcast shape
        dsigma = (z * z - 1.0) / sigma       # d value / d sigma, on the broadcast shape
        lp, grad = self._log_prior(u, sites, jacobian, want_grad=not self.hierarchical)
        h = self.FD_STEP
        o = 0
        for s in self.sites:
            for j in range(s.size):
                k = o + j
                if self.model_coord[k]:
                    e = np.zeros(self.dim)
                    e[k] = h
                    mp = self.mu(self._run(u + e)[0])
                    mm = self.mu(self._run(u - e)[0])
                    grad[k] += float(np.sum(dmu * (mp - mm) / (2 * h)))
                elif self.m.noise_prior:
                    e = np.zeros(self.dim)
                    e[k] = h
                    grad[k] += float(np.sum(dsigma * (self._run(u + e)[1] - self._run(u - e)[1]) / (2 * h)))
                else:                        # sigma is the "noise" site itself
                    ds = np.zeros(sigma.shape)
                    ds.flat[j] = float(s.prior.dtheta_du(u[k]))
                    grad[k] += float(np.sum(dsigma * ds))
            o += s.size
        if self.hierarchical:
            for k in range(self.dim):
                e = np.zeros(self.dim)
                e[k] = h
                lpp, _ = self._log_prior(u + e, self._run(u + e)[2], jacobian, want_grad=False)
                lpm, _ = self._log_prior(u - e, self._run(u - e)[2], jacobian, want_grad=False)
                grad[k] += (lpp - lpm) / (2 * h)
        return val + lp, grad


class sPM:
    """
    Structured probabilistic model (gpax/models/spm.py:29-218): `sPM(model, model_prior, noise_prior=None,
    noise_prior_dist=None)`.

    Args:
        model: deterministic model of the system, ``model(X, params) -> mu``
        model_prior: prior program over the model's parameters, written against gpax_b200.priors
            (``from gpax_b200 import priors as numpyro``); returns the ``params`` dict
        noise_prior: deprecated program returning the observation noise
        noise_prior_dist: prior of the "noise" site (a gpax_b200.priors distribution); LogNormal(0, 1) by default
    """

    def __init__(self, model: Callable, model_prior: Callable, noise_prior: Optional[Callable] = None,
                 noise_prior_dist=None) -> None:
        self._model = model
        self.model_prior = model_prior
        if noise_prior is not None:          # spm.py:51-58
            warnings.warn(
                "`noise_prior` is deprecated and will be removed in a future version. "
                "Please use `noise_prior_dist` instead, which accepts an instance of a "
                "numpyro.distributions Distribution object, e.g., `dist.HalfNormal(scale=0.1)`, "
                "rather than a function that calls `numpyro.sample`.",
                FutureWarning,
            )
        self.noise_prior = noise_prior
        self.noise_prior_dist = noise_prior_dist
        self.mcmc = None

    def _program(self):
        """the prior statements of spm.py:63-77 (everything but the likelihood): (params, noise)"""
        params = self.model_prior()
        if self.noise_prior:
            noise = self.noise_prior()
        else:
            noise = P.sample("noise", self.noise_prior_dist if self.noise_prior_dist is not None else P.LogNormal(0.0, 1.0))
        return params, noise

    def fit(self, rng_key, X, y, num_warmup: int = 2000, num_samples: int = 2000, num_chains: int = 1,
            chain_method: str = "sequential", progress_bar: bool = True, print_summary: bool = True, device=None) -> None:
        """spm.py:86-125: NUTS over the sites of the prior program and the noise (inference.run_nuts on SPMLogJoint,
        init_to_median), then the deterministic site `mu` = model(X, params) once per kept draw"""
        X, y = self._set_data(X, y)
        lj = SPMLogJoint(self, X, y)
        res = run_nuts(lj, rng_key, num_warmup, num_samples, num_chains, progress_bar, chain_method)
        by_chain = res.get_samples(group_by_chain=True)
        C, S = next(iter(by_chain.values())).shape[:2]
        mu = np.stack([lj.mu_at({k: v[c, s] for k, v in by_chain.items()}) for c in range(C) for s in range(S)])
        by_chain["mu"] = mu.reshape((C, S) + mu.shape[1:])
        self.mcmc = MCMCResult(by_chain, res.stats)
        if print_summary:
            self._print_summary()

    def get_samples(self, chain_dim: bool = False) -> Dict[str, np.ndarray]:
        """spm.py:127-129: the sites and `mu`, [S, ...] or by chain [C, S, ...]"""
        if self.mcmc is None:
            raise RuntimeError("no posterior samples: call fit() first or pass `samples=` to predict()")
        return self.mcmc.get_samples(group_by_chain=chain_dim)

    def get_param_means(self) -> Dict[str, float]:
        """spm.py:131-139: the mean over draws of every site but `mu`, as a Python scalar"""
        return {k: np.asarray(v).mean(0).item() for k, v in self.get_samples().items() if k != "mu"}

    def sample_from_prior(self, rng_key, X, num_samples: int = 10) -> np.ndarray:
        """spm.py:141-148: y [num_samples, ...mu's shape] from the prior predictive at X.  The sites are drawn from their
        priors and y = mu + noise * eps, all from NumPy's generator seeded from the key (the reference's distribution;
        NumPyro's key stream is not reproduced)."""
        rng = seed_from_key(rng_key)
        out = []
        for _ in range(int(num_samples)):
            (params, noise), _, _ = P.run_program(self._program, rng=rng)
            mu = np.asarray(self._model(X, params), dtype=np.float64)
            out.append(mu + np.asarray(noise, dtype=np.float64) * rng.standard_normal(mu.shape))
        return np.stack(out)

    def _loc(self, X_new, params):
        return np.asarray(self._model(X_new, params), dtype=np.float64)

    def sample_single_posterior_predictive(self, rng_key, X_new, params, n_draws) -> Tuple[np.ndarray, np.ndarray]:
        """spm.py:150-154 for one draw of the sites: (loc, mean of n_draws Normal(loc, noise) samples).  The standard
        normals are jax.random.normal(rng_key, (n_draws,) + loc.shape)."""
        loc = self._loc(X_new, params)
        eps = posterior_eps(rng_key, 1, int(n_draws), loc.size, _eps_dtype(), per_draw_keys=False)[0]
        return loc, loc + np.asarray(params["noise"], dtype=np.float64) * eps.mean(0).reshape(loc.shape)

    def predict(self, rng_key, X_new, samples: Optional[Dict[str, np.ndarray]] = None, n: int = 1, filter_nans: bool = False,
                take_point_predictions_mean: bool = True, device=None) -> Tuple[np.ndarray, np.ndarray]:
        """spm.py:173-208: (mean over draws of loc, or loc [S, ...] without take_point_predictions_mean; y_sampled
        [S, ...]).  Draw s gives loc_s = model(X_new, samples[s]) and y_s = loc_s + noise_s * (mean of n normals), the
        normals jax.random.normal(k_s, (n,) + loc.shape) of the s-th key of jax.random.split(rng_key, S).
        filter_nans drops the draws whose y_s has a NaN."""
        X_new = self._set_data(X_new)
        if samples is None:
            samples = self.get_samples(chain_dim=False)
        S = len(next(iter(samples.values())))
        locs = np.stack([self._loc(X_new, {k: np.asarray(v)[s] for k, v in samples.items()}) for s in range(S)])
        shape = locs.shape[1:]
        eps = posterior_eps(rng_key, S, int(n), int(np.prod(shape)), _eps_dtype())
        sigma = np.asarray(samples["noise"], dtype=np.float64).reshape((S,) + (1,) * len(shape))
        y_sampled = locs + sigma * eps.mean(1).reshape((S,) + shape)
        if filter_nans:
            y_sampled = y_sampled[[s for s in range(S) if not np.isnan(y_sampled[s]).any()]]
        y_pred = locs.mean(0) if take_point_predictions_mean else locs
        return y_pred, y_sampled

    def _print_summary(self):
        for k, v in self.get_samples(1).items():
            if k == "mu":
                continue
            v = np.asarray(v)
            print(f"{k:>12s}  mean {np.mean(v, axis=(0, 1))}  std {np.std(v, axis=(0, 1))}")

    def _set_data(self, X, y=None):
        """spm.py:213-218: X and y as they were passed, no reshaping"""
        if y is not None:
            return X, y
        return X
