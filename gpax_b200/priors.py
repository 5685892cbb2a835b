"""
priors.py -- prior distributions and prior *programs* for `.fit()`.

The reference passes numpyro.distributions objects (gpax/models/gp.py:222-247 defaults to LogNormal(0, 1) on k_length,
k_scale, noise, period) and, for `kernel_prior` / `noise_prior` / `mean_fn_prior`, functions that call `numpyro.sample`
(gp.py:141-154; tests/test_gp.py:29-38).  NumPyro is not a dependency here.  This module carries the two things those
call sites need:

* distributions with their support transform theta(u), so that inference runs on an unconstrained vector u as NumPyro's
  does;
* the effect primitives a prior program uses -- `sample`, `deterministic`, `plate`, and `distributions` as a namespace --
  so that the reference's programs run with one changed import:

      from gpax_b200 import priors as numpyro
      def mean_fn_prior():
          a = numpyro.sample("a", numpyro.distributions.LogNormal(0, 1))
          b = numpyro.sample("b", numpyro.distributions.Normal(3, 1))
          return {"a": a, "b": b}

  `run_program(fn, values)` executes such a function with the sample sites substituted (or at the prior medians) and
  returns what it returned together with the sites it visited; inference.LogJoint drives it.
"""
import math
import sys
import threading
from collections import OrderedDict

import numpy as np


class Prior:
    """theta = transform(u); log_prob is the density over theta."""
    positive = True
    shape = ()

    def expand(self, batch_shape):
        """numpyro's Distribution.expand: independent copies over a batch shape"""
        import copy
        c = copy.copy(self)
        c.shape = tuple(int(b) for b in batch_shape)
        return c

    def transform(self, u):            # theta(u); a leapfrog step far out may overflow to inf, which the log joint rejects
        with np.errstate(over="ignore"):
            return np.exp(u)

    def dtheta_du(self, u):
        with np.errstate(over="ignore"):
            return np.exp(u)

    def log_abs_jac(self, u):          # log |dtheta/du|
        return u

    def dlog_abs_jac(self, u):
        return np.ones_like(u)

    def inverse(self, theta):
        return np.log(theta)

    def median(self):
        raise NotImplementedError

    def log_prob(self, theta):
        raise NotImplementedError

    def dlog_prob(self, theta):
        raise NotImplementedError

    def sample(self, rng, shape=()):
        raise NotImplementedError


class LogNormal(Prior):
    def __init__(self, loc=0.0, scale=1.0):
        self.loc, self.scale = float(loc), float(scale)

    def median(self):
        return math.exp(self.loc)

    def log_prob(self, t):
        z = (np.log(t) - self.loc) / self.scale
        return -np.log(t) - 0.5 * z * z - math.log(self.scale) - 0.5 * math.log(2 * math.pi)

    def dlog_prob(self, t):
        return (-1.0 - (np.log(t) - self.loc) / self.scale ** 2) / t

    def sample(self, rng, shape=()):
        return np.exp(self.loc + self.scale * rng.standard_normal(shape))


class HalfNormal(Prior):
    def __init__(self, scale=1.0):
        self.scale = float(scale)

    def median(self):
        return 0.6744897501960817 * self.scale

    def log_prob(self, t):
        return 0.5 * math.log(2 / math.pi) - math.log(self.scale) - 0.5 * (t / self.scale) ** 2

    def dlog_prob(self, t):
        return -t / self.scale ** 2

    def sample(self, rng, shape=()):
        return np.abs(self.scale * rng.standard_normal(shape))


class Gamma(Prior):
    def __init__(self, concentration, rate=1.0):
        self.a, self.b = float(concentration), float(rate)

    def median(self):
        from scipy.stats import gamma
        return float(gamma.median(self.a, scale=1.0 / self.b))

    def log_prob(self, t):
        return self.a * math.log(self.b) - math.lgamma(self.a) + (self.a - 1) * np.log(t) - self.b * t

    def dlog_prob(self, t):
        return (self.a - 1) / t - self.b

    def sample(self, rng, shape=()):
        return rng.gamma(self.a, 1.0 / self.b, shape)


class Uniform(Prior):
    def __init__(self, low, high):
        self.low, self.high = float(low), float(high)

    def _sig(self, u):
        return 1.0 / (1.0 + np.exp(-u))

    def transform(self, u):
        return self.low + (self.high - self.low) * self._sig(u)

    def dtheta_du(self, u):
        s = self._sig(u)
        return (self.high - self.low) * s * (1 - s)

    def log_abs_jac(self, u):
        s = self._sig(u)
        return math.log(self.high - self.low) + np.log(s) + np.log1p(-s)

    def dlog_abs_jac(self, u):
        return 1.0 - 2.0 * self._sig(u)

    def inverse(self, theta):
        p = (theta - self.low) / (self.high - self.low)
        return np.log(p) - np.log1p(-p)

    def median(self):
        return 0.5 * (self.low + self.high)

    def log_prob(self, t):
        return np.full_like(np.asarray(t, dtype=float), -math.log(self.high - self.low))

    def dlog_prob(self, t):
        return np.zeros_like(np.asarray(t, dtype=float))

    def sample(self, rng, shape=()):
        return rng.uniform(self.low, self.high, shape)


class Normal(Prior):
    """real support: theta = u"""
    positive = False

    def __init__(self, loc=0.0, scale=1.0):
        self.loc, self.scale = float(loc), float(scale)

    def transform(self, u):
        return np.asarray(u, dtype=float) * 1.0

    def dtheta_du(self, u):
        return np.ones_like(np.asarray(u, dtype=float))

    def log_abs_jac(self, u):
        return np.zeros_like(np.asarray(u, dtype=float))

    def dlog_abs_jac(self, u):
        return np.zeros_like(np.asarray(u, dtype=float))

    def inverse(self, theta):
        return np.asarray(theta, dtype=float) * 1.0

    def median(self):
        return self.loc

    def log_prob(self, t):
        z = (t - self.loc) / self.scale
        return -0.5 * z * z - math.log(self.scale) - 0.5 * math.log(2 * math.pi)

    def dlog_prob(self, t):
        return -(t - self.loc) / self.scale ** 2

    def sample(self, rng, shape=()):
        return self.loc + self.scale * rng.standard_normal(shape)


class Exponential(Prior):
    def __init__(self, rate=1.0):
        self.rate = float(rate)

    def median(self):
        return math.log(2.0) / self.rate

    def log_prob(self, t):
        return math.log(self.rate) - self.rate * t

    def dlog_prob(self, t):
        return np.full_like(np.asarray(t, dtype=float), -self.rate)

    def sample(self, rng, shape=()):
        return rng.exponential(1.0 / self.rate, shape)


class HalfCauchy(Prior):
    def __init__(self, scale=1.0):
        self.scale = float(scale)

    def median(self):
        return self.scale

    def log_prob(self, t):
        return math.log(2.0 / math.pi) - math.log(self.scale) - np.log1p((t / self.scale) ** 2)

    def dlog_prob(self, t):
        return -2.0 * t / (self.scale ** 2 + t * t)

    def sample(self, rng, shape=()):
        return np.abs(self.scale * rng.standard_cauchy(shape))


class Cauchy(Normal):
    """real support, theta = u: the bias prior of DKL / viDKL (dkl.py:160-164, vidkl.py:96)"""

    def log_prob(self, t):
        z = (t - self.loc) / self.scale
        return -math.log(math.pi * self.scale) - np.log1p(z * z)

    def dlog_prob(self, t):
        z = (t - self.loc) / self.scale
        return -2.0 * z / (self.scale * (1.0 + z * z))

    def sample(self, rng, shape=()):
        return self.loc + self.scale * rng.standard_cauchy(shape)


# ---------------------------------------------------------------------------------------------- prior programs
distributions = sys.modules[__name__]      # `priors.distributions.LogNormal(...)`, as `numpyro.distributions.LogNormal(...)`
_tls = threading.local()


class Site:
    """one `sample` statement met while a program ran"""

    def __init__(self, name, prior, shape, value):
        self.name, self.prior, self.shape, self.value = name, prior, shape, value
        self.size = int(np.prod(shape)) if shape else 1


class _Run:
    def __init__(self, values, rng=None):
        self.values = values or {}
        self.rng = rng
        self.sites = OrderedDict()
        self.plates = []
        self.plate_dims = []
        self.deterministic = OrderedDict()


def _current():
    run = getattr(_tls, "run", None)
    if run is None:
        raise RuntimeError("priors.sample / plate / deterministic are only meaningful inside a prior program run by fit()")
    return run


def sample(name, fn, obs=None, rng_key=None, sample_shape=()):
    """numpyro.sample: inside a program run by `run_program`, returns the substituted value of the site (or the prior
    median when none was given) and records the site.  `obs` sites belong to the likelihood, which the GPU evaluates:
    a prior program must not contain them."""
    if obs is not None:
        raise NotImplementedError("observed sites are not part of a prior program")
    if not isinstance(fn, Prior):
        raise TypeError(f"site '{name}': priors must be gpax_b200.priors objects (numpyro distributions cannot be used here)")
    run = _current()
    if name in run.sites:
        raise ValueError(f"site '{name}' is sampled twice")
    shape = tuple(sample_shape) + (_plate_shape(run) if not fn.shape else ()) + tuple(fn.shape)
    if name in run.values:
        v = np.asarray(run.values[name], dtype=np.float64)
        if v.shape != shape:
            v = np.broadcast_to(v, shape) * 1.0
    elif run.rng is not None:
        v = np.asarray(fn.sample(run.rng, shape), dtype=np.float64)        # prior draw (numpyro's Predictive / seed handler)
    else:
        v = np.full(shape, float(fn.median()))
    v = v if shape else float(v)
    run.sites[name] = Site(name, fn, shape, v)
    return v


def deterministic(name, value):
    """numpyro.deterministic: recorded, returned unchanged"""
    _current().deterministic[name] = value
    return value


def _plate_shape(run):
    """batch shape of a scalar site inside the open plates: one leading dimension per plate, outermost first; when a
    plate names its `dim` (numpyro.plate(..., dim=-2)), NumPyro's layout -- the named dims at their place counted from the
    right, the others at the rightmost free places, size 1 elsewhere (mtgp.py:198-203 gives `period` the shape (L, 1))"""
    if all(dm is None for dm in run.plate_dims):
        return tuple(run.plates)
    rank = max([len(run.plates)] + [-dm for dm in run.plate_dims if dm is not None])
    shape = [1] * rank
    for size, dm in zip(run.plates, run.plate_dims):
        if dm is not None:
            shape[rank + dm] = size
    free = [i for i in range(rank - 1, -1, -1) if i not in {rank + dm for dm in run.plate_dims if dm is not None}]
    for size, dm in zip(run.plates, run.plate_dims):
        if dm is None:
            shape[free.pop(0)] = size
    return tuple(shape)


class plate:
    """numpyro.plate(name, size, dim=None): sample sites inside gain a batch dimension (gp.py:237 uses it for ARD)"""

    def __init__(self, name, size, dim=None, **_):
        self.name, self.size, self.dim = name, int(size), dim

    def __enter__(self):
        _current().plates.append(self.size)
        _current().plate_dims.append(self.dim)
        return np.arange(self.size)

    def __exit__(self, *exc):
        _current().plates.pop()
        _current().plate_dims.pop()
        return False


def run_program(fn, values=None, rng=None):
    """run `fn()` with its sample sites substituted from `values` (name -> array); sites without a value are set to their
    prior median, or -- with a numpy Generator `rng` -- drawn from their prior.  Returns (fn's result, sites, deterministics)"""
    prev = getattr(_tls, "run", None)
    _tls.run = run = _Run(values, rng)
    try:
        out = fn()
    finally:
        _tls.run = prev
    return out, run.sites, run.deterministic
